"""NativeOps: the primitive set of gvd_b200.train.TrainStep on the device — every method is one (or a fixed few) C-ABI call(s) into
csrc/gvd_train.cu, dense products through the wgmma GEMM.  torch is used for device memory only (allocation, views, cat/stack,
dtype conversion of masks), never for arithmetic on float data.

EXPERIMENTAL: not yet run on a device (see train.py).  The mathematical definition of each method is the method of the same name
in tests/ops_ref.py; tests/test_gpu_zz_train.py compares them one by one.
"""
import ctypes

import torch

try:
    from . import capi
except ImportError:                        # drop-in layout: the package directory itself is on sys.path
    import capi

_vp, _ci, _ll, _cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
_SIGS = {
    "gvd_tr_ew": [_ci, _vp, _vp, _vp, _cf, _vp, _ll, _vp],
    "gvd_tr_outer_rows": [_vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_outer_rows_acc": [_vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_colsum": [_vp, _vp, _ci, _ll, _ci, _vp],
    "gvd_tr_rowsum": [_vp, _vp, _ll, _ci, _vp],
    "gvd_tr_sum_all": [_vp, _vp, _ll, _vp],
    "gvd_tr_mean_dim1": [_vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_ln_fwd": [_vp, _vp, _ll, _ci, _vp],
    "gvd_tr_ln_bwd": [_vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_ln_star_fwd": [_vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_ln_star_bwd": [_vp, _vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_softmax_fwd": [_vp, _cf, _vp, _ll, _ci, _vp],
    "gvd_tr_softmax_bwd": [_vp, _vp, _cf, _vp, _ll, _ci, _vp],
    "gvd_tr_lm_nll": [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_pos_nll": [_vp, _vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_cls_nll": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _ci, _vp],
    "gvd_tr_count_inv": [_vp, _ll, _ci, _vp, _vp],
    "gvd_tr_scalar_mul": [_vp, _vp, _vp, _vp],
    "gvd_tr_targets": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _ci, _ci, _vp, _vp, _vp, _vp, _vp],
    "gvd_tr_lstm_cell_fwd": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _vp],
    "gvd_tr_lstm_cell_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _vp],
    "gvd_tr_gru_cell_fwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _vp],
    "gvd_tr_gru_cell_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _vp],
    "gvd_tr_att_scores_fwd": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_att_scores_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_att_scores_mul_fwd": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_att_scores_mul_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_gather_rows": [_vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_index_add_rows": [_vp, _vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_bn_normalize": [_vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_bn_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ci, _vp],
    "gvd_tr_adam_first_step": [_vp, _vp, _cf, _cf, _cf, _cf, _cf, _vp, _ll, _vp],
    "gvd_tr_dropout": [_vp, _vp, _ll, _cf, _ll, _ci, _ll, _vp],
    "gvd_tr_grad_norm": [_vp, _ll, _cf, _vp, _vp, _vp],
    "gvd_tr_adam_flat": [_vp, _vp, _vp, _vp, _ll, _vp, _vp, _ci, _vp, _cf, _cf, _cf, _cf, _ci, _vp],
    "gvd_tr_sgd_flat": [_vp, _vp, _vp, _ll, _vp, _vp, _vp, _ci, _vp, _cf, _cf, _vp],
    "gvd_tr_adamax_flat": [_vp, _vp, _vp, _vp, _ll, _vp, _vp, _vp, _ci, _vp, _cf, _cf, _cf, _cf, _vp],
    "gvd_tr_gemm_nt_batched": [_vp, _ll, _ll, _vp, _ll, _ll, _vp, _ll, _ll, _ci, _ci, _ci, _ci, _vp],
    "gvd_tr_transpose": [_vp, _vp, _ci, _ci, _ci, _vp],
    "gvd_tr_mha_fwd": [_vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _ci, _ci, _cf, _cf, _ll, _ci, _ll, _vp],
    "gvd_tr_mha_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _ci, _ci, _cf, _cf, _ll, _ci, _ll, _vp],
}
_bound = False


def _L():
    global _bound
    L = capi.lib()
    if not _bound:
        for name, sig in _SIGS.items():
            getattr(L, name).argtypes = sig
        L.gvd_tr_sumsq_scratch_bytes.restype = ctypes.c_size_t
        _bound = True
    return L


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _f(t):
    """fp32, contiguous, on the device (memory plumbing only)."""
    if t.dtype != torch.float32 or not t.is_cuda:
        raise capi.GvdError("NativeOps expects fp32 CUDA tensors, got %s on %s" % (t.dtype, t.device))
    return t if t.is_contiguous() else t.contiguous()


def _inv(n):
    """1 / count of a mean; an empty set gives NaN like torch's mean over nothing (the reference's empty-positive-set quirk)."""
    return 1.0 / n if n else float("nan")


def _pad_last(t, mult=4):
    k = t.shape[-1]
    if k % mult == 0:
        return t
    out = torch.zeros(*t.shape[:-1], (k + mult - 1) // mult * mult, dtype=t.dtype, device=t.device)
    out[..., :k] = t
    return out


class NativeOps:
    def __init__(self):
        if not torch.cuda.is_available():
            raise capi.GvdError("gvd_b200 has no CPU path: NativeOps needs a CUDA device")
        self.device = torch.device("cuda")
        self.L = _L()

    def _st(self):
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _new(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.device)

    # ---- plumbing
    def to_device(self, t): return t.to(self.device)
    def to_host(self, t): return t.detach().cpu()
    def zeros(self, shape): return torch.zeros(shape, dtype=torch.float32, device=self.device)
    def cat(self, ts, dim): return torch.cat([t for t in ts], dim=dim)
    def stack1(self, ts): return torch.stack(list(ts), dim=1)

    # ---- dense algebra (wgmma / CUDA-core GEMM of the library; contraction length padded to a multiple of 4 with zeros)
    def _gemm(self, A, W, batch):
        """A [batch, M, K], W [batch, N, K] -> [batch, M, N]"""
        A, W = _pad_last(_f(A)), _pad_last(_f(W))
        b, M, K = A.shape
        N = W.shape[1]
        C = self._new(b, M, N)
        capi.check(self.L.gvd_tr_gemm_nt_batched(_p(A), K, M * K, _p(W), K, N * K, _p(C), N, M * N, M, N, K, b, self._st()))
        return C

    def _t(self, x):
        """batched transpose [b, R, C] -> [b, C, R]"""
        x = _f(x)
        b, R, C = x.shape
        out = self._new(b, C, R)
        capi.check(self.L.gvd_tr_transpose(_p(x), _p(out), b, R, C, self._st()))
        return out

    def lin(self, x, W, b, relu):
        x2 = _pad_last(_f(x).reshape(-1, x.shape[-1]))
        Wp = _pad_last(_f(W))
        y = capi.op_linear(x2, Wp, _f(b) if b is not None else None, 1 if relu else 0, tc=False)
        return y.reshape(*x.shape[:-1], W.shape[0])

    def mm_nn(self, A, B): return self._gemm(A.unsqueeze(0), self._t(B.unsqueeze(0)), 1)[0]
    def mm_tn(self, A, B): return self._gemm(self._t(A.unsqueeze(0)), self._t(B.unsqueeze(0)), 1)[0]
    def bmm_nt(self, A, B): return self._gemm(A, B, A.shape[0])
    def bmm_nn(self, A, B): return self._gemm(A, self._t(B), A.shape[0])
    def bmm_tn(self, A, B): return self._gemm(self._t(A), self._t(B), A.shape[0])

    def colsum(self, x):
        x = _f(x)
        out = self._new(x.shape[1])
        capi.check(self.L.gvd_tr_colsum(_p(x), _p(out), 1, x.shape[0], x.shape[1], self._st()))
        return out

    def rowsum(self, x):
        x = _f(x)
        out = self._new(x.shape[0])
        capi.check(self.L.gvd_tr_rowsum(_p(x), _p(out), x.shape[0], x.shape[1], self._st()))
        return out

    def sum_all(self, x):
        x = _f(x)
        out = self._new(1)
        capi.check(self.L.gvd_tr_sum_all(_p(x), _p(out), x.numel(), self._st()))
        return out

    def mean_dim1(self, x):
        x = _f(x)
        out = self._new(x.shape[0], x.shape[2])
        capi.check(self.L.gvd_tr_mean_dim1(_p(x), _p(out), x.shape[0], x.shape[1], x.shape[2], self._st()))
        return out

    # ---- element-wise
    def _ew(self, op, a, b=None, mask=None, s=0.0):
        a = _f(a)
        if b is not None:
            b = _f(b)
            if b.shape != a.shape:
                raise capi.GvdError("element-wise operands differ in shape: %s vs %s" % (tuple(a.shape), tuple(b.shape)))
        if mask is not None:
            mask = mask.to(torch.uint8).contiguous()
            if mask.shape != a.shape:
                raise capi.GvdError("mask shape %s != %s" % (tuple(mask.shape), tuple(a.shape)))
        out = torch.empty_like(a)
        capi.check(self.L.gvd_tr_ew(op, _p(a), _p(b), _p(mask), float(s), _p(out), a.numel(), self._st()))
        return out

    def add(self, a, b): return self._ew(0, a, b)
    def mul(self, a, b): return self._ew(1, a, b)
    def scale(self, a, s): return self._ew(2, a, s=s)
    def relu(self, x): return self._ew(3, x)
    def relu_bwd(self, dy, y): return self._ew(4, dy, y)
    def masked_fill(self, x, mask, v): return self._ew(5, x, mask=mask, s=v)

    def dropout(self, x, p, seed, site, step):
        """x * Bernoulli(1 - p) / (1 - p) with the Philox mask of (seed, site, step); applied to a gradient it is the backward."""
        x = _f(x)
        y = torch.empty_like(x)
        capi.check(self.L.gvd_tr_dropout(_p(x), _p(y), x.numel(), float(p), int(seed), int(site), int(step), self._st()))
        return y

    def outer_rows(self, a, v):
        a, v = _f(a), _f(v)
        out = self._new(a.shape[0], a.shape[1], v.shape[1])
        capi.check(self.L.gvd_tr_outer_rows(_p(a), _p(v), _p(out), a.shape[0], a.shape[1], v.shape[1], self._st()))
        return out

    def outer_rows_acc_(self, acc, a, v):
        """acc[b,n,:] += a[b,n] * v[b,:] in place (acc is a buffer owned by the backward pass)."""
        a, v = _f(a), _f(v)
        if not acc.is_contiguous() or acc.shape != (a.shape[0], a.shape[1], v.shape[1]):
            raise capi.GvdError("outer_rows_acc_: accumulator must be a contiguous [B,N,H] buffer")
        if v.shape[1] % 4:
            acc.copy_(self.add(acc, self.outer_rows(a, v)))
            return acc
        capi.check(self.L.gvd_tr_outer_rows_acc(_p(a), _p(v), _p(acc), a.shape[0], a.shape[1], v.shape[1], self._st()))
        return acc

    # ---- normalisations / softmax (rows = everything but the last dim)
    def ln(self, x):
        x = _f(x)
        y = torch.empty_like(x)
        capi.check(self.L.gvd_tr_ln_fwd(_p(x), _p(y), x.numel() // x.shape[-1], x.shape[-1], self._st()))
        return y

    def ln_bwd(self, dy, y, x):
        dy, y, x = _f(dy), _f(y), _f(x)
        dx = torch.empty_like(x)
        capi.check(self.L.gvd_tr_ln_bwd(_p(dy), _p(y), _p(x), _p(dx), x.numel() // x.shape[-1], x.shape[-1], self._st()))
        return dx

    def ln_star(self, x, g, b):
        x = _f(x)
        y = torch.empty_like(x)
        capi.check(self.L.gvd_tr_ln_star_fwd(_p(x), _p(_f(g)), _p(_f(b)), _p(y), x.numel() // x.shape[-1], x.shape[-1], self._st()))
        return y

    def ln_star_bwd(self, dy, x, gamma):
        dy, x = _f(dy), _f(x)
        n = x.shape[-1]
        dx, tmp = torch.empty_like(x), torch.empty_like(x)
        capi.check(self.L.gvd_tr_ln_star_bwd(_p(dy), _p(x), _p(_f(gamma)), _p(dx), _p(tmp), x.numel() // n, n, self._st()))
        return dx, self.colsum(tmp.reshape(-1, n)), self.colsum(dy.reshape(-1, n))

    def softmax(self, x, scale):
        x = _f(x)
        p = torch.empty_like(x)
        capi.check(self.L.gvd_tr_softmax_fwd(_p(x), float(scale), _p(p), x.numel() // x.shape[-1], x.shape[-1], self._st()))
        return p

    def softmax_bwd(self, dp, p, scale):
        dp, p = _f(dp), _f(p)
        dx = torch.empty_like(p)
        capi.check(self.L.gvd_tr_softmax_bwd(_p(dp), _p(p), float(scale), _p(dx), p.numel() // p.shape[-1], p.shape[-1], self._st()))
        return dx

    def bn_train(self, e):
        e = _f(e)
        M, N = e.shape
        mu = self.scale(self.colsum(e), 1.0 / M)
        cen = self.add(e, self.scale(mu, -1.0).unsqueeze(0).expand(M, N).contiguous())
        var = self.scale(self.colsum(self.mul(cen, cen)), 1.0 / M)
        out = torch.empty_like(e)
        capi.check(self.L.gvd_tr_bn_normalize(_p(e), _p(mu), _p(var), _p(out), M, N, self._st()))
        return out, var

    def bn_train_bwd(self, dxh, e_hat, var):
        dxh, e_hat = _f(dxh), _f(e_hat)
        M, N = dxh.shape
        s1, s2 = self.colsum(dxh), self.colsum(self.mul(dxh, e_hat))
        de = torch.empty_like(dxh)
        capi.check(self.L.gvd_tr_bn_bwd(_p(dxh), _p(e_hat), _p(_f(var)), _p(s1), _p(s2), _p(de), M, N, self._st()))
        return de

    # ---- recurrent cells
    def lstm_cell(self, gates, c):
        gates, c = _f(gates), _f(c)
        B, H = c.shape
        h2, c2, act = torch.empty_like(c), torch.empty_like(c), torch.empty_like(gates)
        capi.check(self.L.gvd_tr_lstm_cell_fwd(_p(gates), _p(c), _p(h2), _p(c2), _p(act), B, H, self._st()))
        return h2, c2, act

    def lstm_cell_bwd(self, dh2, dc2, act, c, c2):
        B, H = c.shape
        dgates, dc = torch.empty_like(act), torch.empty_like(c)
        capi.check(self.L.gvd_tr_lstm_cell_bwd(_p(_f(dh2)), _p(_f(dc2)), _p(_f(act)), _p(_f(c)), _p(_f(c2)), _p(dgates), _p(dc), B, H, self._st()))
        return dgates, dc

    def gru_cell(self, gi, gh, h):
        gi, gh, h = _f(gi), _f(gh), _f(h)
        B, G = h.shape
        h2, r, z, n = (torch.empty_like(h) for _ in range(4))
        capi.check(self.L.gvd_tr_gru_cell_fwd(_p(gi), _p(gh), _p(h), _p(h2), _p(r), _p(z), _p(n), B, G, self._st()))
        return h2, r, z, n

    def gru_cell_bwd(self, dh, r, z, n, h, ghn):
        B, G = h.shape
        dgi, dgh, keep = self._new(B, 3 * G), self._new(B, 3 * G), self._new(B, G)
        capi.check(self.L.gvd_tr_gru_cell_bwd(_p(_f(dh)), _p(_f(r)), _p(_f(z)), _p(_f(n)), _p(_f(h)), _p(_f(ghn)), _p(dgi), _p(dgh), _p(keep), B, G,
                                              self._st()))
        return dgi, dgh, keep

    # ---- additive attention scores
    def att_scores(self, p, q, w, b):
        p, q = _f(p), _f(q)
        B, N, A = p.shape
        s = self._new(B, N)
        capi.check(self.L.gvd_tr_att_scores_fwd(_p(p), _p(q), _p(_f(w).reshape(-1)), _p(_f(b).reshape(-1)), _p(s), B, N, A, self._st()))
        return s

    def att_scores_bwd(self, ds, p, q, w):
        ds, p, q = _f(ds), _f(p), _f(q)
        B, N, A = p.shape
        dpre, dst = torch.empty_like(p), torch.empty_like(p)
        capi.check(self.L.gvd_tr_att_scores_bwd(_p(ds), _p(p), _p(q), _p(_f(w).reshape(-1)), _p(dpre), _p(dst), B, N, A, self._st()))
        dq = self._new(B, A)
        capi.check(self.L.gvd_tr_colsum(_p(dpre), _p(dq), B, N, A, self._st()))            # per clip: sum over the N rows
        return dpre, dq, self.colsum(dst.reshape(B * N, A)), self.sum_all(ds)

    # ---- multiplicative attention scores (region_attn_mode 'mix_mul')  s[b,n] = w . tanh(p[b,n,:] * q[b,:]) + b
    def att_scores_mul(self, p, q, w, b):
        p, q = _f(p), _f(q)
        B, N, A = p.shape
        s = self._new(B, N)
        capi.check(self.L.gvd_tr_att_scores_mul_fwd(_p(p), _p(q), _p(_f(w).reshape(-1)), _p(_f(b).reshape(-1)), _p(s), B, N, A, self._st()))
        return s

    def att_scores_mul_bwd(self, ds, p, q, w):
        """(dp, dq, dw, db): the per-element terms come from one kernel, their sums from the deterministic colsum kernel (no atomics)."""
        ds, p, q = _f(ds), _f(p), _f(q)
        B, N, A = p.shape
        dp, dqt, dst = torch.empty_like(p), torch.empty_like(p), torch.empty_like(p)
        capi.check(self.L.gvd_tr_att_scores_mul_bwd(_p(ds), _p(p), _p(q), _p(_f(w).reshape(-1)), _p(dp), _p(dqt), _p(dst), B, N, A, self._st()))
        dq = self._new(B, A)
        capi.check(self.L.gvd_tr_colsum(_p(dqt), _p(dq), B, N, A, self._st()))             # per clip: sum over the N rows
        return dp, dq, self.colsum(dst.reshape(B * N, A)), self.sum_all(ds)

    # ---- embeddings
    def gather_rows(self, table, idx):
        table = _f(table)
        idx = idx.to(torch.int64).contiguous()
        out = self._new(idx.numel(), table.shape[1])
        capi.check(self.L.gvd_tr_gather_rows(_p(table), _p(idx), _p(out), idx.numel(), table.shape[1], self._st()))
        return out

    def index_add_rows(self, n_rows, idx, rows):
        rows = _f(rows)
        idx = idx.to(torch.int64).contiguous()
        out = self._new(n_rows, rows.shape[1])
        capi.check(self.L.gvd_tr_index_add_rows(_p(idx), _p(rows), _p(out), n_rows, rows.shape[0], rows.shape[1], self._st()))
        return out

    # ---- multi-head attention of the transformer captioner's decoder (csrc/gvd_tfm_train.cu)
    def mha_fwd(self, q, k, v, causal, scale, p=0.0, seed=0, site_base=0, step=0):
        """q [B, Lq, H], k / v [B, N, H] -> (o [B, Lq, H], lse [B, heads, Lq]); p > 0: per-head probability dropout at site site_base + head."""
        q, k, v = _f(q), _f(k), _f(v)
        B, Lq, H = q.shape
        N = k.shape[1]
        if k.shape != (B, N, H) or v.shape != (B, N, H):
            raise capi.GvdError("mha_fwd: q %s, k %s, v %s" % (tuple(q.shape), tuple(k.shape), tuple(v.shape)))
        c = -(-H // 6)                                                                      # torch.chunk(6, -1) column ranges
        o, lse = torch.empty_like(q), self._new(B, -(-H // c), Lq)
        capi.check(self.L.gvd_tr_mha_fwd(_p(q), _p(k), _p(v), _p(o), _p(lse), B, Lq, N, H, 1 if causal else 0, float(scale), float(p), int(seed),
                                         int(site_base), int(step), self._st()))
        return o, lse

    def mha_bwd(self, do, q, k, v, o, lse, causal, scale, p=0.0, seed=0, site_base=0, step=0):
        """-> (dq, dk, dv) for the upstream gradient do of mha_fwd's o (same dropout arguments: the masks are regenerated)."""
        q, k, v, o, do, lse = _f(q), _f(k), _f(v), _f(o), _f(do), _f(lse)
        B, Lq, H = q.shape
        N = k.shape[1]
        if do.shape != q.shape or o.shape != q.shape or k.shape != (B, N, H) or v.shape != (B, N, H):
            raise capi.GvdError("mha_bwd: shapes differ from the forward's")
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        capi.check(self.L.gvd_tr_mha_bwd(_p(q), _p(k), _p(v), _p(o), _p(do), _p(lse), _p(dq), _p(dk), _p(dv), B, Lq, N, H, 1 if causal else 0,
                                         float(scale), float(p), int(seed), int(site_base), int(step), self._st()))
        return dq, dk, dv

    # ---- loss heads (value + gradient for d(loss) = 1); the 1/n of every masked mean stays on the device: no host round trip
    def _count_inv(self, t):
        inv = self._new(1)
        capi.check(self.L.gvd_tr_count_inv(_p(t), t.numel(), t.element_size(), _p(inv), self._st()))
        return inv

    def _smul(self, a, b):
        out = self._new(1)
        capi.check(self.L.gvd_tr_scalar_mul(_p(a), _p(b), _p(out), self._st()))
        return out

    def lm_nll(self, logits, target, txt_mask):
        logits = _f(logits)
        B, S, V = logits.shape
        m8 = txt_mask.to(torch.uint8).contiguous()
        inv = self._count_inv(m8)
        rowloss, d = self._new(B * S), torch.empty_like(logits)
        capi.check(self.L.gvd_tr_lm_nll(_p(logits), _p(target.to(torch.int64).contiguous()), _p(m8), _p(inv), _p(rowloss), _p(d), B * S, V, self._st()))
        return self._smul(self.sum_all(rowloss), inv), d

    def pos_nll(self, x, pos):
        x = _f(x)
        p8 = pos.to(torch.uint8).contiguous()
        inv = self._count_inv(p8)
        rows, cols = x.numel() // x.shape[-1], x.shape[-1]
        rowloss, dx = self._new(rows), torch.empty_like(x)
        capi.check(self.L.gvd_tr_pos_nll(_p(x), _p(p8), _p(inv), _p(rowloss), _p(dx), rows, cols, self._st()))
        return self._smul(self.sum_all(rowloss), inv), dx

    def cls_nll(self, simT, cls_target):
        simT = _f(simT)
        B, R, C = simT.shape
        tgt = cls_target.to(torch.int32).contiguous()                                       # B, NB, R
        NB = tgt.shape[1]
        inv = self._count_inv(tgt)
        part, d = self._new(B * NB * R), torch.empty_like(simT)
        capi.check(self.L.gvd_tr_cls_nll(_p(simT), _p(tgt), _p(inv), _p(part), _p(d), B, R, NB, C, self._st()))
        return self._smul(self.sum_all(part), inv), d

    # ---- optimiser
    def adam_first_step(self, w, g, coef, lr, b1, b2, eps):
        w, g = _f(w), _f(g).reshape(w.shape)
        out = torch.empty_like(w)
        capi.check(self.L.gvd_tr_adam_first_step(_p(w), _p(g), float(coef), float(lr), float(b1), float(b2), float(eps), _p(out), w.numel(), self._st()))
        return out

    # ---- flat-buffer optimiser (no host round trip: the clip coefficient stays on the device)
    def grad_norm_(self, flat_g, max_norm, norm_out):
        """norm_out[0] = ||flat_g||_2, norm_out[1] = min(max_norm / (norm + 1e-6), 1)   (clip_grad_norm_, main.py:265)"""
        if getattr(self, "_sq_scratch", None) is None:
            self._sq_scratch = torch.empty(int(self.L.gvd_tr_sumsq_scratch_bytes()), dtype=torch.uint8, device=self.device)
        capi.check(self.L.gvd_tr_grad_norm(_p(_f(flat_g)), flat_g.numel(), float(max_norm), _p(self._sq_scratch), _p(norm_out), self._st()))

    def adam_flat_(self, w, g, m, v, seg_end, seg_lr, norm, b1, b2, eps, weight_decay, t):
        """One torch.optim.Adam step on flat buffers, in place (w, m, v updated; g clipped by norm[1])."""
        capi.check(self.L.gvd_tr_adam_flat(_p(w), _p(g), _p(m), _p(v), w.numel(), _p(seg_end), _p(seg_lr), seg_end.numel(),
                                           _p(norm) if norm is not None else None, float(b1), float(b2), float(eps), float(weight_decay), int(t),
                                           self._st()))

    def sgd_flat_(self, w, g, buf, seg_end, seg_lr, seg_step, norm, momentum, weight_decay):
        """One torch.optim.SGD(momentum) step on flat buffers, in place (w, buf, seg_step updated; g clipped by norm[1])."""
        capi.check(self.L.gvd_tr_sgd_flat(_p(w), _p(g), _p(buf), w.numel(), _p(seg_end), _p(seg_lr), _p(seg_step), seg_end.numel(),
                                          _p(norm) if norm is not None else None, float(momentum), float(weight_decay), self._st()))

    def adamax_flat_(self, w, g, m, u, seg_end, seg_lr, seg_step, norm, b1, b2, eps, weight_decay):
        """One torch.optim.Adamax step on flat buffers, in place (w, m, u, seg_step updated; g clipped by norm[1])."""
        capi.check(self.L.gvd_tr_adamax_flat(_p(w), _p(g), _p(m), _p(u), w.numel(), _p(seg_end), _p(seg_lr), _p(seg_step), seg_end.numel(),
                                             _p(norm) if norm is not None else None, float(b1), float(b2), float(eps), float(weight_decay),
                                             self._st()))

    # ---- integer / mask targets of the teacher forcing, on the device (gvd_losses.cu kernels)
    def host_targets(self, step, opt, inp, host):
        ppls, gt = _f(inp["ppls"]), _f(inp["gt_boxes"])
        B, R, _ = ppls.shape
        NB = gt.shape[1]
        L1 = opt.seq_length + 1
        S = opt.seq_length
        frm = inp["frm_mask"].to(torch.uint8).contiguous()
        pnt = inp["pnt_mask"].to(torch.uint8).contiguous()
        mb = inp["mask_boxes"][:, 0].to(torch.uint8).contiguous()                           # B, NB, L+1
        ov = self._new(B, R, NB)
        cls_target = torch.empty(B, NB, R, dtype=torch.int32, device=self.device)
        labels = torch.empty(B, S, R, dtype=torch.uint8, device=self.device)
        fm = torch.empty(B, S, R + 1, dtype=torch.uint8, device=self.device)
        capi.check(self.L.gvd_tr_targets(_p(ppls), _p(gt), _p(frm), _p(pnt), _p(mb), B, R, NB, S, L1, _p(ov), _p(cls_target), _p(labels), _p(fm),
                                         self._st()))
        fmb = fm[:, :, 1:].bool()
        return dict(cls_target=cls_target, labels=labels.bool(), fm=[fmb[:, i].contiguous() for i in range(S)], fm_all=fmb.contiguous())
