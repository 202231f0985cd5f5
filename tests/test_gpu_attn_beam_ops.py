"""The decode attention and the beam-search bookkeeping op by op against float64 / the oracle's bookkeeping (whole-model runs reach these
kernels only at a few shapes):

  gvd_op_attention             attn_partial_kernel<AJ> (AJ = 1..4 and the generic shared-memory path) with its fused last-CTA merge, and
                               attn_combine_kernel: every AttnArgs field the decode step sets
  gvd_op_beam_topk             beam_topk_kernel (log_softmax + K best, ties to the lower index)
  gvd_op_row_argmax            row_argmax_kernel
  gvd_op_beam_search_scripted  beam_topk -> beam_update -> beam_gather_rows -> row_argmax -> beam_finish, the sequence gvd_beam_decode runs,
                               on scripted logits / region scores, against beam_ref.scripted_search (pinned to the oracle in
                               test_beam_emulation.py)

Every case launches once per variant.  Outputs are allocated filled with a sentinel, so elements a kernel must not touch (the unused words
of the chunk records, the neighbours of a column window) are checked as well as the ones it must write."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from beam_ref import make_script, scripted_search, step_topk
from gvd_b200 import capi
from test_gpu_tcgen05 import _decode_f16x3

pytestmark = pytest.mark.gpu

NAN = float("nan")
MIN_VALUE = -1e8               # AttModel.py:29,66 (exact in fp32)
EPS32 = 2.0 ** -24
TANH_ERR = 4e-7                # max |tanh_mufu(x) - tanh(x)| (ex2.approx + rcp.approx)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rup(x, a):
    return (x + a - 1) // a * a


# ------------------------------------------------------------------------------------------------------------ a. decode attention
class _Attn:
    """One attention problem: B query rows over B / feat_div clips, features, weights and masks as the decode step holds them."""

    def __init__(self, B, R, T, A, H, RC, TC, feat_div=1, seed=0, mask_stride=False):
        g = _gen(seed)
        Bf = B // feat_div
        self.B, self.R, self.T, self.A, self.H, self.RC, self.TC, self.div = B, R, T, A, H, RC, TC, feat_div
        c = lambda t: t.cuda().contiguous()
        self.p_pool = c(torch.randn(Bf, R, A, generator=g) * 0.5)
        self.pool = c(torch.randn(Bf, R, H, generator=g))
        self.p_conv = c(torch.randn(Bf, T, A, generator=g) * 0.5)
        self.conv = c(torch.randn(Bf, T, H, generator=g))
        self.q = c(torch.randn(B, 2 * A, generator=g) * 0.5)
        self.w1 = c(torch.randn(A, generator=g) / A ** 0.5)
        self.w2 = c(torch.randn(A, generator=g) / A ** 0.5)
        self.b1 = c(torch.randn(1, generator=g) * 0.1)
        self.b2 = c(torch.randn(1, generator=g) * 0.1)
        am = (torch.rand(Bf, R + 1, generator=g) < 0.25).to(torch.uint8)
        om = (torch.rand(Bf, 3, R + 1, generator=g) < 0.25).to(torch.uint8)
        am[:, 0] = 1                                       # the legacy leading column is set and must be ignored
        om[:, :, 0] = 1
        if R > RC:
            am[0, 1:RC + 1] = 1                            # clip 0: a fully masked region chunk next to unmasked ones
        if Bf >= 2:
            am[Bf - 1, 1:] = 1                             # last clip: every proposal masked (uniform average, like the reference)
        self.att_mask = c(am)
        self.om_full = c(om)
        self.out_mask = self.om_full[:, 1] if mask_stride else c(om[:, 1])   # a step slice of a [Bf, S, R+1] mask, or a dense mask
        self.nch_r, self.nch_t = -(-R // RC), -(-T // TC)

    def run(self, q=None, q_part=None, q_bias=None, fused=True, ticket=None, x_ld=None, image=False):
        """Launch once; returns (z window, z buffer, x window, x buffer, image or None, partial records, ticket)."""
        B, R, H = self.B, self.R, self.H
        zbuf = torch.full((B, R + 5), NAN, device="cuda")
        xbuf = torch.full((B, x_ld or H), NAN, device="cuda")
        x = xbuf[:, H:2 * H] if x_ld else xbuf
        img = torch.full((B, 2 * _rup(H, 32)), -1, dtype=torch.int32, device="cuda") if image else None
        part = torch.full((B, self.nch_r + self.nch_t, H + 4), NAN, device="cuda")
        if fused and ticket is None:
            ticket = torch.zeros(B, dtype=torch.int32, device="cuda")
        if q is None and q_part is None:
            q = self.q
        capi.op_attention(self.p_pool, self.pool, self.p_conv, self.conv, self.w1, self.b1, self.w2, self.b2, self.att_mask, self.out_mask,
                          zbuf[:, :R], part, x, self.RC, self.TC, q=q, q_part=q_part, q_bias=q_bias, ticket=ticket if fused else None,
                          x_pk=img[:, :_rup(H, 32)] if image else None, feat_div=self.div)
        torch.cuda.synchronize()
        return zbuf[:, :R], zbuf, x, xbuf, img, part, ticket

    def reference(self, q=None):
        """fp64 core_step attention (oracle/gvd_oracle.py:205-216, AttModel.py:33-53 / :71-108): scores s [B,T], masked logits z [B,R]
        (softmax mask), z_out (also out_mask), x = att + att2, and the per-row features."""
        A = self.A
        d = lambda t: t.double()
        idx = torch.arange(self.B, device="cuda") // self.div
        q = d(self.q if q is None else q)
        s = torch.tanh(d(self.p_conv)[idx] + q[:, None, :A]) @ d(self.w1) + d(self.b1)
        z = torch.tanh(d(self.p_pool)[idx] + q[:, None, A:]) @ d(self.w2) + d(self.b2)
        z = z.masked_fill(self.att_mask[idx][:, 1:].bool(), MIN_VALUE)
        conv, pool = d(self.conv)[idx], d(self.pool)[idx]
        x = torch.einsum("bt,bth->bh", torch.softmax(s, 1), conv) + torch.einsum("br,brh->bh", torch.softmax(z, 1), pool)
        z_out = z.masked_fill(self.out_mask[idx][:, 1:].bool(), MIN_VALUE)
        return s, z, z_out, x, conv, pool

    def bars(self, q=None):
        """Error bars of a logit: the tanh_mufu error times ||w||_1, the fp32 rounding of p + q, and the fp32 sum (per-lane fmaf chain of
        A/32 terms, 5-level warp tree, bias)."""
        q = self.q if q is None else q
        A = self.A
        out = []
        for p, qq, w in ((self.p_conv, q[:, :A], self.w1), (self.p_pool, q[:, A:], self.w2)):
            pq = float(p.abs().max()) + float(qq.abs().max())
            out.append(float(w.abs().sum()) * (TANH_ERR + EPS32 * (pq + A / 32 + 8)))
        return out


def _chunk_ref(scores, feat, C):
    """fp64 chunk records of one branch: scores [B,N] split into chunks of C rows -> max m, sum of exp l, unnormalised weighted sum acc."""
    B, N = scores.shape
    nch = -(-N // C)
    pad = nch * C - N
    s = F.pad(scores, (0, pad), value=-float("inf")).view(B, nch, C)
    m = s.max(-1).values
    e = torch.exp(s - m[..., None])
    f = F.pad(feat, (0, 0, 0, pad)).view(B, nch, C, feat.shape[-1])
    return m, e.sum(-1), torch.einsum("bnc,bnch->bnh", e, f)


def _check_attention(P, z, zbuf, x, xbuf, img, part, tag, q=None):
    s, zm, z_out, x_ref, conv, pool = P.reference(q)
    bar_t, bar_r = P.bars(q)
    R, H = P.R, P.H
    # masked region logits: MIN_VALUE exactly where either mask is set, elsewhere within the bar; pad columns untouched
    masked = z_out == MIN_VALUE
    assert torch.equal(z.double()[masked], z_out[masked]), tag
    err_z = float((z.double() - z_out)[~masked].abs().max()) if (~masked).any() else 0.0
    assert err_z <= bar_r, (tag, err_z, bar_r)
    assert torch.isnan(zbuf[:, R:]).all(), tag
    # chunk records: region chunks first, then temporal; words 2..3 never written
    recs = [(0, P.nch_r, zm, pool, P.RC, bar_r), (P.nch_r, P.nch_r + P.nch_t, s, conv, P.TC, bar_t)]
    err_rec = 0.0
    for c0, c1, sc, feat, C, bar in recs:
        m, l, acc = _chunk_ref(sc, feat, C)
        got = part[:, c0:c1].double()
        fmax = float(feat.abs().max())
        em = float((got[..., 0] - m).abs().max())
        el = float(((got[..., 1] - l) / l).abs().max())
        ea = float(((got[..., 4:] - acc).abs() / (l[..., None] * fmax)).abs().max())
        assert em <= bar and el <= 2 * bar + 1e-6 * C and ea <= 2 * bar + 1e-6 * C, (tag, em, el, ea, bar)
        err_rec = max(err_rec, em, el, ea)
    assert torch.isnan(part[..., 2:4]).all(), tag
    # att + att2 at a relative bar: each softmax weight carries twice its logit bar, plus the fp32 merge
    fmax = max(float(conv.abs().max()), float(pool.abs().max()))
    err_x = float((x.double() - x_ref).abs().max()) / fmax
    bar_x = 2 * (bar_t + bar_r) + 1e-5
    assert err_x <= bar_x, (tag, err_x, bar_x)
    if xbuf.shape[1] > H:
        assert torch.isnan(xbuf[:, :H]).all() and torch.isnan(xbuf[:, 2 * H:]).all(), tag
    if img is not None:
        Hp = _rup(H, 32)
        val, _ = _decode_f16x3(img[:, :Hp].contiguous(), H, 4.0)
        xv = x.cpu().double().numpy()
        assert float(np.abs(val - xv).max()) <= 2.0 ** -20 * max(1.0, float(np.abs(xv).max())), tag
        assert bool((img[:, Hp:] == -1).all()), tag
    return err_z, bar_r, err_rec, err_x, bar_x


# B, R, T, A, H, RC, TC, feat_div
_ATT_CASES = [
    (5, 52, 10, 96, 248, 16, 16, 1),        # generic path (A not a multiple of 128), the planned chunks at B = 5
    (5, 52, 10, 128, 248, 16, 16, 1),       # AJ = 1
    (5, 52, 10, 256, 248, 7, 7, 1),         # AJ = 2, chunks below 16 rows, ragged
    (5, 52, 10, 384, 248, 16, 1, 1),        # AJ = 3, one temporal row per chunk
    (5, 52, 10, 512, 248, 16, 16, 1),       # AJ = 4
    (5, 52, 10, 132, 248, 16, 16, 1),       # generic path with a ragged 128-column tail
    (3, 129, 10, 512, 36, 128, 7, 1),       # H = 36: 9 active threads; one row in the last region chunk
    (2, 1, 1, 128, 36, 1, 1, 1),            # one region, one frame
    (3, 129, 480, 512, 1024, 80, 128, 1),   # T = 480, H = 1024
    (5, 1000, 480, 512, 1024, 16, 16, 1),   # full dimensions, the planned chunks at B = 5
    (100, 1000, 10, 512, 1024, 128, 16, 1), # the planned chunks at B = 100: ragged last region chunk (104 rows)
    (100, 1000, 480, 512, 1024, 128, 80, 1),  # ... at T = 480
    (128, 52, 10, 96, 248, 16, 16, 1),      # B = 128
    (12, 52, 10, 512, 1024, 16, 16, 3),     # beam rows: 3 query rows per clip, masks per clip
    (128, 13, 10, 256, 248, 7, 16, 4),
]


@pytest.mark.parametrize("B,R,T,A,H,RC,TC,div", _ATT_CASES, ids=["B%d-R%d-T%d-A%d-H%d-RC%d-TC%d-div%d" % c for c in _ATT_CASES])
def test_attention_against_fp64(B, R, T, A, H, RC, TC, div):
    """z_out, every chunk record and att + att2 against fp64 through the fused merge (x written as the middle third of a [B, 3H] buffer with
    its fp16x3 image, out_mask a step slice of a [B, 3, R+1] mask); then the same tickets relaunched, and the separate combine kernel: both
    bit-equal to the first launch; the tickets are back at 0 after each fused launch."""
    P = _Attn(B, R, T, A, H, RC, TC, div, seed=B * 7 + R + T + A + H + RC + TC, mask_stride=True)
    z, zbuf, x, xbuf, img, part, ticket = P.run(x_ld=3 * H, image=True)
    errs = _check_attention(P, z, zbuf, x, xbuf, img, part, "fused")
    print("attention B=%d R=%d T=%d A=%d H=%d RC=%d TC=%d div=%d: |z err| %.2e (bar %.2e), records %.2e, |x err|/max|f| %.2e (bar %.2e)"
          % ((B, R, T, A, H, RC, TC, div) + errs))
    assert bool((ticket == 0).all()), "the last CTA of a row must reset its ticket"
    z2, _, x2, _, _, part2, ticket2 = P.run(ticket=ticket)                  # same ticket buffer: the next decode step / graph replay
    assert ticket2 is ticket and bool((ticket == 0).all())
    assert torch.equal(z2, z) and torch.equal(x2, x) and torch.equal(part2[..., [0, 1]], part[..., [0, 1]])
    z3, _, x3, _, _, part3, _ = P.run(fused=False)                           # partial kernel + attn_combine_kernel
    assert torch.equal(z3, z) and torch.equal(x3, x), "fused merge and separate combine differ"
    assert torch.equal(part3[..., 4:], part[..., 4:])


@pytest.mark.parametrize("q_S", [1, 2, 3, 4])
@pytest.mark.parametrize("A", [96, 512])
def test_attention_query_from_split_k_planes(q_S, A):
    """The query as q_bias + q_part[0] + ... + q_part[q_S-1] summed inside the kernel: bit-equal to the same fp32 sum given as q, and the
    fp64 reference on the exact sum."""
    B, R, T, H = 7, 52, 10, 1024
    P = _Attn(B, R, T, A, H, 16, 16, seed=q_S + A)
    g = _gen(100 + q_S)
    q_part = (torch.randn(q_S, B, 2 * A, generator=g) * 0.3).cuda()
    q_bias = (torch.randn(2 * A, generator=g) * 0.3).cuda()
    q = q_bias.expand(B, 2 * A).clone()
    for s in range(q_S):                                   # the kernel's order: bias, then ascending planes
        q += q_part[s]
    z, zbuf, x, xbuf, img, part, _ = P.run(q_part=q_part, q_bias=q_bias, x_ld=3 * H)
    z_d, _, x_d, _, _, part_d, _ = P.run(q=q)
    assert torch.equal(z, z_d) and torch.equal(x, x_d) and torch.equal(part[..., 4:], part_d[..., 4:])
    errs = _check_attention(P, z, zbuf, x, xbuf, img, part, "q_part", q=q)
    print("attention q_S=%d A=%d: |z err| %.2e (bar %.2e), records %.2e, |x err|/max|f| %.2e (bar %.2e)" % ((q_S, A) + errs))


def test_attention_rejects_bad_arguments():
    P = _Attn(2, 13, 4, 128, 64, 16, 16, seed=1)
    with pytest.raises(capi.GvdError):                     # chunks hold at most 128 rows
        P.RC = 129
        P.run()
    P.RC = 16
    with pytest.raises(capi.GvdError):                     # the separate combine writes dense rows and no image
        P.run(fused=False, x_ld=3 * P.H)
    with pytest.raises(capi.GvdError):                     # q and q_part are exclusive
        P.run(q=P.q, q_part=P.q[None], q_bias=P.q[0])


# ------------------------------------------------------------------------------------------------------------ b. beam_topk / row_argmax
def _topk_rows(V, K, seed):
    """Rows of logits [n, V]: continuous values, values on a coarse grid (many exact ties, across warps too), rows with -inf words, rows
    with fewer than K finite words, an all -inf row."""
    rs = np.random.RandomState(seed)
    rows = [rs.randn(4, V) * 3, rs.randint(-3, 1, size=(8, V)) * 0.5]
    r = rs.randint(-6, 1, size=(4, V)) * 0.25
    r[rs.rand(4, V) < 0.3] = -np.inf
    r[:, 0] = -np.inf
    rows.append(r)
    few = np.full((2, V), -np.inf)
    for i in range(2):
        few[i, rs.choice(V, max(K - 1, 0), replace=False)] = rs.randint(-4, 5, size=max(K - 1, 0))
    rows += [few, np.full((1, V), -np.inf)]
    return np.concatenate(rows).astype(np.float32)


_TOPK_CASES = [(V, K) for V in (9, 255, 256, 257, 4905) for K in (1, 2, 3, 5, 8)] + [(K, K) for K in (1, 2, 3, 5, 8)]


@pytest.mark.parametrize("V,K", _TOPK_CASES)
def test_beam_topk_against_fp64(V, K):
    """topi exactly the stable descending order (ties to the lower index, -inf words after finite ones in index order); topv the fp64
    log_softmax of those words within 1e-5 (-inf / NaN where the reference has them).  Logits read at a pitch of V + 3."""
    x = _topk_rows(V, K, seed=V * 10 + K)
    n = x.shape[0]
    buf = torch.full((n, V + 3), NAN, device="cuda")
    buf[:, :V] = torch.from_numpy(x).cuda()
    topv, topi = capi.op_beam_topk(buf[:, :V], K)
    torch.cuda.synchronize()
    x64 = torch.from_numpy(x).double()
    lp = torch.log_softmax(x64, 1).numpy()
    ix = np.argsort(-x.astype(np.float64), axis=1, kind="stable")[:, :K]
    assert np.array_equal(topi.cpu().numpy(), ix)
    want = np.take_along_axis(lp, ix, axis=1)
    got = topv.cpu().double().numpy()
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[np.isinf(want)], want[np.isinf(want)])
    err = float(np.abs(got[fin] - want[fin]).max()) if fin.any() else 0.0
    assert err <= 1e-5, err


def test_beam_topk_all_nan_rows():
    """A row without one finite comparison (every logit NaN) ranks words 0 .. K-1 like a stable torch.sort(descending=True) (the default
    sort gives no order among equal NaNs); its log-probabilities are NaN.  Neighbouring ordinary rows are unaffected."""
    for V, K in ((9, 8), (257, 3), (4905, 5), (2, 1)):
        x = np.random.RandomState(V).randn(3, V).astype(np.float32)
        x[1] = np.nan
        t = torch.from_numpy(x).cuda()
        topv, topi = capi.op_beam_topk(t, K)
        torch.cuda.synchronize()
        ref = torch.sort(torch.from_numpy(x[1:2]), dim=1, descending=True, stable=True)[1][0, :K]
        assert topi[1].cpu().tolist() == list(range(K)) == ref.tolist()
        assert torch.isnan(topv[1]).all()
        ix = np.argsort(-x[[0, 2]], axis=1, kind="stable")[:, :K]
        assert np.array_equal(topi[[0, 2]].cpu().numpy(), ix)


def test_beam_topk_rejects_bad_beam_sizes():
    x = torch.zeros(2, 12, device="cuda")
    for V, K in ((12, 9), (5, 6), (12, 0)):
        with pytest.raises(capi.GvdError):
            capi.op_beam_topk(x[:, :V], K)


@pytest.mark.parametrize("R", [1, 13, 256, 257, 1000])
def test_row_argmax(R):
    """First index of the row maximum: ties (within a warp, across warps, at the last index), an all -inf row and an all-NaN row give 0."""
    rs = np.random.RandomState(R)
    z = np.concatenate([rs.randn(4, R), rs.randint(-3, 1, size=(8, R)) * 0.5, np.full((2, R), -np.inf), np.full((1, R), np.nan)])
    z[0, -1] = 100.0                                       # maximum at the last index
    if R > 40:
        z[1, [7, 39, R - 1]] = 50.0                        # a tie across warps
    z = z.astype(np.float32)
    buf = torch.full((z.shape[0], R + 2), NAN, device="cuda")
    buf[:, :R] = torch.from_numpy(z).cuda()
    idx = capi.op_row_argmax(buf[:, :R])
    torch.cuda.synchronize()
    want = np.argmax(np.where(np.isnan(z), -np.inf, z), axis=1)
    assert np.array_equal(idx.cpu().numpy(), want)
    assert want[-1] == 0 and want[-2] == 0 and want[-3] == 0
    assert np.array_equal(want[:-1], torch.argmax(torch.from_numpy(z[:-1]), 1).numpy())


# ------------------------------------------------------------------------------------------------------------ c. scripted beam search
_BEAM_CASES = [  # B, K, L, V, R
    (1, 2, 1, 9, 13), (1, 8, 64, 257, 13), (7, 3, 20, 257, 52), (7, 5, 2, 9, 13), (7, 8, 20, 8, 13), (7, 2, 64, 9, 1),
    (7, 8, 20, 4905, 13),
    (100, 2, 20, 257, 1000), (100, 3, 64, 257, 13), (100, 8, 20, 257, 13), (100, 5, 1, 9, 13)]


@pytest.mark.parametrize("kind", ["random", "ties", "eos", "no_eos"])
@pytest.mark.parametrize("B,K,L,V,R", _BEAM_CASES)
def test_scripted_beam_search(B, K, L, V, R, kind):
    """gvd_beam_decode's bookkeeping on a script, bit for bit against beam_ref: seq, att2 indices and every step's parents exactly, the
    log-probabilities bitwise (the same fp32 adds of the same beam_topk values).  beam_topk's word order on the script equals the
    reference's; the probe state ends as the composition of the per-step parents (reordered after every step but the last)."""
    logits, z = make_script(B, K, L, V, R, seed=B * 1000 + K * 100 + L + V, ties=kind == "ties", eos_at=L // 2 if kind == "eos" else None,
                            no_eos=kind in ("ties", "no_eos"))
    BK, H = B * K, 64
    lt, zt = torch.from_numpy(logits).cuda(), torch.from_numpy(z).cuda()
    topv, topi = capi.op_beam_topk(lt.view(L * BK, V), K)
    probe0 = torch.randn(BK, H, generator=_gen(B + K + L)).cuda()
    probe = probe0.clone()
    seq, lp, att, parents = capi.op_beam_search_scripted(lt, zt, probe, K)
    torch.cuda.synchronize()
    ys, ix = step_topk(logits.reshape(L * BK, V), K)
    assert np.array_equal(topi.cpu().numpy(), ix)
    assert float(np.abs(topv.cpu().numpy() - ys).max()) <= 1e-5
    topk = (topv.cpu().numpy().reshape(L, BK, K), topi.cpu().numpy().reshape(L, BK, K))
    rseq, rlp, ratt, rpar, ties = scripted_search(logits, z, K, L, topk=topk)
    assert np.array_equal(parents.cpu().numpy(), rpar)
    assert np.array_equal(seq.cpu().numpy(), rseq)
    assert np.array_equal(att.cpu().numpy(), ratt)
    assert np.array_equal(lp.cpu().numpy().view(np.int32), rlp.view(np.int32))
    base = (torch.arange(BK, device="cuda") // K) * K
    want = probe0
    for t in range(L - 1):
        want = want[base + parents[t].long()]
    assert torch.equal(probe, want)
    if kind == "ties" and L > 1 and K < V:
        assert ties > 0
    if kind == "no_eos" and K < V:
        assert not bool((seq[:, :-1] == 0).any())
    if kind == "eos" and K < V:
        assert bool((seq[:, L // 2] == 0).all())


def test_scripted_beam_search_rejects_bad_sizes():
    logits, z = make_script(2, 3, 65, 9, 13, seed=1)
    probe = torch.zeros(6, 64, device="cuda")
    with pytest.raises(capi.GvdError):                     # seq_length <= 64
        capi.op_beam_search_scripted(torch.from_numpy(logits).cuda(), torch.from_numpy(z).cuda(), probe, 3)
    logits, z = make_script(1, 9, 2, 20, 13, seed=2)
    with pytest.raises(capi.GvdError):                     # beam_size <= 8
        capi.op_beam_search_scripted(torch.from_numpy(logits).cuda(), torch.from_numpy(z).cuda(), torch.zeros(9, 64, device="cuda"), 9)
