"""The decode step's default path and the tensor-core GRU layer, op by op against float64 (whole-model runs reach these kernels only
at a handful of batch sizes and two vocabulary sizes):

  gvd_op_skinny_partials   wg_gemm_kernel MODE_TRANS + ksplit: operand-swapped, split along K (3xTF32, in-kernel fp16x3, fp16x3 images)
  gvd_op_reduce_lstm / gvd_op_reduce_bias / gvd_op_reduce_pick        the three reductions of the partial planes
  gvd_op_greedy_pick, gvd_op_reduce_pick, gvd_op_logit_pick_tc        three implementations of one sampling rule (sampler_ref.py)
  gvd_op_gru_layer         MODE_GRU layer kernel and the per-step GEMM + pointwise loop

Every case launches once.  Outputs are allocated filled with a sentinel, so an element a kernel must not touch (pad columns of the
partial planes, the neighbours of a column window inside a concatenated buffer) is checked as well as the ones it must write."""
import numpy as np
import pytest
import torch

from gvd_b200 import capi
from sampler_ref import pick_reference, special_rows, top2_gap
from test_gpu_tcgen05 import _decode_f16x3

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(autouse=True)
def _restore_backend():
    prev = capi.get_backend()
    yield
    capi.set_backend(prev)


def _rup(x, a):
    return (x + a - 1) // a * a


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# (backend, f16_images): 3xTF32 split in the kernel, fp16x3 split in the kernel, both operands as fp16x3 images (the default path)
PRODUCT_VARIANTS = [(3, 0), (19, 0), (923, 1)]


# ------------------------------------------------------------------------------------------------------------ a. split-K partials
def _check_partials(W, X, S, ldp, backend, f16_images):
    capi.set_backend(backend)
    Nw, K = W.shape
    part = capi.op_skinny_partials(W, X, S=S, f16_images=f16_images, ldp=ldp)
    torch.cuda.synchronize()
    S = part.shape[0]
    Ks = K // S
    W64, X64 = W.double(), X.double()
    ref = X64 @ W64.t()
    bar = 2e-5 * max(1.0, float(ref.abs().max()))
    assert torch.isnan(part[:, :, Nw:]).all(), "pad columns [Nw, ldp) of the partial planes were written"
    got = part[:, :, :Nw].double()
    assert not torch.isnan(got).any(), "an element of the partial planes was not written"
    assert float((got.sum(0) - ref).abs().max()) <= bar
    for s in range(S):                                     # every plane against the product over ITS K range
        ref_s = X64[:, s * Ks:(s + 1) * Ks] @ W64[:, s * Ks:(s + 1) * Ks].t()
        assert float((got[s] - ref_s).abs().max()) <= bar, s


# the four products of the decode step with their planned S (0), a small ragged one, and one below a full tile with S = 1 and S = 2
_SHAPES = [((4096, 1536, 0, 4096), (1, 5, 63, 64, 65, 100, 128)), ((4096, 3072, 0, 4096), (5, 64, 100)), ((1024, 1024, 0, 1024), (1, 65, 128)),
           ((4905, 1024, 0, 4908), (100,)), ((4905, 1024, 0, 4928), (5, 63, 100)), ((992, 320, 0, 992), (5, 64, 100)),
           ((130, 64, 1, 132), (1, 65, 128)), ((130, 64, 2, 132), (1, 65, 128))]


@pytest.mark.parametrize("backend,f16_images", PRODUCT_VARIANTS)
@pytest.mark.parametrize("shape,B", [(s, b) for s, bs in _SHAPES for b in bs],
                         ids=["%dx%d-S%d-ldp%d-B%d" % (s + (b,)) for s, bs in _SHAPES for b in bs])
def test_skinny_partials(shape, B, backend, f16_images):
    """sum_s part[s] and every plane on its own against fp64, for batch sizes around the two 64-column tiles of the batch side
    (rows >= B come from TMA zero fill), with the activations read at a row pitch larger than K."""
    Nw, K, S, ldp = shape
    g = _gen(Nw + K + B)
    W = (torch.randn(Nw, K, generator=g) / K ** 0.5).cuda()
    X = torch.randn(B, K + 32, generator=g).cuda()[:, :K]
    _check_partials(W, X, S, ldp, backend, f16_images)


@pytest.mark.parametrize("backend,f16_images", PRODUCT_VARIANTS)
def test_skinny_partials_operand_range(backend, f16_images):
    """Operands that are not O(1): activations ~1e3, weights ~1e-3, same relative bar.  The fp16x3 variants scale activations by 4 and
    weights by 256 before the fp16 split, so they hold |activation| <= 16376 and |weight| <= 255; beyond that the split overflows to
    inf and the product is NaN / inf (not tested: the decode step's operands are bounded by construction)."""
    g = _gen(7)
    W = (torch.randn(4096, 1536, generator=g) / 1536 ** 0.5 * 1e-3).cuda()
    X = (torch.randn(100, 1536, generator=g) * 1e3).cuda()
    assert float(X.abs().max()) > 255
    _check_partials(W, X, 0, 4096, backend, f16_images)


# ------------------------------------------------------------------------------------------------------------ b. the reductions
@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("S", [1, 2, 4, 16])
def test_reduce_bias(S, with_bias):
    B, Nw, ldp, ld_out = 100, 1024, 1032, 1040
    g = _gen(S)
    part = torch.randn(S, B, ldp, generator=g).cuda()
    bias = torch.randn(Nw, generator=g).cuda() if with_bias else None
    buf = torch.full((B, ld_out), NAN, device="cuda")
    capi.op_reduce_bias(part, Nw, bias, buf[:, :Nw])
    torch.cuda.synchronize()
    same = part[0, :, :Nw].clone()
    for s in range(1, S):                                  # the kernel's order: ascending s, then the bias
        same += part[s, :, :Nw]
    ref = part[:, :, :Nw].double().sum(0)
    if with_bias:
        same += bias
        ref += bias.double()
    assert torch.equal(buf[:, :Nw], same)
    assert float((buf[:, :Nw].double() - ref).abs().max()) <= 1e-6 * max(1.0, float(ref.abs().max()))
    assert torch.isnan(buf[:, Nw:]).all()


@pytest.mark.parametrize("pre,b1,b2", [(1, 0, 0), (0, 1, 1), (1, 1, 0), (0, 0, 0)])
@pytest.mark.parametrize("S", [1, 2, 4, 16])
@pytest.mark.parametrize("B,H", [(128, 64), (5, 248), (100, 1024)])
def test_reduce_lstm(B, H, S, pre, b1, b2):
    """h, c against the fp64 cell; the three h destinations (distinct pitches, as the state buffer and the slots of the two concatenated
    inputs) bitwise equal with their neighbouring columns untouched; both fp16x3 images decode to h; c_out may alias c_prev."""
    g = _gen(B + H + S)
    ldp = 4 * H + 8
    part = (torch.randn(S, B, ldp, generator=g) / S ** 0.5).cuda()
    pre_t = torch.randn(B, 4 * H, generator=g).cuda() if pre else None
    bias1 = torch.randn(4 * H, generator=g).cuda() if b1 else None
    bias2 = torch.randn(4 * H, generator=g).cuda() if b2 else None
    c_prev = torch.randn(B, H, generator=g).cuda()
    images = H % 32 == 0
    c_out = torch.full((B, H), NAN, device="cuda")
    d0, d1, d2 = (torch.full((B, w), NAN, device="cuda") for w in (H, 32 + H, 3 * H))
    h0, h1, h2 = d0, d1[:, 32:], d2[:, H:2 * H]
    i1, i2 = (torch.full((B, w), -1, dtype=torch.int32, device="cuda") for w in (32 + H, 3 * H))
    pk1, pk2 = i1[:, 32:], i2[:, H:2 * H]
    if not images:
        with pytest.raises(capi.GvdError):                 # images need whole 32-column K slices
            capi.op_reduce_lstm(part, c_prev, c_out, h0, h1, h2, pre_t, bias1, bias2, pk1, pk2)
    capi.op_reduce_lstm(part, c_prev, c_out, h0, h1, h2, pre_t, bias1, bias2, pk1 if images else None, pk2 if images else None)
    c_alias = c_prev.clone()
    h_alias = torch.empty(B, H, device="cuda")
    capi.op_reduce_lstm(part, c_alias, c_alias, h_alias, None, None, pre_t, bias1, bias2)
    torch.cuda.synchronize()
    gates = part[:, :, :4 * H].double().sum(0)
    for t in (pre_t, bias1, bias2):
        if t is not None:
            gates = gates + t.double()
    i, f, gg, o = gates.chunk(4, dim=1)
    c_ref = torch.sigmoid(f) * c_prev.double() + torch.sigmoid(i) * torch.tanh(gg)
    h_ref = torch.sigmoid(o) * torch.tanh(c_ref)
    assert float((h0.double() - h_ref).abs().max()) <= 2e-6 and float((c_out.double() - c_ref).abs().max()) <= 2e-6
    assert torch.equal(h1, h0) and torch.equal(h2, h0)
    assert torch.isnan(d1[:, :32]).all() and torch.isnan(d2[:, :H]).all() and torch.isnan(d2[:, 2 * H:]).all()
    assert torch.equal(c_alias, c_out) and torch.equal(h_alias, h0)
    if images:
        for img, pk, lo, hi in ((i1, pk1, 32, 32 + H), (i2, pk2, H, 2 * H)):
            val, _ = _decode_f16x3(pk.contiguous(), H, 4.0)
            assert float(np.abs(val - h0.cpu().double().numpy()).max()) <= 2.0 ** -20
            assert bool((img[:, :lo] == -1).all()) and bool((img[:, hi:] == -1).all())
    else:
        assert bool((i1 == -1).all()) and bool((i2 == -1).all())


# ------------------------------------------------------------------------------------------------------------ c. the samplers
E_ = 32          # embedding width of the sampler cases
L_, T_ = 5, 2    # seq / logp destinations are column T_ of [B, L_] buffers


class _PickOut:
    """Destinations of one sampler launch, sentinel-filled: it [B], column T_ of seq / logp [B, L_], xt as a window of a wider buffer
    (or dense for the fused head, which writes it with pitch E), optionally the fp16x3 image of xt."""

    def __init__(self, B, dense_xt=False, image=False):
        self.it = torch.full((B,), -1, dtype=torch.int64, device="cuda")
        self.seq = torch.full((B, L_), -7, dtype=torch.int64, device="cuda")
        self.logp = torch.full((B, L_), NAN, device="cuda")
        self.xt_buf = torch.full((B, E_ if dense_xt else E_ + 8), NAN, device="cuda")
        self.xt = self.xt_buf[:, :E_]
        self.img = torch.full((B, 64), -1, dtype=torch.int32, device="cuda") if image else None

    def args(self, embed):
        kw = dict(seq=self.seq[:, T_], logp=self.logp[:, T_], embed=embed, xt=self.xt)
        if self.img is not None:
            kw["xt_pk"] = self.img[:, :32]
        return kw

    def check(self, tag, want_tok, want_lp, embed, lp_tol, rows=None, kinds=None):
        torch.cuda.synchronize()
        tok = self.it.cpu().numpy()
        rows = np.arange(len(tok)) if rows is None else rows
        bad = rows[tok[rows] != want_tok[rows]]
        assert bad.size == 0, (tag, [(int(b), kinds[b] if kinds else "", int(tok[b]), int(want_tok[b])) for b in bad[:8]])
        lp = self.logp[:, T_].cpu().double().numpy()
        if lp_tol is not None:
            err = np.abs(lp[rows] - want_lp[rows])
            assert not np.isnan(err).any() and float(err.max()) <= lp_tol, (tag, float(np.nanmax(err)), int(rows[np.nanargmax(err)]))
        assert torch.equal(self.seq[:, T_], self.it), tag
        other = [c for c in range(L_) if c != T_]
        assert bool((self.seq[:, other] == -7).all()) and torch.isnan(self.logp[:, other]).all(), tag
        assert torch.equal(self.xt, embed[self.it].clamp(min=0)), tag
        assert torch.isnan(self.xt_buf[:, E_:]).all(), tag
        if self.img is not None:
            val, _ = _decode_f16x3(self.img[:, :32].contiguous(), E_, 4.0)
            x = self.xt.cpu().double().numpy()
            assert float(np.abs(val - x).max()) <= 2.0 ** -20 * max(1.0, float(np.abs(x).max())), tag
            assert bool((self.img[:, 32:] == -1).all()), tag


def _exact_operands(x, seed, nplanes=3):
    """The logits x [B, V] (multiples of 1/8) as exact sums: planes [nplanes, B, ldp] + bias for reduce_pick, and one-hot rows h [B, 128]
    with W [V, 128] (W[v, b] = x[b, v] - bias[v]) for the products: every operand has at most 8 significant bits, so the tf32 and fp16
    splits are exact (lo = 0) and all paths see bit-identical logits."""
    B, V = x.shape
    rs = np.random.RandomState(seed)
    ldp = _rup(V, 4) + 4
    bias = rs.randint(-32, 33, size=V) * 0.125
    planes = np.zeros((nplanes, B, ldp))
    planes[1:, :, :V] = rs.randint(-16, 17, size=(nplanes - 1, B, V)) * 0.125
    planes[0, :, :V] = x - bias - planes[1:, :, :V].sum(0)
    W = np.zeros((V, 128))
    W[:, :B] = (x - bias).T
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float().cuda()
    return f(planes), f(bias), f(np.eye(B, 128)), f(W)


def _run_all_samplers(x, unk, seed, want_tok, want_lp, lp_tol, kinds=None, mask=None):
    """x [B, V] float64 exact logits (+ an optional additive mask of 0 / -inf per word, applied through the bias) through
    greedy_pick, reduce_pick, the fused head (3xTF32 and fp16x3) and, from 128 words on, the three product -> reduce_pick chains."""
    B, V = x.shape
    planes, bias, h, W = _exact_operands(x, seed)
    if mask is not None:
        bias = bias + torch.from_numpy(mask).float().cuda()
    embed = torch.randn(V, E_, generator=_gen(seed)).cuda()
    logits = torch.full((B, _rup(V, 4) + 4), NAN, device="cuda")
    logits[:, :V] = torch.from_numpy(x if mask is None else x + mask).float().cuda()
    chk = dict(want_tok=want_tok, want_lp=want_lp, embed=embed, lp_tol=lp_tol, kinds=kinds)

    o = _PickOut(B)
    capi.op_greedy_pick(logits[:, :V], unk, o.it, **o.args(embed))
    o.check("greedy_pick", **chk)

    o = _PickOut(B, image=True)
    capi.op_reduce_pick(planes, bias, V, unk, o.it, **o.args(embed))
    o.check("reduce_pick", **chk)

    for backend in (3, 19):
        capi.set_backend(backend)
        o = _PickOut(B, dense_xt=True)
        capi.op_logit_pick_tc(h, W, bias, unk, o.it, **o.args(embed))
        o.check("logit_pick_tc backend %d" % backend, **chk)

    if V >= 128:
        for backend, f16_images in PRODUCT_VARIANTS:
            capi.set_backend(backend)
            part = capi.op_skinny_partials(W, h, f16_images=f16_images, ldp=_rup(V, 4) + 4)
            o = _PickOut(B, image=True)
            capi.op_reduce_pick(part, bias, V, unk, o.it, **o.args(embed))
            o.check("skinny_partials(%d, %d) -> reduce_pick" % (backend, f16_images), **chk)
            assert torch.isnan(part[:, :, V:]).all()


_VOCABS = [2, 64, 65, 301, 2048, 2049, 4905, 5120, 5121, 6144]          # 2048|2049 and 5120|5121: reduce_pick_kernel<2|5|6> boundaries
_PICK_CASES = ([(V, 128, V - 1) for V in _VOCABS] + [(V, 128, u) for V in (65, 301, 4905, 6144) for u in (0, V // 2)] +
               [(V, B, V - 1) for V in (301, 4905) for B in (1, 100)])


@pytest.mark.parametrize("V,B,unk", _PICK_CASES)
def test_samplers_on_tie_and_unk_rows(V, B, unk):
    """One exact reference, three implementations: token ids equal on rows built to hit every tie / UNK branch (sampler_ref.KINDS),
    log-probabilities within 1e-5, strided seq / logp destinations, xt = ReLU(embed[token]) bitwise."""
    x, kinds = special_rows(B, V, unk, seed=V * 3 + B + unk)
    want_tok, want_lp = pick_reference(x, unk)
    _run_all_samplers(x, unk, V + B, want_tok, want_lp, 1e-5, kinds=kinds)


def test_samplers_with_masked_words():
    """Words masked with -inf (through the bias), a whole 64-column tile among them: the fused head's tile of -inf has no finite
    maximum of its own and must not poison the merged log-sum-exp."""
    V, B, unk = 1500, 64, 7
    x, kinds = special_rows(B, V, unk, seed=11)
    mask = np.zeros(V)
    mask[64:128] = -np.inf
    mask[np.random.RandomState(5).choice(V, 40, replace=False)] = -np.inf
    want_tok, want_lp = pick_reference(x + mask, unk)
    _run_all_samplers(x, unk, 13, want_tok, want_lp, 1e-5, kinds=kinds, mask=mask)


def test_samplers_reject_unsupported_shapes():
    B, V = 4, 6145
    part = torch.zeros(1, B, V + 3, device="cuda")
    bias = torch.zeros(V, device="cuda")
    embed = torch.zeros(V, E_, device="cuda")
    o = _PickOut(B)
    with pytest.raises(capi.GvdError):                     # reduce_pick holds a row in registers: at most 6 x 1024 words
        capi.op_reduce_pick(part, bias, V, 0, o.it)
    with pytest.raises(capi.GvdError):                     # the packed xt needs a 32-multiple pitch
        capi.op_reduce_pick(torch.zeros(1, B, 304, device="cuda"), bias[:301].contiguous(), 301, 0, o.it, embed=embed, xt=o.xt,
                            xt_pk=torch.zeros(B, 40, dtype=torch.int32, device="cuda"))
    embed6 = torch.zeros(301, 6, device="cuda")
    with pytest.raises(capi.GvdError):                     # the fused head copies the embedding row in 16-byte pieces
        capi.op_logit_pick_tc(torch.zeros(B, 128, device="cuda"), torch.zeros(301, 128, device="cuda"), bias[:301].contiguous(), 0, o.it,
                              embed=embed6, xt=torch.zeros(B, 6, device="cuda"))
    torch.cuda.synchronize()
    assert bool((o.it == -1).all())                        # nothing was launched


def test_samplers_give_token_zero_for_nan_rows():
    """A row without one finite comparison (every logit NaN) has no top-2: all three samplers define the result as token 0, inside the
    embedding table."""
    V, B, unk = 301, 4, 300
    x, _ = special_rows(B, V, unk, seed=1)
    planes, bias, h, W = _exact_operands(x, 2)
    bias[:] = NAN
    embed = torch.randn(V, E_, generator=_gen(3)).cuda()
    zero = np.zeros(B, np.int64)
    chk = dict(want_tok=zero, want_lp=None, embed=embed, lp_tol=None)
    o = _PickOut(B)
    capi.op_greedy_pick(torch.full((B, V), NAN, device="cuda"), unk, o.it, **o.args(embed))
    o.check("greedy_pick", **chk)
    o = _PickOut(B, image=True)
    capi.op_reduce_pick(planes, bias, V, unk, o.it, **o.args(embed))
    o.check("reduce_pick", **chk)
    capi.set_backend(3)
    o = _PickOut(B, dense_xt=True)
    capi.op_logit_pick_tc(h, W, bias, unk, o.it, **o.args(embed))
    o.check("logit_pick_tc", **chk)


@pytest.mark.parametrize("B", [100, 128])
def test_vocabulary_head_chains_on_random_logits(B):
    """The four head + sampler chains of the greedy loop on continuous logits (h [B,1024] against W [4905,1024]): token equal to the
    fp64 reference wherever its top-2 gap exceeds 1e-4, log-probability within 1e-4.  The UNK bias is raised so that UNK is on top of a
    good share of the rows."""
    V, K, unk = 4905, 1024, 4904
    g = _gen(B)
    h = torch.randn(B, K, generator=g).cuda()
    W = (torch.randn(V, K, generator=g) / 32).cuda()
    bias = torch.randn(V, generator=g)
    bias[unk] = 5.0
    bias = bias.cuda()
    embed = torch.randn(V, E_, generator=g).cuda()
    ref = (h.double() @ W.double().t() + bias.double()).cpu().numpy()
    want_tok, want_lp = pick_reference(ref, unk)
    rows = np.nonzero(top2_gap(ref, unk) > 1e-4)[0]
    n_unk = int((ref.argmax(1) == unk).sum())
    assert rows.size >= B - 2 and 0 < n_unk < B, (rows.size, n_unk)
    chk = dict(want_tok=want_tok, want_lp=want_lp, embed=embed, lp_tol=1e-4, rows=rows)
    Vp = _rup(V, 4)

    capi.set_backend(0)
    logits = capi.op_linear(h, W, bias)
    o = _PickOut(B)
    capi.op_greedy_pick(logits, unk, o.it, **o.args(embed))
    o.check("linear -> greedy_pick", **chk)
    for backend, f16_images in PRODUCT_VARIANTS:
        capi.set_backend(backend)
        part = capi.op_skinny_partials(W, h, f16_images=f16_images, ldp=Vp)
        o = _PickOut(B, image=True)
        capi.op_reduce_pick(part, bias, V, unk, o.it, **o.args(embed))
        o.check("skinny_partials(%d, %d) -> reduce_pick" % (backend, f16_images), **chk)
    for backend in (3, 19):
        capi.set_backend(backend)
        o = _PickOut(B, dense_xt=True)
        capi.op_logit_pick_tc(h, W, bias, unk, o.it, **o.args(embed))
        o.check("logit_pick_tc backend %d" % backend, **chk)


# ------------------------------------------------------------------------------------------------------------ d. the GRU layer
def _gru_ref(gi, Whh, bhh, sample_idx):
    """torch.nn.GRU(bidirectional) recurrence in float64 from the input projections: gates in r, z, n order, b_hn inside the r product,
    the reverse direction walks t = T-1-step; rows outside [lo, hi) of sample_idx are zeroed afterwards (model.py:562-566)."""
    B, T, _ = gi.shape
    G = Whh.shape[2]
    gi, Whh, bhh = gi.double(), Whh.double(), bhh.double()
    out = torch.zeros(B, T, 2 * G, dtype=torch.float64, device=gi.device)
    for d in range(2):
        h = torch.zeros(B, G, dtype=torch.float64, device=gi.device)
        for step in range(T):
            t = T - 1 - step if d else step
            x = gi[:, t, d * 3 * G:(d + 1) * 3 * G]
            gh = h @ Whh[d].t() + bhh[d]
            r = torch.sigmoid(x[:, :G] + gh[:, :G])
            z = torch.sigmoid(x[:, G:2 * G] + gh[:, G:2 * G])
            n = torch.tanh(x[:, 2 * G:] + r * gh[:, 2 * G:])
            h = (1 - z) * n + z * h
            out[:, t, d * G:(d + 1) * G] = h
    keep = None
    if sample_idx is not None:
        t = torch.arange(T, device=gi.device)[None, :]
        keep = (t >= sample_idx[:, :1]) & (t < sample_idx[:, 1:])
        out = out * keep[:, :, None]
    return out, keep


@pytest.mark.parametrize("windowed", [False, True])
@pytest.mark.parametrize("B,T,G", [(1, 1, 32), (5, 10, 512), (100, 10, 512), (128, 7, 64), (3, 480, 512)])
def test_gru_layer(B, T, G, windowed):
    """The tensor-core layer kernel (path 1) and the per-step GEMM + pointwise loop (path 0, CUDA-core and wgmma GEMM) against the fp64
    recurrence and against each other; with sample_idx the rows outside each clip's window are exactly 0."""
    g = _gen(B * 1000 + T + G)
    gi = torch.randn(B, T, 6 * G, generator=g).cuda()
    Whh = (torch.randn(2, 3 * G, G, generator=g) / G ** 0.5).cuda()
    bhh = (torch.randn(2, 3 * G, generator=g) * 0.1).cuda()
    sample_idx = None
    if windowed:                                           # whole range, empty, a middle window, a window ending at T
        win = [(0, T), (T // 2, T // 2), (T // 3, max(T // 3, 2 * T // 3)), (T // 2, T)]
        sample_idx = torch.tensor([win[b % 4] for b in range(B)], dtype=torch.int64).cuda()
    ref, keep = _gru_ref(gi, Whh, bhh, sample_idx)
    outs = {}
    for tag, path, backend in (("steps, CUDA cores", 0, 0), ("steps, wgmma", 0, 3), ("layer kernel", 1, 923)):
        capi.set_backend(backend)
        outs[tag] = capi.op_gru_layer(path, gi, Whh, bhh, sample_idx)
    torch.cuda.synchronize()
    errs = {tag: float((o.double() - ref).abs().max()) for tag, o in outs.items()}
    print("gru_layer B=%d T=%d G=%d windowed=%d max|err| vs fp64: %s" % (B, T, G, windowed, errs))
    for tag, o in outs.items():
        assert not torch.isnan(o).any(), tag
        assert errs[tag] <= 2e-5, (tag, errs[tag])
        if keep is not None:
            assert float(o[~keep].abs().max() if (~keep).any() else 0.0) == 0.0, tag
    assert float((outs["layer kernel"] - outs["steps, CUDA cores"]).abs().max()) <= 2e-5
    assert float((outs["layer kernel"] - outs["steps, wgmma"]).abs().max()) <= 2e-5
