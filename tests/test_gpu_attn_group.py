"""The row-grouped decode attention (attn_group_kernel) against the per-row kernel (attn_partial_kernel), bit for bit on the region logits,
x_out and its fp16x3 image, through gvd_op_attention_path: every A the decode takes (generic and register-resident queries), the three
region forms and the three input modes, group sizes up to and beyond 8 rows per clip, masked rows and a fully masked clip, split-K query
partials, video rows and the separate combine."""
import pytest
import torch

from gvd_b200 import capi
from test_gpu_attn_beam_ops import NAN, _gen

pytestmark = pytest.mark.gpu


def _windows(Bf, T, TC, g):
    fixed = [(0, T), (3, 3), (T - 4, T + 3), (TC - 2, TC + 3), (T + 1, T + 5)]
    out = []
    for b in range(Bf):
        if b < len(fixed):
            out.append(fixed[b])
        else:
            lo = int(torch.randint(0, T, (1,), generator=g))
            out.append((lo, int(torch.randint(lo + 1, T + 1, (1,), generator=g))))
    return torch.tensor(out, dtype=torch.int64)


def _both_paths(A, H, G, mode="both", form="mix", nclips=4, R=40, T=30, RC=16, TC=16, q_S=0, video=False, fused=True, seed=0):
    """gvd_op_attention_path with path 0 and 1 on the same inputs: B = nclips * G rows, G per clip; random masks (p = 0.25), clip 1 fully
    masked.  Returns (z, x, x_pk, ticket) of both."""
    g = _gen(1000 * A + 10 * G + seed)
    B = nclips * G
    dual = mode == "dual_region"
    c = lambda t: t.cuda().contiguous()
    V = 3 if video else nclips
    p_pool, pool = c(torch.randn(nclips, R, A, generator=g) * 0.5), c(torch.randn(nclips, R, H, generator=g))
    p_conv, conv = c(torch.randn(V, T, A, generator=g) * 0.5), c(torch.randn(V, T, H, generator=g))
    w1, w2 = c(torch.randn(A, generator=g) / A ** 0.5), c(torch.randn(A, generator=g) / A ** 0.5)
    b1, b2 = c(torch.randn(1, generator=g) * 0.1), c(torch.randn(1, generator=g) * 0.1)
    am = (torch.rand(nclips, R + 1, generator=g) < 0.25).to(torch.uint8)
    am[1] = 1
    om = am | (torch.rand(nclips, R + 1, generator=g) < 0.1).to(torch.uint8)
    att_mask, out_mask = c(am), c(om)
    if q_S:
        qkw = dict(q_part=c(torch.randn(q_S, B, 2 * A, generator=g) * 0.3), q_bias=c(torch.randn(2 * A, generator=g) * 0.1))
    else:
        qkw = dict(q=c(torch.randn(B, 2 * A, generator=g) * 0.5))
    gate = {}
    if dual:
        gate = dict(gate_w=c(torch.randn(H, generator=g) / H ** 0.5), gate_b=c(torch.randn(1, generator=g) * 0.1),
                    gate_h=c(torch.randn(B, H, generator=g)))
    vkw = {}
    if video:
        vkw = dict(_video=(c(torch.randint(0, V, (nclips,), generator=g)), c(_windows(nclips, T, TC, g)), c(torch.randn(A, generator=g) * 0.5)))
    nch_r, nch_t = -(-R // RC), 0 if dual else -(-T // TC)
    nrec = 2 * nch_r if dual else nch_r + nch_t
    HP = (H + 31) // 32 * 32
    outs = []
    for path in (0, 1):
        z = torch.full((B, R), NAN, device="cuda")
        x = torch.full((B, H), NAN, device="cuda")
        xpk = torch.full((B, HP), -1, dtype=torch.int32, device="cuda") if fused else None
        part = torch.full((B, nrec, H + 4), NAN, device="cuda")
        ticket = torch.zeros(B, dtype=torch.int32, device="cuda") if fused else None
        capi.op_attention(p_pool, None if mode == "featmap" else pool, None if dual else p_conv, None if dual else conv, w1, b1,
                          None if form == "dp" else w2, None if form == "dp" else b2, att_mask, out_mask, z, part, x, RC, TC, ticket=ticket,
                          x_pk=xpk, feat_div=G, att_input_mode=mode, region_attn_mode=form, path=path, **qkw, **gate, **vkw)
        torch.cuda.synchronize()
        outs.append((z, x, xpk, ticket))
    return outs


def _same(a, b):
    return (a is None and b is None) or (a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32)))


def _assert_bits(outs):
    (z0, x0, p0, t0), (z1, x1, p1, t1) = outs
    assert not torch.isnan(x0).any() and not torch.isnan(z0).any()
    assert _same(z0, z1), "region logits differ"
    assert _same(x0, x1), "x_out differs"
    assert _same(p0, p1), "x_pk image differs"
    if t1 is not None:
        assert int(t1.abs().sum()) == 0, "tickets not reset"


@pytest.mark.parametrize("form", ["mix", "mix_mul", "dp"])
@pytest.mark.parametrize("mode", ["both", "featmap", "dual_region"])
@pytest.mark.parametrize("A", [96, 128, 256, 384, 512])
def test_grouped_equals_per_row(A, mode, form):
    _assert_bits(_both_paths(A, 248 if A == 96 else 512, 3, mode, form))


@pytest.mark.parametrize("G", [1, 2, 3, 5, 8, 9, 13, 17])
@pytest.mark.parametrize("mode", ["both", "dual_region"])
def test_group_sizes_full_dims(G, mode):
    """A = 512, H = 1024, R = 100; G > 8 spans several row groups per clip."""
    _assert_bits(_both_paths(512, 1024, G, mode, "mix", nclips=3, R=100, T=10, RC=32, TC=16))


@pytest.mark.parametrize("q_S", [1, 4])
@pytest.mark.parametrize("mode", ["both", "featmap", "dual_region"])
def test_query_partials(q_S, mode):
    _assert_bits(_both_paths(512, 1024, 5, mode, "mix_mul", q_S=q_S))


@pytest.mark.parametrize("G", [3, 9])
@pytest.mark.parametrize("mode", ["both", "featmap"])
@pytest.mark.parametrize("A", [96, 512])
def test_video_rows(A, mode, G):
    """Windowed temporal chunks (full, empty, past-T, chunk-straddling windows) with the out-of-window record."""
    _assert_bits(_both_paths(A, 256, G, mode, "mix", nclips=6, T=48, video=True))


def test_separate_combine():
    """ticket = NULL: the partial records of both kernels feed attn_combine_kernel alike."""
    _assert_bits(_both_paths(256, 512, 4, "both", "dp", fused=False))


@pytest.mark.parametrize("path,feat_div", [(2, 2), (1, 3)])
def test_bad_path_or_row_count_refused(path, feat_div):
    z = lambda *shape: torch.zeros(*shape, device="cuda")
    u8 = torch.zeros(1, 9, dtype=torch.uint8, device="cuda")
    with pytest.raises(capi.GvdError):
        capi.op_attention(z(1, 8, 128), z(1, 8, 128), z(1, 4, 128), z(1, 4, 128), z(128), z(1), z(128), z(1), u8, u8, z(2, 8), z(2, 2, 132),
                          z(2, 128), 16, 16, q=z(2, 256), ticket=torch.zeros(2, dtype=torch.int32, device="cuda"), feat_div=feat_div,
                          path=path)
