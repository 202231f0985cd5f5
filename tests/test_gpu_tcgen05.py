"""Tensor-core (wgmma, 3xTF32 / fp16x3) path: the tensor-core GEMM / LSTM kernels against fp64 references and against the
CUDA-core kernels, then the whole greedy decode with the tensor-core backend against the oracle."""

import numpy as np
import pytest
import torch

import gvd_oracle as O
from cases import CASES, build_case, load_fixture
from gvd_b200 import capi
from test_gpu_parity import _model, _sample, _maxerr, TOL

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_backend():
    prev = capi.get_backend()
    yield
    capi.set_backend(prev)


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 32, 64), (100, 1024, 3124), (1000, 432, 2048), (257, 130, 36),
                                   (64, 4905, 1024), (2000, 2048, 2048), (130, 96, 252), (1000, 172, 1000), (100, 4096, 1536)])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("backend", [3, 19])
def test_linear_tc(M, N, K, act, backend):
    """backend 3: 3xTF32 (tf32 wgmma, hi/lo planes); 19 = +16: fp16x3 (f16 wgmma, fp16 hi/lo with power-of-two operand scales)."""
    capi.set_backend(backend)
    g = torch.Generator().manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = A.double() @ W.double().t() + b.double()
    if act:
        ref = ref.clamp(min=0)
    out = capi.op_linear(A.cuda(), W.cuda(), b.cuda(), act, tc=True)
    torch.cuda.synchronize()
    err = _maxerr(out, ref)
    assert err <= 2e-5 * max(1.0, float(ref.abs().max())), err      # fp32-class accuracy (plain TF32 would be ~1e-3)


@pytest.mark.parametrize("B,H,K0,K1", [(100, 1024, 512, 1024), (100, 1024, 2048, 1024), (5, 248, 64, 248), (130, 64, 32, 0)])
@pytest.mark.parametrize("backend", [3, 19])
def test_lstm_step_tc_matches_cuda_core_kernel(B, H, K0, K1, backend):
    capi.set_backend(backend)
    g = torch.Generator().manual_seed(B + H)
    x0 = torch.randn(B, K0, generator=g).cuda()
    w0 = (torch.randn(4 * H, K0, generator=g) / K0 ** 0.5).cuda()
    x1 = torch.randn(B, K1, generator=g).cuda() if K1 else None
    w1 = (torch.randn(4 * H, K1, generator=g) / K1 ** 0.5).cuda() if K1 else None
    b1, b2 = torch.randn(4 * H, generator=g).cuda(), torch.randn(4 * H, generator=g).cuda()
    c0 = torch.randn(B, H, generator=g).cuda()
    h_a, c_a = capi.op_lstm_step(x0, w0, x1, w1, b1, b2, c0, backend=0)
    h_b, c_b = capi.op_lstm_step(x0, w0, x1, w1, b1, b2, c0, backend=1)
    torch.cuda.synchronize()
    gates = x0.double() @ w0.double().t() + b1.double() + b2.double()
    if K1:
        gates = gates + x1.double() @ w1.double().t()
    i, f, gg, o = gates.chunk(4, dim=1)
    c_ref = torch.sigmoid(f) * c0.double() + torch.sigmoid(i) * torch.tanh(gg)
    h_ref = torch.sigmoid(o) * torch.tanh(c_ref)
    for got in ((h_a, c_a), (h_b, c_b)):
        assert _maxerr(got[0], h_ref) <= 2e-5 and _maxerr(got[1], c_ref) <= 2e-5


@pytest.mark.parametrize("wide_backend", [7, 23])
@pytest.mark.parametrize("M,N,K", [(20000, 256, 32), (20000, 512, 1024), (20000, 3096, 1024), (40000, 432, 2048), (10000, 1024, 2780),
                                   (10000, 2048, 544)])       # large M with narrow, wide and ragged N
@pytest.mark.parametrize("act", [0, 1])
def test_linear_tc_wide_tiles(M, N, K, act, wide_backend):
    """backend bit 2 (inert: it selected 256-column tiles) must not change the result of large products."""
    capi.set_backend(wide_backend)
    g = torch.Generator().manual_seed(M + N)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = A.double() @ W.double().t() + b.double()
    if act:
        ref = ref.clamp(min=0)
    out = capi.op_linear(A.cuda(), W.cuda(), b.cuda(), act, tc=True)
    torch.cuda.synchronize()
    assert _maxerr(out, ref) <= 2e-5 * max(1.0, float(ref.abs().max()))


def _decode_f16x3(img, N, scale):
    """fp16x3 operand image (gvd_common.cuh): per row and 32-column slice 16 words of hi pairs then 16 words of lo pairs; value = (hi + lo) / scale."""
    M, Np = img.shape
    h = img.cpu().numpy().view(np.float16).astype(np.float64).reshape(M, Np // 32, 2, 16, 2)      # [row, slice, hi|lo, word, half]
    v = (h[:, :, 0] + h[:, :, 1]).reshape(M, Np) / scale                                       # word i of a slice = columns 2i, 2i+1
    return v[:, :N], v[:, N:]


@pytest.mark.parametrize("M,N,K", [(4000, 2048, 2048), (20000, 3096, 1024), (10000, 1024, 2780), (1500, 432, 2048), (1024, 512, 1024),
                                   (3000, 100, 64), (200, 130, 36)])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("ss_backend", [923, 1947])
def test_linear_f16ss_persistent(M, N, K, act, ss_backend):
    """The conversion-free prologue GEMM (backend bit 7) on its own, against fp64: C, the fp16x3 image of C its epilogue writes for the
    next GEMM (backend bit 9: 22 significant bits of the fp32 value, zero padding columns), and the image-only mode.  1947 = 923 + bit 10:
    the same product with the (unused on Hopper) CTA-pair switch set: it must not change the result."""
    capi.set_backend(ss_backend)
    g = torch.Generator().manual_seed(M + 3 * N)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = A.double() @ W.double().t() + b.double()
    if act:
        ref = ref.clamp(min=0)
    scale = max(1.0, float(ref.abs().max()))
    C, img = capi.op_linear_f16ss(A.cuda(), W.cuda(), b.cuda(), act, want_img=True)
    torch.cuda.synchronize()
    assert _maxerr(C, ref) <= 2e-5 * scale
    val, pad = _decode_f16x3(img, N, 4.0)
    assert float(np.abs(val - C.cpu().double().numpy()).max()) <= 2.0 ** -20 * scale and not pad.any()
    _, img2 = capi.op_linear_f16ss(A.cuda(), W.cuda(), b.cuda(), act, want_img=True, want_c=False)
    torch.cuda.synchronize()
    capi.set_backend(923)
    assert torch.equal(img2, img)


def _attention_ref(qkv, nh, hs, scale):
    nb, R, t = qkv.shape
    HP = t // 3
    q, k, v = (qkv[:, :, i * HP:i * HP + nh * hs].double().reshape(nb, R, nh, hs).permute(0, 2, 1, 3) for i in range(3))
    P = torch.softmax(q @ k.transpose(-1, -2) * scale, -1)
    return (P @ v).permute(0, 2, 1, 3).reshape(nb, R, nh * hs), P


@pytest.mark.parametrize("nb,nh,M,N,hs,ld", [(2, 6, 1000, 1000, 172, 3096), (1, 2, 52, 52, 44, 272), (3, 1, 130, 70, 192, 192),
                                             (2, 3, 128, 64, 32, 96), (1, 1, 1, 1, 4, 4)])
def test_scores_a_stationary(nb, nh, M, N, hs, ld):
    """Short-K batched Q K^T through the A-stationary kernel (operands split in the kernel) against fp64."""
    g = torch.Generator().manual_seed(nb * 100 + M)
    A = torch.randn(nb, M, ld, generator=g).cuda()
    W = torch.randn(nb, N, ld, generator=g).cuda()
    C = capi.op_scores_tc(A, W, nh, hs)
    torch.cuda.synchronize()
    a = A[:, :, :nh * hs].double().reshape(nb, M, nh, hs).permute(0, 2, 1, 3)
    w = W[:, :, :nh * hs].double().reshape(nb, N, nh, hs).permute(0, 2, 1, 3)
    ref = a @ w.transpose(-1, -2)
    assert _maxerr(C, ref) <= 4e-6 * max(1.0, float(ref.abs().max()))


# amp scales the projections: 1 = flat softmax, 6 = sharply peaked rows (logit range ~ +-80, factors down to 1e-24 and
# underflowing numerators), the regime where the per-group running maxima differ by orders of magnitude
@pytest.mark.parametrize("nb,nh,R,hs,HP,scale,amp", [(2, 6, 1000, 172, 1032, 1 / 32, 1.0), (2, 6, 1000, 172, 1032, 1 / 32, 6.0),
                                                     (1, 6, 52, 44, 264, 1 / 16, 1.0), (3, 2, 132, 192, 384, 1 / 8, 1.0),
                                                     (1, 1, 4, 4, 4, 1.0, 1.0), (1, 3, 20, 8, 24, 0.5, 3.0)])
@pytest.mark.parametrize("att_backend", [155, 411])
def test_fused_self_attention(nb, nh, R, hs, HP, scale, amp, att_backend):
    """softmax(Q K^T * scale) V through the fused pair (softmax-numerator scores + row-scaled P.V) against fp64:
    the stored softmax E * F itself, its row sums, the output, and the zero padding of the head columns."""
    capi.set_backend(att_backend)                     # 411: fp16x3 key / value images (bit 8); 155: tf32 hi / lo planes
    g = torch.Generator().manual_seed(int(R * 10 + amp))
    qkv = (torch.randn(nb, R, 3 * HP, generator=g) * amp).cuda()
    out, E, F = capi.op_self_attention_tc(qkv, nh, hs, scale, debug=True)
    torch.cuda.synchronize()
    ref, P = _attention_ref(qkv, nh, hs, scale)
    Fx = F.permute(0, 1, 3, 2).repeat_interleave(32, dim=3)[..., :R]
    Peff = (E * Fx).double()
    assert float((Peff - P).abs().max()) <= 5e-5
    assert float((Peff.sum(-1) - 1).abs().max()) <= 1e-5
    assert _maxerr(out[:, :, :nh * hs], ref) <= 4e-5 * max(1.0, float(ref.abs().max()))
    if nh * hs < HP:
        assert float(out[:, :, nh * hs:].abs().max()) == 0.0


@pytest.mark.parametrize("att_backend", [155, 411])
def test_fused_self_attention_repeated_launches(att_backend):
    """150 full-size launches: every one must meet the bar (a parity-aliased stage barrier once made ~1 launch in 3 wrong)."""
    capi.set_backend(att_backend)
    g = torch.Generator().manual_seed(5)
    for rep in range(30):
        qkv = (torch.randn(3, 1000, 3 * 1032, generator=g) * (6.0 if rep % 2 else 1.0)).cuda()
        out = capi.op_self_attention_tc(qkv, 6, 172, 1 / 32)
        torch.cuda.synchronize()
        ref, _ = _attention_ref(qkv, 6, 172, 1 / 32)
        assert _maxerr(out[:, :, :6 * 172], ref) <= 4e-5 * max(1.0, float(ref.abs().max())), rep


@pytest.mark.parametrize("backend", [0, 1, 3, 7, 11, 15, 19, 27, 31, 91, 155, 411, 923, 1947])
@pytest.mark.parametrize("name", ["greedy_T10_B4", "greedy_T480_B2", "greedy_small_B5", "greedy_T10_B2_nointeract"])
def test_greedy_with_both_backends(name, backend):
    """backend 3 (wgmma 3xTF32 + fused self-attention), 1 (wgmma, unfused attention) and 0 (fp32 CUDA
    cores) all meet the parity bar, and so do the switches on top: bit 2 (+4, inert), bit 3 (+8, operand-swapped
    split-K decode products with the fused reduce + sampler), bit 4 (+16, fp16x3 instead of 3xTF32 in the forward GEMMs), bit 7 (+128, conversion-free prologue GEMMs), bit 8 (+256, fp16x3 images
    in the attention pair), bit 9 (+512, producers store the operand image of the next GEMM: 923 is the default)."""
    capi.set_backend(backend)
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    model = _model(opt, sd)
    seq, att2, sim = _sample(model, inp)
    oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp)
    assert torch.equal(seq.cpu(), oseq) and np.array_equal(seq.cpu().numpy(), fx["seq"])
    assert _maxerr(att2, oatt2) <= TOL and _maxerr(sim, osim) <= TOL


@pytest.mark.parametrize("backend", [3, 19])
def test_gemm_repeated_launches_stress(backend):
    """Ring hand-off stress (mbarrier phase accounting of the TMA ring): 200 launches each of a large problem (several waves of CTAs) and of the
    LSTM-mode kernel at full size, EVERY result checked against fp64 on the device and against the first launch bit for bit."""
    capi.set_backend(backend)
    g = torch.Generator().manual_seed(11)
    A = torch.randn(4000, 2048, generator=g).cuda()
    W = (torch.randn(2048, 2048, generator=g) / 2048 ** 0.5).cuda()
    b = torch.randn(2048, generator=g).cuda()
    ref = (A.double() @ W.double().t() + b.double()).clamp(min=0)
    scale = max(1.0, float(ref.abs().max()))
    first = None
    worst = torch.zeros((), dtype=torch.float64, device="cuda")
    same = torch.ones((), dtype=torch.bool, device="cuda")
    for _ in range(200):
        out = capi.op_linear(A, W, b, 1, tc=True)
        worst = torch.maximum(worst, (out.double() - ref).abs().max())
        if first is None:
            first = out.clone()
        same &= torch.equal(out, first)
    assert float(worst) <= 2e-5 * scale and bool(same)
    B, H, K0, K1 = 100, 1024, 512, 1024
    x0, x1 = torch.randn(B, K0, generator=g).cuda(), torch.randn(B, K1, generator=g).cuda()
    w0, w1 = (torch.randn(4 * H, K0, generator=g) / K0 ** 0.5).cuda(), (torch.randn(4 * H, K1, generator=g) / K1 ** 0.5).cuda()
    b1, b2, c0 = torch.randn(4 * H, generator=g).cuda(), torch.randn(4 * H, generator=g).cuda(), torch.randn(B, H, generator=g).cuda()
    gates = x0.double() @ w0.double().t() + x1.double() @ w1.double().t() + b1.double() + b2.double()
    i, f, gg, o = gates.chunk(4, dim=1)
    c_ref = torch.sigmoid(f) * c0.double() + torch.sigmoid(i) * torch.tanh(gg)
    h_ref = torch.sigmoid(o) * torch.tanh(c_ref)
    first = None
    worst = torch.zeros((), dtype=torch.float64, device="cuda")
    same = torch.ones((), dtype=torch.bool, device="cuda")
    for _ in range(200):
        h, c = capi.op_lstm_step(x0, w0, x1, w1, b1, b2, c0, backend=1)
        worst = torch.maximum(worst, torch.maximum((h.double() - h_ref).abs().max(), (c.double() - c_ref).abs().max()))
        if first is None:
            first = h.clone()
        same &= torch.equal(h, first)
    assert float(worst) <= 2e-5 and bool(same)
