"""The conversion-free prologue GEMM (MODE_SS of wg_gemm_kernel) runs on 128 x 128 tiles; every other mode stays at 128 x 64.

Per output element both widths issue the same fp16 products in the same order and fold them the same way, so:
- at the (N, K) of every prologue GEMM, C and its fp16x3 image are checked against fp64 (the test_linear_f16ss_persistent bounds);
- the 128-wide product equals, bit for bit, the 64-wide fp16x3 product of MODE_STORE on the same operands;
- the Q|K|V image epilogue at the full head layout (R = 1000, HS = 172, HP = 1032: head boundaries inside 128-column tiles, a partly
  empty last tile) gives the same encoder output as the projection without it plus the separate K / V^T pack passes."""
import numpy as np
import pytest
import torch

import gvd_b200.synth as synth
from gvd_b200 import capi
from test_gpu_parity import _maxerr
from test_gpu_tcgen05 import _decode_f16x3

pytestmark = pytest.mark.gpu

# (N, K) of the prologue's MODE_SS GEMMs at the default dims: fc7, similarity, region embedding (K = 2780 and its 32-padded 2784), Q|K|V,
# Wo (K = 1032 and 1056), FFN1 / ctx2pool, FFN2; then narrow N with one partial column tile
SHAPES = [(2048, 2048), (432, 2048), (1024, 2780), (1024, 2784), (3096, 1024), (1024, 1032), (1024, 1056), (512, 1024), (1024, 512),
          (100, 1024), (130, 2048)]


@pytest.fixture(autouse=True)
def _restore_backend():
    prev = capi.get_backend()
    yield
    capi.set_backend(prev)


def _operands(M, N, K):
    g = torch.Generator().manual_seed(M + 7 * N + K)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    return A.cuda(), W.cuda(), b.cuda()


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("M", [2000, 3000])             # 15 + 80 / 23 + 56 rows: a partial last row tile
@pytest.mark.parametrize("act", [0, 1])
def test_wide_tile_against_fp64(M, N, K, act):
    capi.set_backend(923)
    A, W, b = _operands(M, N, K)
    ref = A.double() @ W.double().t() + b.double()
    if act:
        ref = ref.clamp(min=0)
    scale = max(1.0, float(ref.abs().max()))
    C, img = capi.op_linear_f16ss(A, W, b, act, want_img=True)
    torch.cuda.synchronize()
    assert _maxerr(C, ref) <= 2e-5 * scale
    val, pad = _decode_f16x3(img, N, 4.0)
    assert float(np.abs(val - C.cpu().double().numpy()).max()) <= 2.0 ** -20 * scale and not pad.any()
    _, img2 = capi.op_linear_f16ss(A, W, b, act, want_img=True, want_c=False)
    torch.cuda.synchronize()
    assert torch.equal(img2, img)


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("act", [0, 1])
def test_wide_tile_equals_64_wide_product(N, K, act):
    """MODE_SS (128 wide, operands packed into images first) against MODE_STORE (64 wide, operands split in shared memory): both split
    with the same rounding, so every bit of C must agree."""
    M = 2000
    A, W, b = _operands(M, N, K)
    capi.set_backend(923)
    wide = capi.op_linear_f16ss(A, W, b, act)
    capi.set_backend(19)                                   # wgmma + fp16x3, the conversion kernel
    narrow = capi.op_linear(A, W, b, act, tc=True)
    torch.cuda.synchronize()
    assert torch.equal(wide, narrow), _maxerr(wide, narrow)


def test_qkv_image_epilogue_matches_pack_passes():
    """Encoder output at backend 923 (the Q|K|V projection stores K per head and V^T as fp16x3 images in its epilogue) against backend 411
    (pack fusion off: the same projection stores fp32 Q|K|V and pack passes build the images): bit-identical, on 3 clips of the
    default dims (R = 1000, 6 heads of HS = 172 in HP = 1032 columns, N = 3096 = 24 full 128-column tiles + 24 columns)."""
    opt = synth.make_opt(t_attn_size=10)
    sd = synth.make_state_dict(opt)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    B, T = 3, 10
    R, H, A = opt.num_sampled_frm * opt.num_prop_per_frm, opt.rnn_size, opt.att_hid_size
    inp = synth.make_inputs(opt, B, masked=True)
    keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
    dev = [inp[k].cuda() for k in keys]
    out = {}
    for be in (923, 411):
        capi.set_backend(be)
        nm.prologue(*dev)
        torch.cuda.synchronize()
        out[be] = (nm.workspace_tensor(B, T, "pool_feats", (B, R, H)).clone(), nm.workspace_tensor(B, T, "p_pool_feats", (B, R, A)).clone())
    for x, y in zip(out[923], out[411]):
        assert torch.equal(x, y), _maxerr(x, y)
