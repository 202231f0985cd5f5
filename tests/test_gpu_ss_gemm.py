"""ss_gemm_kernel (the prologue's operand-image GEMM: 128 x 128 tiles, a producer warpgroup and the fold of slice i deferred behind the
products of slice i + 1) at row counts around the tile size: M = 100 (one partial row tile), M = 1900 (15 row tiles, the last partial)
and M = 100 000 (782 row tiles, the fc7 GEMM at B = 100).  As in test_gpu_wide_tile.py: C and its fp16x3 image against fp64, and C bit
for bit against the 64-wide fp16x3 product of MODE_STORE.  The Q|K|V image epilogue is checked on 7 clips (7000 rows = 55 row tiles,
the last one partial)."""
import pytest
import torch

import gvd_b200.synth as synth
from gvd_b200 import capi
from test_gpu_parity import _maxerr
from test_gpu_wide_tile import SHAPES, _operands

pytestmark = pytest.mark.gpu

CASES = [(M, N, K) for M in (100, 1900) for (N, K) in SHAPES] + [(100000, 2048, 2048)]


def _err(a, b):
    return float((a.double() - b.double()).abs().max())          # on the device: M = 100 000 rows are 1.6 GB in fp64


def _decode_img(img, N, scale):
    """fp16x3 operand image: per row and 32-column slice 16 words of hi pairs then 16 words of lo pairs; value = (hi + lo) / scale"""
    M, Np = img.shape
    h = img.view(torch.float16).double().reshape(M, Np // 32, 2, 16, 2)
    v = (h[:, :, 0] + h[:, :, 1]).reshape(M, Np) / scale
    return v[:, :N], v[:, N:]


@pytest.fixture(autouse=True)
def _restore_backend():
    prev = capi.get_backend()
    yield
    capi.set_backend(prev)


@pytest.mark.parametrize("M,N,K", CASES)
@pytest.mark.parametrize("act", [0, 1])
def test_ss_gemm_against_fp64_and_64_wide(M, N, K, act):
    A, W, b = _operands(M, N, K)
    capi.set_backend(923)
    C, img = capi.op_linear_f16ss(A, W, b, act, want_img=True)
    torch.cuda.synchronize()
    ref = torch.addmm(b.double(), A.double(), W.double().t())
    if act:
        ref = ref.clamp(min=0)
    scale = max(1.0, float(ref.abs().max()))
    assert _err(C, ref) <= 2e-5 * scale
    del ref
    val, pad = _decode_img(img, N, 4.0)
    assert _err(val, C) <= 2.0 ** -20 * scale and not pad.any()
    del val, pad
    capi.set_backend(19)                                   # wgmma + fp16x3, 128 x 64 tiles, operands split in shared memory
    narrow = capi.op_linear(A, W, b, act, tc=True)
    torch.cuda.synchronize()
    assert torch.equal(C, narrow), _err(C, narrow)


def test_qkv_image_epilogue_seven_clips():
    """Encoder output at backend 923 (Q|K|V projection with the image epilogue) against backend 411 (fp32 Q|K|V + pack passes),
    bit for bit, on 7 clips of the default dims."""
    opt = synth.make_opt(t_attn_size=10)
    sd = synth.make_state_dict(opt)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    B, T = 7, 10
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
