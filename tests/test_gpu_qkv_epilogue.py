"""The Q|K|V epilogue of ss_gemm_kernel (the region encoder's projection storing Q as fp32, K as the per-head fp16x3 image and V as the
fp16x3 image of V^T per clip) on its own, bit for bit against the fp32 product followed by the two pack passes of the unfused path.
C and both images start as a NaN bit pattern, so a word the epilogue never writes (padding words and pad rows included) shows up, and
the K / V columns of C must stay untouched.  Clips of R = 1000 rows (R % 32 = 8; 7 clips and the full batch of 100), 64 (R % 32 = 0) and
998, at the default head size (rnn_size 1024: 6 heads of 172 columns, KH = 192) and at rnn_size 512 (6 x 88, KH = 96)."""
import pytest
import torch

from gvd_b200 import capi

pytestmark = pytest.mark.gpu

NAN = 0x7FC00000


def _heads(H):
    hs = -(-(-(-H // 6)) // 4) * 4
    return len(range(0, H, -(-H // 6))), hs


def _buffers(M, nh, hs, R):
    HP, KH, Rp = nh * hs, -(-hs // 32) * 32, -(-R // 32) * 32
    C = torch.full((M, 3 * HP), NAN, dtype=torch.int32, device="cuda")
    k_img = torch.full((M, nh, KH), NAN, dtype=torch.int32, device="cuda")
    vt_img = torch.full((M // R, HP, Rp), NAN, dtype=torch.int32, device="cuda")
    return C, k_img, vt_img


@pytest.mark.parametrize("H,R,clips", [(1024, 1000, 7), (1024, 1000, 100), (1024, 64, 9), (1024, 998, 5), (512, 1000, 7)])
def test_qkv_epilogue_bit_exact_against_pack_passes(H, R, clips):
    nh, hs = _heads(H)
    HP, M = nh * hs, clips * R
    g = torch.Generator(device="cuda").manual_seed(H + R + clips)
    A = torch.randn(M, H, device="cuda", generator=g)
    W = torch.randn(3 * HP, H, device="cuda", generator=g) * H ** -0.5
    out = {}
    for ref in (False, True):
        C, k_img, vt_img = _buffers(M, nh, hs, R)
        capi.op_linear_f16ss(A, W, qkv=(nh, hs, R, C.view(torch.float32), k_img, vt_img, ref))
        torch.cuda.synchronize()
        out[ref] = (C, k_img, vt_img)
    (C, k_img, vt_img), (C_ref, k_ref, vt_ref) = out[False], out[True]
    assert torch.equal(C[:, :HP], C_ref[:, :HP])
    assert bool((C[:, HP:] == NAN).all())                      # the epilogue stores only Q into C
    assert bool((C_ref != NAN).all())
    assert torch.equal(k_img, k_ref), int((k_img != k_ref).sum())
    assert torch.equal(vt_img, vt_ref), int((vt_img != vt_ref).sum())
