"""Fused self-attention kernel of the region encoder (csrc/gvd_attn.cu): softmax(Q K^T * scale) V with the scores kept on the SM, against
fp64; its operand-image store mode against the fp32 mode split by the pack pass, bit for bit; the whole encoder at the default backend
against the oracle.  The store-plan emulation at the end runs without a GPU."""
import numpy as np
import pytest
import torch

import gvd_oracle as O
from gvd_b200 import capi, synth

gpu = pytest.mark.gpu


def _attention_ref(qkv, nh, hs, scale):
    nb, R, t = qkv.shape
    HP = t // 3
    q, k, v = (qkv[:, :, i * HP:i * HP + nh * hs].double().reshape(nb, R, nh, hs).permute(0, 2, 1, 3) for i in range(3))
    P = torch.softmax(q @ k.transpose(-1, -2) * scale, -1)
    return (P @ v).permute(0, 2, 1, 3).reshape(nb, R, nh * hs)


def _f16x3_word(k):
    return (k >> 5) * 32 + ((k & 31) >> 1)


def _pack_f16x3(x, scale):
    """gvd_pack_f16x3 on the host: fp32 [rows, K] (K % 32 == 0) -> int32 words, per 32-wide slice 16 hi pairs then 16 lo pairs."""
    x = (np.ascontiguousarray(x, dtype=np.float32) * np.float32(scale)).astype(np.float32)
    a = ((x.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    hi = a.astype(np.float16).view(np.uint16).astype(np.uint32)
    lo = (x - a).astype(np.float16).view(np.uint16).astype(np.uint32)
    rows, K = x.shape
    hw = (hi[:, 0::2] | (hi[:, 1::2] << 16)).reshape(rows, K // 32, 16)
    lw = (lo[:, 0::2] | (lo[:, 1::2] << 16)).reshape(rows, K // 32, 16)
    return np.concatenate([hw, lw], axis=2).reshape(rows, K).view(np.int32)


# amp scales the projections: 1 = flat softmax, 6 = sharply peaked rows (logit range ~ +-80), where the running maximum moves by orders of
# magnitude between key blocks
@pytest.mark.parametrize("nb,nh,R,hs,HP,scale,amp", [(2, 6, 1000, 172, 1032, 1 / 32, 1.0), (2, 6, 1000, 172, 1032, 1 / 32, 6.0),
                                                     (1, 6, 52, 44, 264, 1 / 16, 1.0), (3, 2, 132, 192, 384, 1 / 8, 1.0),
                                                     (1, 1, 4, 4, 4, 1.0, 1.0), (1, 3, 20, 8, 24, 0.5, 3.0),
                                                     (1, 6, 1000, 172, 1032, 1 / 32, 1.0), (5, 6, 1000, 172, 1032, 1 / 32, 1.0)])
@gpu
def test_fused_kernel_matches_fp64(nb, nh, R, hs, HP, scale, amp):
    g = torch.Generator().manual_seed(int(R * 10 + amp + nb))
    qkv = (torch.randn(nb, R, 3 * HP, generator=g) * amp).cuda()
    out = capi.op_self_attention_fused(qkv, nh, hs, scale)
    torch.cuda.synchronize()
    ref = _attention_ref(qkv, nh, hs, scale)
    err = float((out[:, :, :nh * hs].double() - ref.to(out.device)).abs().max())
    assert err <= 4e-5 * max(1.0, float(ref.abs().max())), err
    if nh * hs < HP:
        assert float(out[:, :, nh * hs:].abs().max()) == 0.0


@gpu
def test_image_mode_is_the_packed_fp32_output():
    """Operand-image store mode: every word of the [nb * R, 1056] image row is written (prefilled with NaN), the K padding [1032, 1056) is
    zeros, and the words equal the fp32 mode's output split by the pack pass, bit for bit; the decoded image is the output."""
    nb, nh, R, hs, HP, img_ld = 2, 6, 1000, 172, 1032, 1056
    g = torch.Generator().manual_seed(7)
    qkv = torch.randn(nb, R, 3 * HP, generator=g).cuda()
    out = capi.op_self_attention_fused(qkv, nh, hs, 1 / 32)
    img = torch.full((nb * R, img_ld), 0x7E007E00, dtype=torch.int32, device="cuda")   # fp16 NaN in both halves
    capi.op_self_attention_fused(qkv, nh, hs, 1 / 32, img=img)
    torch.cuda.synchronize()
    words = img.cpu().numpy()
    o = out.reshape(nb * R, HP).cpu().numpy()
    want = _pack_f16x3(np.concatenate([o, np.zeros((nb * R, img_ld - HP), np.float32)], axis=1), 4.0)
    assert np.array_equal(words, want), int((words != want).sum())
    assert not np.any(words[:, [_f16x3_word(k) + d for k in range(HP, img_ld, 2) for d in (0, 16)]])
    halves = words.view(np.uint16).view(np.float16).astype(np.float32).reshape(nb * R, img_ld // 32, 2, 32)
    decoded = ((halves[:, :, 0] + halves[:, :, 1]) / 4.0).reshape(nb * R, img_ld)
    assert np.max(np.abs(decoded[:, :HP] - o)) <= 1e-6 * max(1.0, float(np.abs(o).max()))


@gpu
def test_encoder_output_at_default_backend_matches_oracle():
    """pool_feats (both encoder layers through the fused kernel, default backend 923) of 3 full-size clips against the oracle."""
    capi.set_backend(923)
    opt = synth.make_opt(t_attn_size=10)
    sd = synth.make_state_dict(opt)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    B, T = 3, 10
    R, H = opt.num_sampled_frm * opt.num_prop_per_frm, opt.rnn_size
    inp = synth.make_inputs(opt, B, masked=True)
    keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
    nm.prologue(*(inp[k].cuda() for k in keys))
    torch.cuda.synchronize()
    got = nm.workspace_tensor(B, T, "pool_feats", (B, R, H)).cpu()
    feats = O.prologue(sd, opt, *(inp[k] for k in keys))
    err = float((got.double() - feats["pool_feats"].double()).abs().max())
    assert err <= 1e-4, err


def test_fused_store_plan_covers_every_word_of_the_row_once():
    """The store plan of the fused kernel's image mode at reference-size heads (6 heads of 171 / 169 columns in 172-column slots, n176 product,
    Wo operand row of rup32(6 * 172) = 1056 words): per head CTA, each warp's lane pairs (c, c ^ 1) store 4 columns 8 j + 4 (c >> 1) of one row;
    columns past the slot are dropped, the last head's CTA zeroes the K padding.  Every word of the row is written exactly once, with 8-byte
    aligned word pairs that never straddle a 32-wide K slice, and the pad columns (n >= N_h) are the product's zero columns."""
    nh, hs, NV, img_ld = 6, 172, 176, 1056
    N = [171] * 5 + [169]
    written, zero_cols = {}, set()
    for h in range(nh):
        for c in range(4):
            if c & 1:
                continue                                          # (the odd lane stores the same columns of the row 8 further down)
            for j in range(NV // 8):
                n = 8 * j + 4 * (c >> 1)
                if n >= hs:
                    continue
                gc = h * hs + n
                assert gc % 4 == 0 and (gc & 31) + 4 <= 32
                w = _f16x3_word(gc)
                assert w % 2 == 0
                for d in (w, w + 1, w + 16, w + 17):
                    assert d not in written and 0 <= d < img_ld
                    written[d] = (h, n)
                zero_cols.update(gc + e for e in range(4) if n + e >= N[h])
        if h == nh - 1:
            for gc in range(nh * hs, img_ld, 4):
                w = _f16x3_word(gc)
                for d in (w, w + 1, w + 16, w + 17):
                    assert d not in written
                    written[d] = "pad"
    assert sorted(written) == list(range(img_ld))
    assert zero_cols == {h * hs + n for h in range(nh) for n in range(N[h], hs)}
