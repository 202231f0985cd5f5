"""Video-indexed batches, host side: the windowed closed form of the temporal attention against the per-clip oracle at fp64, the frame
bytes a video batch moves, and the refusals of the new argument."""
import os
import sys
import warnings

import pytest
import torch

from cases import SMALL
import gvd_oracle as O
from gvd_b200 import capi, synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import video_batch_bench as VB  # noqa: E402


def _video_problem(B=9, V=4, T=12, seed=3):
    opt = synth.make_opt(**dict(SMALL, t_attn_size=T))
    W = {k: v.double() if v.is_floating_point() else v for k, v in synth.make_state_dict(opt, seed=seed).items()}
    inp = synth.make_video_inputs(opt, B, V, seed=seed)
    return opt, W, inp


def test_synth_video_inputs_cover_the_window_cases():
    opt, _, inp = _video_problem()
    T = opt.t_attn_size
    win, vid = inp["sample_idx"], inp["video_idx"]
    n_in = (torch.minimum(win[:, 1], torch.tensor(T)) - win[:, 0].clamp(min=0)).clamp(min=0)
    assert inp["segs_feat"].shape == (4, T, opt.fc_feat_size) and vid.dtype == torch.int64 and vid.shape == (9,)
    assert sorted(set(vid.tolist())) == [0, 1, 2, 3]
    assert (n_in == T).any() and (n_in == 0).any() and (n_in == 1).any() and (win[:, 1] == T).any() and (win[:, 1] > T).any()


def test_closed_form_equals_the_per_clip_oracle():
    """The per-clip oracle on segs_feat[video_idx] (masked frame branch, softmax over all T rows) equals the windowed form on the video-level,
    unmasked frame branch: the in-window rows of the video plus one term (s0, T - n_in) for the rows outside, at fp64."""
    opt, W, inp = _video_problem()
    T, A = opt.t_attn_size, opt.att_hid_size
    segs, vid, win = inp["segs_feat"].double(), inp["video_idx"], inp["sample_idx"]
    conv_c, pconv_c = O.frame_branch(W, segs[vid], win)                          # the per-clip restatement
    full = torch.tensor([[0, T]] * segs.shape[0])
    conv_v, pconv_v = O.frame_branch(W, segs, full)                               # video level, unmasked
    t = torch.arange(T)[None, :]
    keep = (t >= win[:, 0:1]) & (t < win[:, 1:2])
    assert torch.allclose(conv_c[keep], conv_v[vid][keep], rtol=0, atol=1e-12)
    assert torch.allclose(pconv_c[keep], pconv_v[vid][keep], rtol=0, atol=1e-12)
    assert torch.equal(conv_c[~keep], torch.zeros_like(conv_c[~keep]))
    assert torch.allclose(pconv_c[~keep], W["ctx2att.bias"].expand_as(pconv_c[~keep]), rtol=0, atol=1e-12)
    g = torch.Generator().manual_seed(0)
    q = torch.randn(segs[vid].shape[0], A, generator=g, dtype=torch.float64) * 0.5
    w, b = W["core.attention.alpha_net.weight"].view(-1), W["core.attention.alpha_net.bias"]
    s = torch.tanh(pconv_c + q[:, None]) @ w + b
    att = torch.einsum("bt,bth->bh", torch.softmax(s, 1), conv_c)
    for i in range(len(vid)):
        rows = keep[i].nonzero().view(-1)
        si = torch.tanh(pconv_v[vid[i], rows] + q[i]) @ w + b
        s0 = torch.tanh(W["ctx2att.bias"] + q[i]) @ w + b
        n_out = T - len(rows)
        m = torch.cat((si, s0.view(1) if n_out else si[:0])).max()
        l = torch.exp(si - m).sum() + n_out * torch.exp(s0 - m).sum()
        acc = torch.exp(si - m) @ conv_v[vid[i], rows]
        assert torch.allclose(acc / l, att[i], rtol=0, atol=1e-12), i


def test_frame_bytes_of_a_video_batch():
    """The host-buffer entry point stages V videos' frames: V * T * F * 4 bytes instead of B * T * F * 4."""
    assert VB.frame_h2d_bytes(B=100, V=28, T=480, F=3072) == 28 * 480 * 3072 * 4
    assert VB.frame_h2d_bytes(B=100, V=None, T=480, F=3072) == 100 * 480 * 3072 * 4
    win = torch.tensor([[0, 480], [10, 10], [470, 500], [-5, 3]])
    # per-clip path: every row of every clip's copy; video path: in-window rows only
    assert VB.temporal_attn_bytes(win, T=480, A=512, H=1024, video=False) == 4 * 480 * (512 + 1024) * 4
    assert VB.temporal_attn_bytes(win, T=480, A=512, H=1024, video=True) == (480 + 0 + 10 + 3) * (512 + 1024) * 4


def _batch(B=6, V=3):
    opt = synth.make_opt(**dict(SMALL, t_attn_size=8))
    return opt, synth.make_video_inputs(opt, B, V, seed=4)


def test_video_batch_validation():
    opt, inp = _batch()
    args = lambda vid: (inp["segs_feat"], vid, inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    assert capi.check_video_batch(*args(inp["video_idx"])) == 6
    with pytest.raises(ValueError, match="int64"):
        capi.check_video_batch(*args(inp["video_idx"].int()))
    with pytest.raises(ValueError, match="1-D"):
        capi.check_video_batch(*args(inp["video_idx"].view(2, 3)))
    with pytest.raises(ValueError, match="rows"):
        capi.check_video_batch(*args(inp["video_idx"][:5]))
    bad = inp["video_idx"].clone()
    bad[2] = 3
    with pytest.raises(ValueError, match=r"\[0, 3\)"):
        capi.check_video_batch(*args(bad))
    bad[2] = -1
    with pytest.raises(ValueError):
        capi.check_video_batch(*args(bad))
    # segs_feat with fewer rows than the videos video_idx names
    with pytest.raises(ValueError):
        capi.check_video_batch(inp["segs_feat"][:2], *args(inp["video_idx"])[1:])


def _module(**over):
    from gvd_b200.misc.AttModel import TopDownModel
    opt = synth.make_opt(**dict(SMALL, t_attn_size=8, **over))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return opt, TopDownModel(opt)


def _call(model, inp, mode):
    z = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8)
    return model(inp["segs_feat"], z, z, inp["num"], inp["ppls"], z, z, inp["ppls_feat"], z, inp["sample_idx"], inp["pnt_mask"], mode,
                 {"video_idx": inp["video_idx"]})


@pytest.mark.parametrize("mode", ["sample", "MLE", "GRD"])
def test_transformer_refuses_video_idx(mode):
    opt, model = _module(att_model="transformer")
    _, inp = _batch()
    model.eval()
    with pytest.raises(NotImplementedError, match="transformer"):
        _call(model, inp, mode)


def test_train_mode_refuses_video_idx():
    opt, model = _module()
    _, inp = _batch()
    model.train()
    with pytest.raises(NotImplementedError, match="training"):
        _call(model, inp, "MLE")
