"""Video-indexed batches on the device: B events of V videos, the frame features passed once per video (eval_opt['video_idx']).

The definition is the per-clip call on segs_feat[video_idx]: the windowed decode attention against fp64 op by op, every top-down fixture
rerun with video_idx = arange(B), and B = 100 events over V = 28 videos against the per-clip path."""
import gc
import warnings

import numpy as np
import pytest
import torch

from cases import CASES, build_case, load_fixture
from gvd_b200 import capi, synth
from input_mode_cases import INPUT_MODE_CASES
from test_gpu_attn_beam_ops import MIN_VALUE, NAN, _gen

pytestmark = pytest.mark.gpu

KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
TOL = 1e-4
SHARE_TOL = 1e-5


@pytest.fixture(autouse=True, scope="module")
def _release_models():
    """The device memory of this module's models goes back before the next module runs."""
    yield
    _SHARE.clear()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _restore_backend():
    b = capi.get_backend()
    yield
    capi.set_backend(b)


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _model(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _windows(B, T, TC, seed):
    """Full, empty, one-row, ending-at-T, chunk-straddling and past-T windows, then seeded random ones."""
    fixed = [(0, T), (3, 3), (T // 2, T // 2 + 1), (T - 5, T), (TC - 2, TC + 3), (T - 2, T + 4), (-3, 2), (T + 1, T + 5)]
    g = _gen(seed)
    out = []
    for b in range(B):
        if b < len(fixed):
            out.append(fixed[b])
        else:
            lo = int(torch.randint(0, T, (1,), generator=g))
            out.append((lo, int(torch.randint(lo + 1, T + 1, (1,), generator=g))))
    return torch.tensor(out, dtype=torch.int64)


# ------------------------------------------------------------------------------------------------------------ the decode attention, op by op
@pytest.mark.parametrize("mode", ["both", "featmap"])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,V,T,A,H,TC,div", [(12, 5, 40, 128, 248, 16, 1), (12, 3, 37, 96, 128, 8, 3), (10, 4, 480, 512, 1024, 128, 1)])
def test_windowed_attention_against_fp64(B, V, T, A, H, TC, div, fused, mode):
    """gvd_op_attention_video against fp64 on the expanded, masked per-clip features: the temporal attention of row b over video
    video_idx[b / div] with the rows outside its window replaced by (p_conv = ctx2att.bias, conv = 0)."""
    g = _gen(B * T + div)
    Bf, R, RC = B // div, 26, 16
    c = lambda t: t.cuda().contiguous()
    p_pool, pool = c(torch.randn(Bf, R, A, generator=g) * 0.5), c(torch.randn(Bf, R, H, generator=g))
    p_conv, conv = c(torch.randn(V, T, A, generator=g) * 0.5), c(torch.randn(V, T, H, generator=g))
    ctx_bias = c(torch.randn(A, generator=g) * 0.5)
    q = c(torch.randn(B, 2 * A, generator=g) * 0.5)
    w1, w2 = c(torch.randn(A, generator=g) / A ** 0.5), c(torch.randn(A, generator=g) / A ** 0.5)
    b1, b2 = c(torch.randn(1, generator=g) * 0.1), c(torch.randn(1, generator=g) * 0.1)
    am = (torch.rand(Bf, R + 1, generator=g) < 0.25).to(torch.uint8)
    att_mask, out_mask = c(am), c(am)
    vid = c(torch.randint(0, V, (Bf,), generator=g))
    win = c(_windows(Bf, T, TC, B + T))
    nch_r, nch_t = -(-R // RC), -(-T // TC)
    z = torch.full((B, R), NAN, device="cuda")
    x = torch.full((B, H), NAN, device="cuda")
    part = torch.full((B, nch_r + nch_t, H + 4), NAN, device="cuda")
    ticket = torch.zeros(B, dtype=torch.int32, device="cuda") if fused else None
    capi.op_attention_video(vid, win, ctx_bias, p_pool, pool if mode == "both" else None, p_conv, conv, w1, b1, w2, b2, att_mask, out_mask,
                            z, part, x, RC, TC, q=q, ticket=ticket, feat_div=div, att_input_mode=mode)
    torch.cuda.synchronize()
    d = lambda t: t.double()
    idx = torch.arange(B, device="cuda") // div
    t = torch.arange(T, device="cuda")[None, :]
    keep = ((t >= win[:, 0:1]) & (t < win[:, 1:2]))[idx]
    pc = torch.where(keep[..., None], d(p_conv)[vid[idx]], d(ctx_bias))
    cv = d(conv)[vid[idx]] * keep[..., None]
    s = torch.tanh(pc + d(q)[:, None, :A]) @ d(w1) + d(b1)
    ref = torch.einsum("bt,bth->bh", torch.softmax(s, 1), cv)
    zr = (torch.tanh(d(p_pool)[idx] + d(q)[:, None, A:]) @ d(w2) + d(b2)).masked_fill(att_mask[idx][:, 1:].bool(), MIN_VALUE)
    if mode == "both":
        ref = ref + torch.einsum("br,brh->bh", torch.softmax(zr, 1), d(pool)[idx])
    assert _maxerr(x, ref) <= 1e-5
    assert _maxerr(z, zr) <= 1e-5
    empty = ~keep.any(1)
    if mode == "featmap" and bool(empty.any()):
        assert float(x[empty].abs().max()) == 0.0                    # an empty window: uniform weights over zero rows
    if fused:
        assert int(ticket.abs().sum()) == 0


@pytest.mark.parametrize("q_S", [1, 3])
def test_windowed_attention_query_from_split_k_planes(q_S):
    """The query as split-K planes + bias (the fp16x3 decode path) gives the same result as the summed query."""
    g = _gen(50 + q_S)
    B, V, T, A, H, R, RC, TC = 8, 3, 50, 128, 256, 13, 16, 16
    c = lambda t: t.cuda().contiguous()
    args = [c(torch.randn(B, R, A, generator=g) * 0.5), c(torch.randn(B, R, H, generator=g)), c(torch.randn(V, T, A, generator=g) * 0.5),
            c(torch.randn(V, T, H, generator=g)), c(torch.randn(A, generator=g) / 12), c(torch.randn(1, generator=g) * 0.1),
            c(torch.randn(A, generator=g) / 12), c(torch.randn(1, generator=g) * 0.1), c(torch.zeros(B, R + 1, dtype=torch.uint8)),
            c(torch.zeros(B, R + 1, dtype=torch.uint8))]
    vid, win, cb = c(torch.randint(0, V, (B,), generator=g)), c(_windows(B, T, TC, 9)), c(torch.randn(A, generator=g))
    q_part = c(torch.randn(q_S, B, 2 * A, generator=g) * 0.3)
    q_bias = c(torch.randn(2 * A, generator=g) * 0.1)
    outs = []
    for kw in (dict(q_part=q_part, q_bias=q_bias), dict(q=(q_part.double().sum(0) + q_bias.double()).float().contiguous())):
        z = torch.full((B, R), NAN, device="cuda")
        x = torch.full((B, H), NAN, device="cuda")
        part = torch.full((B, 1 + -(-T // TC), H + 4), NAN, device="cuda")
        capi.op_attention_video(vid, win, cb, *args, z, part, x, RC, TC, ticket=torch.zeros(B, dtype=torch.int32, device="cuda"), **kw)
        outs.append(x)
    torch.cuda.synchronize()
    assert _maxerr(outs[0], outs[1]) <= 1e-5


# ------------------------------------------------------------------------------------------------------------ the fixtures, video_idx = arange(B)
_TOPDOWN = {**{n: c for n, c in CASES.items() if c["kind"] in ("greedy", "beam", "mle", "grd")},
            **{n: c for n, c in INPUT_MODE_CASES.items() if c["kind"] in ("greedy", "beam", "mle", "grd")}}
_MULTINOMIAL = {"multinomial_T10_B3": (dict(kind="greedy", B=3, opt=dict(t_attn_size=10)), 1.0, 2024),
                "multinomial_small_B5_t07": (dict(CASES["greedy_small_B5"]), 0.7, 7),
                "multinomial_small_B5_t15": (dict(CASES["greedy_small_B5"]), 1.5, 15)}
def _case(name, case):
    """(opt, state_dict, inputs, module): built per test, so that no full-size model outlives it."""
    opt, sd, inp = build_case(case)
    return opt, sd, inp, _model(opt, sd)


def _video_call(model, inp, mode, eval_opt):
    dev = {k: v.cuda() for k, v in inp.items()}
    B = dev["ppls"].shape[0]
    eval_opt = dict(eval_opt, video_idx=torch.arange(B, device="cuda"))
    d = dev.get
    with torch.no_grad():
        if mode == "sample":
            out = model._sample(*(dev[k] for k in KEYS), eval_opt)
        else:
            out = model(d("segs_feat"), d("input_seq"), d("gt_seq"), d("num"), d("ppls"), d("gt_boxes"), d("mask_boxes"), d("ppls_feat"),
                        d("frm_mask"), d("sample_idx"), d("pnt_mask"), mode, eval_opt)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", sorted(_TOPDOWN))
def test_fixtures_with_identity_video_index(name):
    case = _TOPDOWN[name]
    opt, sd, inp, model = _case(name, case)
    fx = load_fixture(name)
    kind = case["kind"]
    if kind == "greedy":
        seq, logp, att2, _ = _video_call(model, inp, "sample", {"sample_max": 1, "beam_size": 1})
        assert np.array_equal(seq.cpu().numpy(), fx["seq"])
        assert np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL and np.max(np.abs(att2.cpu().numpy() - fx["att2"])) <= TOL
    elif kind == "beam":
        seq, logp, att, _ = _video_call(model, inp, "sample", {"beam_size": case["beam_size"]})
        assert np.array_equal(seq.cpu().numpy(), fx["seq"]) and np.array_equal(att.cpu().numpy(), fx["att2_idx"])
        assert np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL
    elif kind == "mle":
        got = np.array([float(v) for v in _video_call(model, inp, "MLE", {})])
        ref = fx["losses"]
        assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.nanmax(np.abs(got - ref)) <= TOL
    else:
        cls_pred, att_idx, grd_idx = _video_call(model, inp, "GRD", {})
        assert np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
        assert np.array_equal(att_idx.cpu().numpy(), fx["att_idx"]) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


@pytest.mark.parametrize("name", sorted(_MULTINOMIAL))
def test_multinomial_fixtures_with_identity_video_index(name):
    case, tau, seed = _MULTINOMIAL[name]
    opt, sd, inp, model = _case(name, case)
    fx = load_fixture(name)
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    B, T = inp["segs_feat"].shape[:2]
    nm.prologue(*(dev[k] for k in KEYS), video_idx=torch.arange(B, device="cuda"))
    seq, logp, att2 = (o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], seed, tau))
    assert np.array_equal(seq.numpy(), fx["seq"])
    assert np.max(np.abs(logp.numpy() - fx["logp"])) <= TOL and np.max(np.abs(att2.numpy() - fx["att2"])) <= TOL


# ------------------------------------------------------------------------------------------------------------ sharing: B = 100 over V = 28
_SHARE = {}
_SHARE_OPT = dict(CASES["greedy_small_B5"]["opt"], t_attn_size=48)


def _share(mode):
    if mode not in _SHARE:
        opt = synth.make_opt(**dict(_SHARE_OPT, att_input_mode=mode))
        sd = synth.make_state_dict(opt, seed=3)
        inp = synth.make_video_inputs(opt, 100, 28, seed=11)
        _SHARE[mode] = (opt, sd, inp, _model(opt, sd))
    return _SHARE[mode]


def _both_paths(model, inp, run):
    """run(nm, dev, video_idx or None) once on the video batch and once per clip on segs_feat[video_idx]."""
    nm = model._native_model()
    dev = {k: v.cuda() for k, v in inp.items()}
    per_clip = dict(dev, segs_feat=dev["segs_feat"][dev["video_idx"]].contiguous())
    a = run(nm, dev, dev["video_idx"])
    b = run(nm, per_clip, None)
    torch.cuda.synchronize()
    return a, b


@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("mode", ["both", "featmap", "dual_region"])
def test_shared_videos_greedy_equals_per_clip(mode, backend):
    capi.set_backend(backend)
    opt, sd, inp, model = _share(mode)
    B, T = inp["ppls"].shape[0], opt.t_attn_size

    def run(nm, dev, vid):
        nm.prologue(*(dev[k] for k in KEYS), video_idx=vid)
        out = nm.decode_greedy(B, T, dev["pnt_mask"])
        conv = nm.workspace_tensor(B, T, "conv_feats", (dev["segs_feat"].shape[0], T, opt.rnn_size)).clone()
        pconv = nm.workspace_tensor(B, T, "p_conv_feats", (dev["segs_feat"].shape[0], T, opt.att_hid_size)).clone()
        return [o.cpu() for o in out] + [conv.cpu(), pconv.cpu()]

    (seq, logp, att2, conv_v, pconv_v), (seq0, logp0, att20, conv_c, pconv_c) = _both_paths(model, inp, run)
    assert torch.equal(seq, seq0)
    assert _maxerr(logp, logp0) <= SHARE_TOL and _maxerr(att2, att20) <= SHARE_TOL
    if mode != "dual_region":                # (dual_region runs no frame branch)
        vid, win = inp["video_idx"], inp["sample_idx"]
        t = torch.arange(T)[None, :]
        keep = (t >= win[:, 0:1]) & (t < win[:, 1:2])
        # the frame GEMMs run with V * T instead of B * T rows, which may change their tiling: equal up to the last bits
        assert _maxerr(conv_v[vid][keep], conv_c[keep]) <= SHARE_TOL and _maxerr(pconv_v[vid][keep], pconv_c[keep]) <= SHARE_TOL


@pytest.mark.parametrize("mode", ["both", "featmap"])
def test_shared_videos_multinomial_equals_per_clip(mode):
    opt, sd, inp, model = _share(mode)
    B, T = inp["ppls"].shape[0], opt.t_attn_size

    def run(nm, dev, vid):
        nm.prologue(*(dev[k] for k in KEYS), video_idx=vid)
        return [o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], 1234, 0.8)]

    (seq, logp, att2), (seq0, logp0, att20) = _both_paths(model, inp, run)
    assert torch.equal(seq, seq0)
    assert _maxerr(logp, logp0) <= SHARE_TOL and _maxerr(att2, att20) <= SHARE_TOL


def test_shared_videos_beam_equals_per_clip():
    opt, sd, inp, model = _share("both")
    B, T, K = inp["ppls"].shape[0], opt.t_attn_size, 3

    def run(nm, dev, vid):
        nm.prologue(*(dev[k] for k in KEYS), beam=K, video_idx=vid)
        return [o.cpu() for o in nm.beam_decode(B, T, K, dev["pnt_mask"])]

    (seq, logp, att), (seq0, logp0, att0) = _both_paths(model, inp, run)
    # a beam whose two best continuations are closer than the parity tolerance may rank them either way: such clips are exempt
    near = torch.zeros(B, dtype=torch.bool)
    diff = (seq != seq0).any(1) | (att != att0).any(1)
    if bool(diff.any()):
        near = (logp - logp0).abs().max(1).values <= SHARE_TOL
    assert bool((~diff | near).all())
    assert _maxerr(logp[~diff], logp0[~diff]) <= SHARE_TOL


def test_shared_videos_teacher_forced_equals_per_clip():
    opt = synth.make_opt(**_SHARE_OPT)
    sd = synth.make_state_dict(opt, seed=3)
    inp = synth.make_video_inputs(opt, 30, 9, seed=12, train=True)
    model = _model(opt, sd)
    dev = {k: v.cuda() for k, v in inp.items()}
    args = lambda segs: (segs, dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"], dev["ppls_feat"],
                         dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"])
    per_clip = dev["segs_feat"][dev["video_idx"]].contiguous()
    with torch.no_grad():
        mle = torch.cat(model(*args(dev["segs_feat"]), "MLE", {"video_idx": dev["video_idx"]}))
        mle0 = torch.cat(model(*args(per_clip), "MLE"))
        grd = model(*args(dev["segs_feat"]), "GRD", {"video_idx": dev["video_idx"]})
        grd0 = model(*args(per_clip), "GRD")
    torch.cuda.synchronize()
    assert _maxerr(mle, mle0) <= SHARE_TOL
    assert all(torch.equal(a, b) for a, b in zip(grd, grd0))


def test_shared_videos_host_buffer_equals_device_path():
    opt, sd, inp, model = _share("both")
    B, T = inp["ppls"].shape[0], opt.t_attn_size
    nm = model._native_model()
    dev = {k: v.cuda() for k, v in inp.items()}
    sim = nm.prologue(*(dev[k] for k in KEYS), video_idx=dev["video_idx"])
    seq, logp, att2 = (o.cpu() for o in nm.decode_greedy(B, T, dev["pnt_mask"]))
    sim = sim.cpu()
    pinned = {k: v.pin_memory() for k, v in inp.items()}
    out = nm.sample_greedy_host(*(pinned[k] for k in KEYS), video_idx=pinned["video_idx"])
    assert torch.equal(out["seq"], seq) and torch.equal(out["logp"], logp) and torch.equal(out["att2"], att2) and torch.equal(out["sim"], sim)
    bad = pinned["video_idx"].clone()
    bad[3] = 28
    with pytest.raises(ValueError):
        nm.sample_greedy_host(*(pinned[k] for k in KEYS), video_idx=bad)


def test_per_clip_prologue_after_video_prologue_restores_the_per_clip_layout():
    opt, sd, inp, model = _share("both")
    B, T = inp["ppls"].shape[0], opt.t_attn_size
    nm = model._native_model()
    dev = {k: v.cuda() for k, v in inp.items()}
    per_clip = dict(dev, segs_feat=dev["segs_feat"][dev["video_idx"]].contiguous())
    nm.prologue(*(per_clip[k] for k in KEYS))
    ref = [o.cpu() for o in nm.decode_greedy(B, T, dev["pnt_mask"])]
    nm.prologue(*(dev[k] for k in KEYS), video_idx=dev["video_idx"])
    nm.decode_greedy(B, T, dev["pnt_mask"])
    nm.prologue(*(per_clip[k] for k in KEYS))
    again = [o.cpu() for o in nm.decode_greedy(B, T, dev["pnt_mask"])]
    assert all(torch.equal(a, b) for a, b in zip(ref, again))


def test_refusals_on_the_device():
    opt, sd, inp, model = _share("both")
    dev = {k: v.cuda() for k, v in inp.items()}
    call = lambda vid: model(dev["segs_feat"], None, None, dev["num"], dev["ppls"], None, None, dev["ppls_feat"], None, dev["sample_idx"],
                             dev["pnt_mask"], "sample", {"video_idx": vid})
    with pytest.raises(ValueError):
        call(dev["video_idx"].int())
    with pytest.raises(ValueError):
        call(torch.cat((dev["video_idx"], dev["video_idx"][:1])))
    bad = dev["video_idx"].clone()
    bad[7] = 28
    with pytest.raises(ValueError):
        call(bad)
    with pytest.raises(ValueError):
        call(dev["video_idx"].cpu())
