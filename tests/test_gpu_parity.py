"""GPU parity tests: the CUDA path (through the C-ABI / the nn.Module surface) against the CPU
oracle on the same seeded inputs, and against the committed golden fixtures of the reference.

Bars (BASELINE.json north_star): greedy token ids bit-exact; attention logits, similarity matrix,
log-probs and prologue activations within 1e-4 abs (fp32)."""
import warnings

import numpy as np
import pytest
import torch

import gvd_oracle as O
import gvd_b200.synth as synth
from cases import CASES, SMALL, build_case, load_fixture, subsample
from gvd_b200 import capi

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _model(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


def _sample(model, inp):
    dev = {k: v.cuda() for k, v in inp.items()}
    d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
    with torch.no_grad():
        out = model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"],
                    dev["pnt_mask"], "sample", {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    return out


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


# ----------------------------------------------------------------------------- single kernels
@pytest.mark.parametrize("M,N,K", [(1, 8, 4), (100, 1024, 3124), (1000, 432, 2048), (257, 130, 36), (64, 4905, 1024),
                                   (2000, 2048, 2048), (130, 96, 252)])
@pytest.mark.parametrize("act", [0, 1])
def test_linear_kernel(M, N, K, act):
    g = torch.Generator().manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = A.double() @ W.double().t() + b.double()
    if act:
        ref = ref.clamp(min=0)
    out = capi.op_linear(A.cuda(), W.cuda(), b.cuda(), act)
    torch.cuda.synchronize()
    assert _maxerr(out, ref) <= 2e-5 * max(1.0, float(ref.abs().max()))


def test_tanh_accuracy():
    x = torch.cat((torch.linspace(-12, 12, 200001), torch.tensor([0.0, 1e-8, -1e-8, 30.0, -30.0, 1e-3, -1e-3])))
    y = capi.op_tanh(x.cuda())
    torch.cuda.synchronize()
    err = _maxerr(y, torch.tanh(x.double()))
    assert err <= 4e-7, err          # absolute; the attention logit sums 512 of these times |w|


# ----------------------------------------------------------------------------- greedy decode
GREEDY = [n for n, c in CASES.items() if c["kind"] == "greedy"]


@pytest.mark.parametrize("name", GREEDY)
def test_greedy_matches_oracle_and_reference_fixture(name):
    case = CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    model = _model(opt, sd)
    seq, att2, sim = _sample(model, inp)
    B, T = inp["segs_feat"].shape[:2]
    R, H, A = opt.num_sampled_frm * opt.num_prop_per_frm, opt.rnn_size, opt.att_hid_size
    nm = model._native
    feats = O.prologue(sd, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    shapes = dict(fc_feats=(B, H), g_pool=(B, R, 2048), pool_embed=(B, R, H), pool_feats=(B, R, H), p_pool_feats=(B, R, A),
                  conv_feats=(B, T, H), p_conv_feats=(B, T, A))
    for k, shp in shapes.items():
        got = nm.workspace_tensor(B, T, k, shp).cpu()
        assert _maxerr(got, feats[k]) <= TOL, (k, _maxerr(got, feats[k]))          # full tensor vs live oracle
        if k in fx:
            assert np.max(np.abs(subsample(k, got).numpy() - fx[k])) <= TOL, k        # vs the reference's own output
    oseq, ologp, oatt2, osim = O.sample_greedy(sd, opt, inp, feats=feats)
    # token ids: bit-exact against the oracle AND the reference fixture
    assert torch.equal(seq.cpu(), oseq)
    assert np.array_equal(seq.cpu().numpy(), fx["seq"])
    assert fx["min_margin"] > 10 * TOL / 10 and fx["unk_top1_steps"] >= 0
    assert _maxerr(att2, oatt2) <= TOL
    assert np.max(np.abs(att2.cpu().numpy() - fx["att2"])) <= TOL
    assert torch.equal(att2.cpu() == -1e8, oatt2 == -1e8)                             # mask fills are exact
    assert _maxerr(sim, osim) <= TOL
    assert np.max(np.abs(subsample("sim_mat", sim.cpu()).numpy() - fx["sim_mat"])) <= TOL
    assert np.max(np.abs(sim.sum(dim=1).cpu().numpy() - fx["sim_mat_colsum"])) <= TOL
    # log-probs through the C-ABI (forward() drops them, like the reference's forward)
    nm.prologue(*(inp[k].cuda() for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")))
    seq2, logp, att2b = nm.decode_greedy(B, T, inp["pnt_mask"].cuda())
    torch.cuda.synchronize()
    assert torch.equal(seq2, seq) and torch.equal(att2b, att2)                        # deterministic re-run
    assert _maxerr(logp, ologp) <= TOL
    assert np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL


@pytest.mark.parametrize("serial", [False, True])
def test_host_buffer_entry_point_matches_device_path(serial):
    """gvd_sample_greedy_host (pinned host buffers -> H2D on the copy stream -> region stages, frame stages on their own stream -> loop
    -> D2H) returns exactly the device path's outputs, also with the frame stages on the caller's stream (serial: under the stage profiler,
    which runs them there).  The chunked schedule at the benchmarked size is checked by test_full_batch_properties_B100."""
    opt, sd, inp = build_case(CASES["greedy_small_B5"])
    model = _model(opt, sd)
    seq, att2, sim = _sample(model, inp)
    pinned = {k: inp[k].pin_memory() for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")}
    capi.profile_enable(serial)
    try:
        out = model._native.sample_greedy_host(pinned["segs_feat"], pinned["ppls"], pinned["num"], pinned["ppls_feat"],
                                               pinned["sample_idx"], pinned["pnt_mask"])
    finally:
        capi.profile_enable(False)
        capi.profile_reset()
    assert torch.equal(out["seq"], seq.cpu())
    assert torch.equal(out["att2"], att2.cpu())
    assert torch.equal(out["sim"], sim.cpu())
    oseq, _, oatt2, osim = O.sample_greedy(sd, opt, inp)
    assert torch.equal(out["seq"], oseq) and _maxerr(out["att2"], oatt2) <= TOL and _maxerr(out["sim"], osim) <= TOL


def test_empty_and_fully_masked_edges():
    """All proposals masked on one clip (uniform softmax over -1e8 logits, AttModel.py:99-102) and a
    single-frame segment; compared with the oracle."""
    opt = synth.make_opt(**SMALL)
    sd = synth.make_state_dict(opt, seed=3)
    inp = synth.make_inputs(opt, 3, seed=11)
    inp["pnt_mask"][1, 1:] = 1
    inp["ppls"][1] = 0
    inp["ppls_feat"][1] = 0
    inp["sample_idx"][2] = torch.tensor([3, 4])
    inp["sample_idx"][0] = torch.tensor([0, 0])          # empty segment: every frame row zeroed
    model = _model(opt, sd)
    seq, att2, sim = _sample(model, inp)
    oseq, _, oatt2, osim = O.sample_greedy(sd, opt, inp)
    assert torch.equal(seq.cpu(), oseq)
    assert _maxerr(att2, oatt2) <= TOL and _maxerr(sim, osim) <= TOL
    assert bool((att2[1] == -1e8).all())


def test_error_reporting_through_the_abi():
    opt, sd, inp = build_case(CASES["greedy_small_B5"])
    nm = capi.NativeModel(opt)
    with pytest.raises(capi.GvdError, match="never set|finalized"):
        nm.prologue(*(inp[k].cuda() for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")))
    bad = dict(sd)
    bad["logit.bias"] = torch.zeros(3)
    with pytest.raises(capi.GvdError, match="size mismatch"):
        nm.load_state_dict(bad)
    with pytest.raises(capi.GvdError, match="CUDA tensor"):
        nm.load_state_dict(sd)
        nm.prologue(*(inp[k] for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")))


# ----------------------------------------------------------------------------- full-size properties
KEYS6 = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


@pytest.mark.parametrize("T,n_oracle", [(10, 16), (480, 4)])
def test_full_batch_properties_B100(T, n_oracle):
    """BASELINE config 2 size (B=100, R=1000; T=10 = the BASELINE literal, T=480 = the reference default opts.py:50): the oracle is too
    slow for the whole batch, so (1) clips are independent — clips decoded inside the batch of 100 give the same tokens / logits as the
    same clips decoded in a small batch, and THAT batch (16 clips spread over the 100 at T=10, 4 at T=480) is checked against the
    oracle; (2) run-to-run determinism; (3) the class softmax columns sum to 1; (4) mask fills exact; (5) the host-buffer entry point
    (chunked H2D schedule of gvd_sample_greedy_host at the benchmarked size) returns exactly the device path's outputs."""
    opt = synth.make_opt(t_attn_size=T)
    sd = synth.make_state_dict(opt)
    model = _model(opt, sd)
    inp = synth.make_inputs(opt, 100, seed=2024 + T)
    seq, att2, sim = _sample(model, inp)
    seq_b, att2_b, sim_b = _sample(model, inp)
    assert torch.equal(seq, seq_b) and torch.equal(att2, att2_b) and torch.equal(sim, sim_b)
    assert float((sim.sum(dim=1) - 1).abs().max()) <= 1e-5
    m = inp["pnt_mask"][:, 1:].bool().cuda()
    assert bool((att2[m.unsqueeze(1).expand_as(att2)] == -1e8).all())
    assert bool((att2[~m.unsqueeze(1).expand_as(att2)] > -1e7).all())
    assert len(torch.unique(seq)) > 20           # captions are not degenerate
    # (5) host buffers -> chunked H2D -> prologue -> loop -> D2H, at full size
    pinned = {k: inp[k].pin_memory() for k in KEYS6}
    out = model._native.sample_greedy_host(*(pinned[k] for k in KEYS6))
    assert torch.equal(out["seq"], seq.cpu())
    assert torch.equal(out["att2"], att2.cpu())
    assert torch.equal(out["sim"], sim.cpu())
    del out, pinned
    # (1) clip independence, then the oracle on the small batch
    pick = sorted(set(int(round(i * 99 / (n_oracle - 1))) for i in range(n_oracle)))
    assert len(pick) == n_oracle and pick[0] == 0 and pick[-1] == 99
    sub = {k: v[pick].contiguous() for k, v in inp.items()}
    seq4, att4, sim4 = _sample(model, sub)
    assert torch.equal(seq4, seq[pick])
    assert _maxerr(att4, att2[pick]) <= 1e-5 and _maxerr(sim4, sim[pick]) <= 1e-6
    oseq, _, oatt2, osim = O.sample_greedy(sd, opt, sub)
    assert torch.equal(seq4.cpu(), oseq)
    assert _maxerr(att4, oatt2) <= TOL and _maxerr(sim4, osim) <= TOL


# ----------------------------------------------------------------------------- beam search
BEAM = [n for n, c in CASES.items() if c["kind"] == "beam"]


@pytest.mark.parametrize("name", BEAM)
def test_beam_matches_oracle_and_repaired_reference(name):
    """Device-side batched beam search vs the oracle (live) and the shimmed reference's fixture:
    token ids and attended-region indices bit-exact, log-probs within 1e-4."""
    case = CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    model = _model(opt, sd)
    dev = {k: v.cuda() for k, v in inp.items()}
    with torch.no_grad():
        seq, logp, att, sim = model._sample(dev["segs_feat"], dev["ppls"], dev["num"], dev["ppls_feat"], dev["sample_idx"],
                                            dev["pnt_mask"], {"beam_size": case["beam_size"]})
        d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
        seq_f, att_f, sim_f = model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"],
                                    dev["pnt_mask"], "sample", {"sample_max": 1, "beam_size": case["beam_size"]})
    torch.cuda.synchronize()
    oseq, ologp, oatt = O.sample_beam(sd, opt, inp, case["beam_size"])
    assert torch.equal(seq.cpu(), oseq) and np.array_equal(seq.cpu().numpy(), fx["seq"])
    assert torch.equal(att.cpu(), oatt) and np.array_equal(att.cpu().numpy(), fx["att2_idx"])
    assert _maxerr(logp, ologp) <= TOL and np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL
    assert torch.equal(seq_f, seq) and torch.equal(att_f, att)          # forward(..., 'sample') with beam_size > 1 works (repair D2)
    # a greedy decode right after must not be disturbed by the larger beam workspace
    seq_g, att_g, _ = _sample(model, inp)
    og = O.sample_greedy(sd, opt, inp)
    assert torch.equal(seq_g.cpu(), og[0])


# ----------------------------------------------------------------------------- teacher-forced: MLE losses / GRD
def _teacher(model, inp, mode):
    dev = {k: v.cuda() for k, v in inp.items()}
    with torch.no_grad():
        out = model(dev["segs_feat"], dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"],
                    dev["ppls_feat"], dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], mode)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["kind"] == "mle"])
def test_mle_losses_match_oracle_and_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    model = _model(opt, sd)
    losses = _teacher(model, inp, "MLE")
    assert all(tuple(l.shape) == (1,) for l in losses)                  # model.py:483 (unsqueeze(0) for DataParallel gather)
    got = np.array([float(l) for l in losses])
    ref = np.array([float(x) for x in O.forward_teacher(sd, opt, inp)])
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isnan(got), np.isnan(fx["losses"]))   # quirk Q11: empty set => NaN
    ok = ~np.isnan(got)
    assert np.max(np.abs(got[ok] - ref[ok])) <= TOL and np.max(np.abs(got[ok] - fx["losses"][ok])) <= TOL, (got, ref)
    again = np.array([float(l) for l in _teacher(model, inp, "MLE")])
    assert np.array_equal(got, again, equal_nan=True)                   # fixed-order reductions: bitwise reproducible


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["kind"] == "grd"])
def test_grd_outputs_match_oracle_and_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    model = _model(opt, sd)
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    ocls, oatt, ogrd = O.forward_teacher(sd, opt, inp, eval_obj_ground=True)
    assert torch.equal(cls_pred.cpu(), ocls) and np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
    assert torch.equal(att_idx.cpu(), oatt) and np.array_equal(att_idx.cpu().numpy(), fx["att_idx"])
    assert torch.equal(grd_idx.cpu(), ogrd) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


def test_train_mode_dispatch():
    """model.train(): 'MLE' is the training forward (autograd node over the explicit backward: losses require grad; with dropout off and
    the batch statistics of BatchNorm they differ from the eval-mode losses only through BatchNorm); the evaluation modes 'GRD' and
    'sample' refuse to run in train mode (main.py:90,315 switch to eval first) instead of silently using train-mode arithmetic."""
    opt, sd, inp = build_case(CASES["mle_small_B5"])
    model = _model(opt, sd).train()
    model.train_dropout = False
    dv = {k: v.cuda() for k, v in inp.items()}
    losses = model(dv["segs_feat"], dv["input_seq"], dv["gt_seq"], dv["num"], dv["ppls"], dv["gt_boxes"], dv["mask_boxes"], dv["ppls_feat"],
                   dv["frm_mask"], dv["sample_idx"], dv["pnt_mask"], "MLE")
    assert all(l.shape == (1,) and l.requires_grad for l in losses) and all(torch.isfinite(l).all() for l in losses)
    with pytest.raises(capi.GvdError):
        _teacher(model, inp, "GRD")
    dev = {k: v.cuda() for k, v in inp.items()}
    d = torch.zeros(inp["ppls"].shape[0], dtype=torch.uint8, device="cuda")
    with pytest.raises(capi.GvdError):
        model(dev["segs_feat"], d, d, dev["num"], dev["ppls"], d, d, dev["ppls_feat"], d, dev["sample_idx"], dev["pnt_mask"], "sample",
              {"sample_max": 1, "beam_size": 1})


def test_beam_full_batch_properties_B100():
    """BASELINE config 4 size (B=100, beam 3): clips are independent — a clip searched inside the batch of 100 gives the
    same tokens / region indices as in a batch of 8 (spread over the 100) that the oracle verifies; run-to-run determinism."""
    opt = synth.make_opt(t_attn_size=10)
    sd = synth.make_state_dict(opt)
    model = _model(opt, sd)
    inp = synth.make_inputs(opt, 100, seed=2024)
    dev = {k: v.cuda() for k, v in inp.items()}

    def run(d):
        with torch.no_grad():
            out = model._sample(d["segs_feat"], d["ppls"], d["num"], d["ppls_feat"], d["sample_idx"], d["pnt_mask"], {"beam_size": 3})
        torch.cuda.synchronize()
        return out
    seq, logp, att, _ = run(dev)
    seq_b, logp_b, att_b, _ = run(dev)
    assert torch.equal(seq, seq_b) and torch.equal(att, att_b) and torch.equal(logp, logp_b)
    pick = [0, 1, 17, 42, 55, 71, 98, 99]                        # spread over the batch (and both ends of it)
    sub = {k: v[pick].contiguous() for k, v in inp.items()}
    seq3, logp3, att3, _ = run({k: v.cuda() for k, v in sub.items()})
    assert torch.equal(seq3, seq[pick]) and torch.equal(att3, att[pick])
    oseq, ologp, oatt = O.sample_beam(sd, opt, sub, 3)
    assert torch.equal(seq3.cpu(), oseq) and torch.equal(att3.cpu(), oatt)
    assert _maxerr(logp3, ologp) <= TOL


def test_argument_validation_through_the_abi():
    opt, sd, inp = build_case(CASES["greedy_small_B5"])
    model = _model(opt, sd)
    _sample(model, inp)
    nm = model._native
    with pytest.raises(capi.GvdError, match="uint8|torch.uint8"):
        nm.decode_greedy(5, 7, inp["pnt_mask"].cuda().float())
    with pytest.raises(capi.GvdError, match="beam_size"):
        nm.beam_decode(5, 7, 1, inp["pnt_mask"].cuda())
    with pytest.raises(capi.GvdError, match="beam"):
        nm.beam_decode(5, 7, 99, inp["pnt_mask"].cuda())


def test_graph_replay_equals_kernel_by_kernel_enqueue():
    """gvd_decode_greedy replays the 20-step loop as ONE CUDA graph; with the stage profiler on it enqueues kernel by kernel.  Both
    must give the same bits (tokens, log-probs, attention logits), also on a second replay of the cached graph."""
    opt, sd, inp = build_case(CASES["greedy_T10_B4"])
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    dev = {k: inp[k].cuda() for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")}
    B, T = dev["segs_feat"].shape[0], dev["segs_feat"].shape[1]
    nm.prologue(*(dev[k] for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")))
    g1 = nm.decode_greedy(B, T, dev["pnt_mask"])
    g2 = nm.decode_greedy(B, T, dev["pnt_mask"])
    capi.profile_enable(True)
    try:
        d = nm.decode_greedy(B, T, dev["pnt_mask"])
    finally:
        capi.profile_enable(False)
        capi.profile_reset()
    torch.cuda.synchronize()
    for a, b, c in zip(g1, g2, d):
        assert torch.equal(a, c) and torch.equal(b, c)
