"""att_input_mode 'featmap' and 'dual_region' of the top-down captioner on the CPU: the oracle's steps of both modes
(tests/input_mode_oracle.py) against the unmodified reference's outputs (tests/golden/input_mode_cases.py, make_golden_input_mode.py), the training step's orchestration (gvd_b200/train.py over
the torch mock of its primitives) against the oracle, and the option surface.  Same bars as tests/test_oracle_golden.py."""
import warnings

import numpy as np
import pytest
import torch

from cases import build_case, load_fixture, subsample
from gvd_b200 import capi
import gvd_b200.synth as synth
from input_mode_cases import DUAL_KEYS_FIXTURE, INPUT_MODE_CASES as CASES
from input_mode_oracle import oracle_mode

TOL = 1e-4
REGION_BRANCH = ("core.attention2.", "ctx2pool.", "pool_embed.", "loc_fc.", "obj_interact.")
FRAME_BRANCH = ("att_embed.", "att_embed_aux.", "context_enc.", "ctx2att.", "core.attention.")


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol, np.max(np.abs(a - b))


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


@pytest.mark.parametrize("name", _names("greedy"))
def test_input_mode_greedy_matches_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_mode(opt) as O:
        feats = O.prologue(sd, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
        for k in ("fc_feats", "p_pool_feats", "p_conv_feats"):
            if k in fx:                                   # (dual_region: the reference never computes p_conv_feats)
                _close(subsample(k, feats[k]).numpy(), fx[k])
        seq, logp, att2, sim = O.sample_greedy(sd, opt, inp, feats=feats)
    assert fx["min_margin"] > TOL
    assert np.array_equal(seq.numpy(), fx["seq"])
    _close(logp.numpy(), fx["logp"])
    _close(att2.numpy(), fx["att2"])
    _close(subsample("sim_mat", sim).numpy(), fx["sim_mat"])


@pytest.mark.parametrize("name", ["featmap_greedy_small_B5", "dual_greedy_small_B5"])
def test_input_mode_changes_the_decode(name):
    """The fixtures would also pass with an oracle that ignored the mode only if the mode did not change the captions."""
    opt, sd, inp = build_case(CASES[name])
    import gvd_oracle as O
    seq_both, _, att2_both, _ = O.sample_greedy(sd, opt, inp)
    fx = load_fixture(name)
    assert not np.array_equal(seq_both.numpy(), fx["seq"]) or np.max(np.abs(att2_both.numpy() - fx["att2"])) > 1e-2


@pytest.mark.parametrize("name", _names("mle"))
def test_input_mode_mle_losses_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    with oracle_mode(opt) as O:
        losses = O.forward_teacher(sd, opt, inp)
    _close(np.array([float(x) for x in losses]), load_fixture(name)["losses"])


@pytest.mark.parametrize("name", _names("grd"))
def test_input_mode_grd_indices_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_mode(opt) as O:
        cls_pred, att_idx, grd_idx = O.forward_teacher(sd, opt, inp, eval_obj_ground=True)
    assert np.array_equal(cls_pred.numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.numpy(), fx["att_idx"]) and np.array_equal(grd_idx.numpy(), fx["grd_idx"])


@pytest.mark.parametrize("name", _names("beam"))
def test_input_mode_beam_matches_repaired_reference(name):
    case = CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    with oracle_mode(opt) as O:
        seq, logp, att = O.sample_beam(sd, opt, inp, case["beam_size"])
    assert np.array_equal(seq.numpy(), fx["seq"]) and np.array_equal(att.numpy(), fx["att2_idx"])
    _close(logp.numpy(), fx["logp"])


@pytest.mark.parametrize("name", _names("train"))
def test_input_mode_train_step_matches_reference(name):
    """Losses, the set of tensors that receive a gradient, per-tensor gradient norms / leading entries and the first Adam update."""
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_mode(opt) as O:
        losses, loss, grads, total_norm, new = O.train_step(sd, opt, inp)
    _close(np.array([float(x) for x in losses]), fx["losses"])
    assert abs(float(loss) - float(fx["loss"])) <= TOL
    keys = [str(k) for k in fx["keys"]]
    assert sorted(grads.keys()) == keys
    no_grad = set(str(k) for k in fx["no_grad_keys"])
    if opt.att_input_mode == "featmap" and not (opt.w_att2 or opt.w_grd):
        region = {k for k in sd if k.startswith(REGION_BRANCH) and "running" not in k}
        assert region and region <= no_grad                       # the reference gives the whole region branch no gradient
    if opt.att_input_mode == "dual_region":
        frame = {k for k in sd if k.startswith(FRAME_BRANCH) and sd[k].is_floating_point() and "running" not in k}
        assert frame and frame <= no_grad                         # no frame branch, no temporal attention
        assert {"core.dual_pointer.0.weight", "core.attention2_dual.h2att.weight"} <= set(keys)
    assert abs(float(total_norm) - float(fx["total_norm"])) <= 1e-3 * float(fx["total_norm"])
    scale = float(fx["total_norm"])
    for i, k in enumerate(keys):
        assert abs(float(grads[k].norm()) - fx["grad_norm"][i]) <= 1e-3 * fx["grad_norm"][i] + 1e-6 * scale, k
        head = np.resize(grads[k].flatten()[:8].numpy(), 8)
        assert np.max(np.abs(head - fx["grad_head"][i])) <= 1e-3 * np.max(np.abs(fx["grad_head"][i])) + 1e-6 * scale, k
        if fx["grad_norm"][i] > 1e-6 * scale:
            un = float((new[k] - sd[k]).norm())
            assert abs(un - fx["update_norm"][i]) <= 5e-3 * fx["update_norm"][i] + 1e-9, k


@pytest.mark.parametrize("name", _names("train"))
def test_input_mode_train_step_orchestration_matches_oracle(name):
    """gvd_b200/train.py's forward tape and explicit backward (run on the CPU over the torch mock of its primitives) against
    autograd over the oracle: same gradient set, every gradient elementwise."""
    from gvd_b200.train import TrainStep
    from ops_ref import TorchRefOps
    opt, sd, inp = build_case(CASES[name])
    with oracle_mode(opt) as O:
        losses, loss, grads, total_norm, new = O.train_step(sd, opt, inp)
    l2, loss2, g2, tn2, new2 = TrainStep(TorchRefOps()).step(sd, opt, inp)
    assert abs(float(loss2) - float(loss)) <= 1e-5
    for a, b in zip(losses, l2):
        assert abs(float(a) - float(b)) <= 1e-5
    assert sorted(g2.keys()) == sorted(grads.keys())
    scale = float(total_norm)
    assert abs(tn2 - scale) <= 1e-5 * scale
    for k in grads:
        a, b = grads[k], g2[k].reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max()) + 1e-7 * scale, k


def test_featmap_trainer_leaves_the_region_branch_untouched():
    """Trainer's rule for tensors without a gradient (lr 0) reproduces torch.optim.Adam skipping them: with w_att2 = w_grd = 0 the region
    branch comes out of two steps bit-identical, and the idle set is the reference's no-gradient set."""
    from gvd_b200.train import Trainer
    from ops_ref import TorchRefOps
    name = "featmap_train_small_w0"
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    tr = Trainer(TorchRefOps(), sd, opt)
    for _ in range(2):
        tr.step(inp)
    no_grad = set(str(k) for k in fx["no_grad_keys"])
    assert set(tr.idle) == no_grad
    for k in no_grad:
        assert torch.equal(tr.weights[k], sd[k]), k
    assert any(not torch.equal(tr.weights[k], sd[k]) for k in tr.keys if k not in no_grad)


def test_dual_region_trainer_keeps_the_frame_branch_and_batchnorm_statistics():
    """dual_region never runs the frame branch: two Trainer steps leave its parameters and att_embed_aux's running statistics as they were;
    the idle set is the reference's no-gradient set; the gate and the second attention train."""
    from gvd_b200.train import Trainer
    from ops_ref import TorchRefOps
    name = "dual_train_small_B5"
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    tr = Trainer(TorchRefOps(), sd, opt)
    for _ in range(2):
        tr.step(inp)
    no_grad = set(str(k) for k in fx["no_grad_keys"])
    assert set(tr.idle) == no_grad
    for k in no_grad:
        assert torch.equal(tr.weights[k], sd[k]), k
    for k in ("att_embed_aux.0.running_mean", "att_embed_aux.0.running_var", "att_embed_aux.0.num_batches_tracked"):
        assert torch.equal(tr.buffers[k], sd[k]), k
    for k in ("core.dual_pointer.0.weight", "core.attention2_dual.alpha_net.weight"):
        assert not torch.equal(tr.weights[k], sd[k]), k


def test_dual_region_gate_varies():
    """The synthetic weights give a gate that really mixes the two attentions: g spans a wide range across clips and steps."""
    opt, sd, inp = build_case(CASES["dual_greedy_small_B5"])
    import input_mode_oracle as IM
    gs = []
    orig = IM.core_step_dual_region

    def tap(W, xt, feats, att_mask, pnt_mask, state):
        out = orig(W, xt, feats, att_mask, pnt_mask, state)
        gs.append(torch.sigmoid(IM.O._lin(out[1][0][0], W, "core.dual_pointer.0")))
        return out
    IM.STEPS["dual_region"] = tap
    try:
        with oracle_mode(opt) as O:
            O.sample_greedy(sd, opt, inp)
    finally:
        IM.STEPS["dual_region"] = orig
    g = torch.cat(gs)
    assert float(g.min()) < 0.25 and float(g.max()) > 0.75, (float(g.min()), float(g.max()))


def test_dual_region_state_dict_matches_reference_keys():
    """TopDownModel(opt) in dual_region: the reference's keys, order and shapes (fixture from the unmodified reference), the synthetic
    state_dict alike, and the native parameter list is the state_dict's float entries minus the BatchNorm buffers."""
    from gvd_b200.misc.AttModel import TopDownModel
    fx = load_fixture(DUAL_KEYS_FIXTURE)
    ref = list(zip((str(k) for k in fx["keys"]), (str(s) for s in fx["shapes"])))
    opt = synth.make_opt(t_attn_size=10, att_input_mode="dual_region")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    got = [(k, ",".join(str(n) for n in v.shape)) for k, v in m.state_dict().items()]
    assert got == ref
    sd = synth.make_state_dict(opt)
    assert [(k, ",".join(str(n) for n in v.shape)) for k, v in sd.items()] == ref
    m.load_state_dict(sd, strict=True)
    base = [k for k in synth.make_state_dict(synth.make_opt(t_attn_size=10)).keys()]
    assert [k for k, _ in ref if not k.startswith(("core.attention2_dual.", "core.dual_pointer."))] == base
    both_sd = synth.make_state_dict(synth.make_opt(t_attn_size=10))
    assert all(torch.equal(both_sd[k], sd[k]) for k in base)          # adding the mode's tensors leaves every other one as it was


def test_option_surface():
    """'featmap' and 'dual_region' are accepted for the top-down captioner; 'region' and unknown values still raise."""
    from gvd_b200.misc.AttModel import TopDownModel
    both, fm = synth.make_opt(), synth.make_opt(att_input_mode="featmap")
    assert bytes(capi.dims_from_opt(both)) == bytes(capi.dims_from_opt(fm))
    assert capi.att_input_mode_code(both) == 0 and capi.att_input_mode_code(fm) == 1
    assert capi.att_input_mode_code(synth.make_opt(att_input_mode="dual_region")) == 2
    for bad in ("region", "x"):
        with pytest.raises(NotImplementedError):
            capi.dims_from_opt(synth.make_opt(att_input_mode=bad))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(fm)
    sd = synth.make_state_dict(fm)
    assert list(m.state_dict().keys()) == list(synth.make_state_dict(both).keys()) == list(sd.keys())
    m.load_state_dict(sd, strict=True)
    assert m._opt_view().att_input_mode == "featmap"
