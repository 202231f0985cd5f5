"""transfer_mode 'none' on the device: every decode / teacher-forced / training entry point against the oracle (tests/region_feat_oracle.py)
and the reference's fixtures (tests/golden/region_feat_cases.py).  Bars as tests/test_gpu_parity.py: token ids and argmax indices
bit-exact, attention logits / log-probs / losses within 1e-4."""
import warnings

import numpy as np
import pytest
import torch

import gvd_oracle as O
import gvd_b200.synth as synth
import sample_ref as SR
from cases import build_case, load_fixture
from gvd_b200 import capi
from region_attn_oracle import oracle_modes
from region_feat_cases import REGION_FEAT_CASES as CASES
from region_feat_oracle import oracle_weights

pytestmark = pytest.mark.gpu
TOL = 1e-4
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


@pytest.fixture(autouse=True)
def _restore_backend():
    b = capi.get_backend()
    yield
    capi.set_backend(b)


def _maxerr(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


def _module(opt, sd):
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return m.cuda().eval()


_models = {}


def _case(name):
    """(opt, state_dict, oracle weights, inputs, module in eval mode), the module built once per case."""
    if name not in _models:
        opt, sd, inp = build_case(CASES[name])
        _models[name] = (opt, sd, oracle_weights(opt, sd), inp, _module(opt, sd))
    return _models[name]


def _greedy(model, inp, eval_opt=None):
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, logp, att2, sim = model._sample(*(dev[k] for k in KEYS), dict({"sample_max": 1, "beam_size": 1}, **(eval_opt or {})))
    torch.cuda.synchronize()
    return seq.cpu(), logp.cpu(), att2.cpu(), sim.cpu()


def _teacher(model, inp, mode):
    dev = {k: v.cuda() for k, v in inp.items()}
    with torch.no_grad():
        out = model(dev["segs_feat"], dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"],
                    dev["ppls_feat"], dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], mode)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------------------ decode entry points
@pytest.mark.parametrize("backend", [923, 3, 0])
@pytest.mark.parametrize("name", _names("greedy"))
def test_none_greedy_matches_oracle_and_reference(name, backend):
    """The three product paths of the step (923: split-K fp16x3 products, 3: tensor-core products, 0: CUDA-core products)."""
    capi.set_backend(backend)
    opt, sd, W, inp, model = _case(name)
    fx = load_fixture(name)
    seq, logp, att2, sim = _greedy(model, inp)
    with oracle_modes(opt):
        oseq, ologp, oatt2, osim = O.sample_greedy(W, opt, inp)
    assert torch.equal(seq, oseq) and np.array_equal(seq.numpy(), fx["seq"])
    assert _maxerr(logp, ologp) <= TOL and np.max(np.abs(logp.numpy() - fx["logp"])) <= TOL
    assert _maxerr(att2, oatt2) <= TOL and np.max(np.abs(att2.numpy() - fx["att2"])) <= TOL
    assert torch.equal(att2 == -1e8, oatt2 == -1e8)
    assert _maxerr(sim, osim) <= TOL


_MODES = [("featmap", "mix"), ("dual_region", "mix"), ("both", "mix_mul"), ("dual_region", "dp")]


@pytest.mark.parametrize("mode,form", _MODES, ids=["%s-%s" % m for m in _MODES])
def test_none_every_attention_mode_matches_oracle(mode, form):
    """'none' reaches every attention mode through the prologue and the grounding: greedy, the teacher-forced losses and the grounding
    indices of each (att_input_mode, region_attn_mode) against the oracle of that mode."""
    case = dict(CASES["none_mle_small_B5"], opt=dict(CASES["none_mle_small_B5"]["opt"], att_input_mode=mode, region_attn_mode=form))
    opt, sd, inp = build_case(case)
    W = oracle_weights(opt, sd)
    model = _module(opt, sd)
    seq, logp, att2, sim = _greedy(model, inp)
    with oracle_modes(opt):
        oseq, ologp, oatt2, osim = O.sample_greedy(W, opt, inp)
        olosses = O.forward_teacher(W, opt, inp)
        ocls, oatt_idx, ogrd_idx = O.forward_teacher(W, opt, inp, eval_obj_ground=True)
    assert torch.equal(seq, oseq)
    assert _maxerr(logp, ologp) <= TOL and _maxerr(att2, oatt2) <= TOL and _maxerr(sim, osim) <= TOL
    losses = _teacher(model, inp, "MLE")
    assert np.max(np.abs(np.array([float(l) for l in losses]) - np.array([float(l) for l in olosses]))) <= TOL
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    assert torch.equal(cls_pred.cpu(), ocls) and torch.equal(att_idx.cpu(), oatt_idx) and torch.equal(grd_idx.cpu(), ogrd_idx)


@pytest.mark.parametrize("name", _names("beam"))
def test_none_beam_matches_oracle_and_reference(name):
    case = CASES[name]
    opt, sd, W, inp, model = _case(name)
    fx = load_fixture(name)
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, logp, att, _ = model._sample(*(dev[k] for k in KEYS), {"beam_size": case["beam_size"]})
    torch.cuda.synchronize()
    oseq, ologp, oatt = O.sample_beam(W, opt, inp, case["beam_size"])
    assert torch.equal(seq.cpu(), oseq) and torch.equal(att.cpu(), oatt)
    assert np.array_equal(seq.cpu().numpy(), fx["seq"]) and np.array_equal(att.cpu().numpy(), fx["att2_idx"])
    assert np.max(np.abs(logp.cpu().numpy() - fx["logp"])) <= TOL


@pytest.mark.parametrize("name", _names("mle"))
def test_none_mle_losses_match_reference(name):
    opt, sd, W, inp, model = _case(name)
    got = np.array([float(l) for l in _teacher(model, inp, "MLE")])
    assert np.max(np.abs(got - load_fixture(name)["losses"])) <= TOL


@pytest.mark.parametrize("name", _names("grd"))
def test_none_grd_indices_match_reference(name):
    opt, sd, W, inp, model = _case(name)
    fx = load_fixture(name)
    cls_pred, att_idx, grd_idx = _teacher(model, inp, "GRD")
    assert np.array_equal(cls_pred.cpu().numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.cpu().numpy(), fx["att_idx"]) and np.array_equal(grd_idx.cpu().numpy(), fx["grd_idx"])


@pytest.mark.parametrize("backend", [923, 0])
def test_none_multinomial_matches_oracle(backend):
    """gvd_decode_sample against the oracle's multinomial loop with the same counter-based noise; the seed is the first whose oracle run has
    no near-tie (top-2 key gap < 1e-3) at any step."""
    capi.set_backend(backend)
    opt, sd, W, inp, model = _case("none_greedy_small_B5")
    B, T = inp["segs_feat"].shape[:2]
    tau = 0.8
    feats = O.prologue(W, opt, *(inp[k] for k in KEYS))
    for seed in range(1, 40):
        oseq, ologp, oatt2, _, gaps = SR.sample_multinomial(W, opt, inp, tau, SR.noise_fn(seed, np.arange(B), opt.vocab_size), feats=feats)
        if (gaps >= 1e-3).all():
            break
    else:
        pytest.fail("no seed without a near-tie")
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    seq, logp, att2 = (o.cpu() for o in nm.decode_sample(B, T, dev["pnt_mask"], seed, tau))
    assert torch.equal(seq, oseq)
    assert _maxerr(logp, ologp) <= TOL and _maxerr(att2, oatt2) <= TOL


def test_none_video_indexed_batch_equals_per_clip():
    """A video-indexed batch (one video per event) gives the per-clip results: greedy and beam."""
    opt, sd, W, inp, model = _case("none_greedy_small_B5")
    B = inp["ppls"].shape[0]
    vid = torch.arange(B, device="cuda")
    a = _greedy(model, inp)
    b = _greedy(model, inp, {"video_idx": vid})
    assert torch.equal(a[0], b[0]) and _maxerr(a[2], b[2]) <= 1e-5 and _maxerr(a[3], b[3]) <= 1e-5


@pytest.mark.parametrize("T", [10, 480])
def test_none_full_batch_sampled_clips_equal_oracle(T):
    """B = 100 clips at the full model dims: the decode of sampled clips against the oracle (token ids bit-exact, attention within 1e-4)."""
    opt = synth.make_opt(t_attn_size=T, transfer_mode="none")
    sd = synth.make_state_dict(opt, seed=11)
    inp = synth.make_inputs(opt, 100, seed=12)
    model = _module(opt, sd)
    seq, logp, att2, sim = _greedy(model, inp)
    W = oracle_weights(opt, sd)
    clips = [0, 37, 99] if T == 480 else [0, 13, 42, 77, 99]
    sub = {k: v[clips] for k, v in inp.items()}
    oseq, ologp, oatt2, osim = O.sample_greedy(W, opt, sub)
    assert torch.equal(seq[clips], oseq)
    assert _maxerr(logp[clips], ologp) <= TOL and _maxerr(att2[clips], oatt2) <= TOL and _maxerr(sim[clips], osim) <= TOL


@pytest.mark.parametrize("name", [n for n in _names("tfm_greedy") if not n.startswith("butd")])
def test_none_transformer_greedy_matches_oracle_and_reference(name):
    opt, sd, W, inp, model = _case(name)
    fx = load_fixture(name)
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, _, _ = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    oseq, _, _ = O.tfm_sample(W, opt, inp)
    assert torch.equal(seq.cpu(), oseq) and np.array_equal(seq.cpu().numpy(), fx["seq"])


# ------------------------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("mode", ["both", "dual_region"])
def test_none_training_step_against_oracle(mode):
    """Every gradient of the step (NativeOps) against autograd over the oracle; no gradient for a class bias the module does not have."""
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    case = CASES["none_train_small_B5"]
    opt, sd, inp = build_case(dict(case, opt=dict(case["opt"], att_input_mode=mode)))
    with oracle_modes(opt):
        losses, loss, grads, total_norm, new = O.train_step(oracle_weights(opt, sd), opt, inp)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    l2, loss2, g2, tn2, new2 = TrainStep(NativeOps()).step({k: v.cuda() for k, v in sd.items()}, opt, dev, host=inp)
    torch.cuda.synchronize()
    assert abs(float(loss2.cpu()) - float(loss)) <= TOL
    for a, b in zip(losses, l2):
        assert abs(float(a) - float(b.cpu())) <= TOL
    assert sorted(g2.keys()) == sorted(grads.keys()) and "vis_classifiers_bias" not in g2
    scale = float(total_norm)
    assert abs(tn2 - scale) <= 1e-4 * scale
    for k in grads:
        a, b = grads[k], g2[k].cpu().reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-6 * scale, k


def test_none_trainer_three_steps():
    """Trainer over NativeOps for three steps against the same Trainer over the torch mock (the flat segments follow the shorter state_dict);
    the tensors without a gradient come out bit-identical."""
    from gvd_b200.train import Trainer
    from gvd_b200.train_ops import NativeOps
    from ops_ref import TorchRefOps
    name = "none_train_small_B5"
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    a, b = Trainer(NativeOps(), sd, opt), Trainer(TorchRefOps(), sd, opt)
    assert a.keys == b.keys and "vis_classifiers_bias" not in a.keys
    for it in range(3):
        la, lossa = a.step(dev, host=inp)
        lb, lossb = b.step(inp)
        torch.cuda.synchronize()
        assert abs(float(lossa.cpu()) - float(lossb)) <= 1e-4 * (1 + 9 * it), it
        for k in a.keys:
            assert float((a.weights[k].cpu() - b.weights[k]).abs().max()) <= 2 * 5e-4 * (it + 1), (it, k)
    no_grad = set(str(k) for k in fx["no_grad_keys"])
    assert set(a.idle) == no_grad
    for k in no_grad:
        assert torch.equal(a.weights[k].cpu(), sd[k]), k


def test_none_dropout_masks_at_shared_sites_unchanged():
    """Train-mode dropout: the 'none' step draws the same masks as the 'cls' step at every site (they are keyed by seed, site and step, not
    by the order of the draws), so with the class bias set to zero both steps give the same losses and gradients."""
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    case = CASES["none_train_small_B5"]
    opt, sd, inp = build_case(case)
    opt_c = synth.make_opt(**dict(case["opt"], transfer_mode="cls"))
    sd_c = dict(vis_classifiers_bias=torch.zeros(opt.detect_size + 1), **sd)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    drop = dict(seed=99, p_lm=0.5, p_interact=0.2, p_gru=0.2, p_loc=0.5)
    out = []
    for o, s in ((opt, sd), (opt_c, sd_c)):
        ts = TrainStep(NativeOps())
        ts.dropout = drop
        out.append(ts.step({k: v.cuda() for k, v in s.items()}, o, dev, host=inp))
    torch.cuda.synchronize()
    (l1, _, g1, _, _), (l2, _, g2, _, _) = out
    for a, b in zip(l1, l2):
        assert torch.equal(a.cpu(), b.cpu())
    assert set(g2) - set(g1) == {"vis_classifiers_bias"}
    for k in g1:
        assert torch.equal(g1[k].cpu(), g2[k].cpu()), k


# ------------------------------------------------------------------------------------------------------------ enable_BUTD
from region_feat_oracle import oracle_region_feats  # noqa: E402


def _tfm_case(name):
    if name not in _models:
        opt, sd, inp = build_case(CASES[name])
        _models[name] = (opt, sd, oracle_weights(opt, sd), inp, _module(opt, sd))
    return _models[name]


@pytest.mark.parametrize("name", [n for n in _names("tfm_greedy") if n.startswith("butd")])
def test_butd_transformer_greedy_matches_oracle_and_reference(name):
    opt, sd, W, inp, model = _tfm_case(name)
    fx = load_fixture(name)
    dev = {k: inp[k].cuda() for k in KEYS}
    with torch.no_grad():
        seq, _, _ = model._sample(*(dev[k] for k in KEYS), {"sample_max": 1, "beam_size": 1})
    torch.cuda.synchronize()
    with oracle_region_feats():
        oseq, _, _ = O.tfm_sample(W, opt, inp)
        feats = O.prologue(W, opt, *(inp[k] for k in KEYS))
    assert torch.equal(seq.cpu(), oseq) and np.array_equal(seq.cpu().numpy(), fx["seq"])
    B, T = inp["segs_feat"].shape[:2]
    pool = model._native.workspace_tensor(B, T, "pool_feats", (B, model._native.R, opt.rnn_size))
    assert _maxerr(pool, feats["pool_feats"]) <= TOL


@pytest.mark.parametrize("name", _names("tfm_mle"))
def test_butd_transformer_teacher_loss_matches_reference(name):
    opt, sd, W, inp, model = _tfm_case(name)
    lm = _teacher(model, inp, "MLE")[0]
    assert abs(float(lm) - float(load_fixture(name)["losses"][0])) <= TOL


def test_butd_prologue_launches_no_pool_in_and_no_similarity():
    """The BUTD prologue (stage profiler): no region-embedding row kernel, and the similarity only when the caller asks for it."""
    opt, sd, W, inp, model = _tfm_case("butd_tfm_greedy_small_B3")
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    stages = {}
    for want in (False, True):
        capi.profile_enable(True)
        capi.profile_reset()
        sim = nm.prologue(*(dev[k] for k in KEYS), want_sim=want)
        torch.cuda.synchronize()
        stages[want] = capi.profile_read()
        capi.profile_enable(False)
        if want:
            with oracle_region_feats():
                osim = O.prologue(W, opt, *(inp[k] for k in KEYS))["sim_mat"]
            assert _maxerr(sim, osim) <= TOL
    assert "region.pool_embed" in stages[False] and "region.fc7" in stages[False]
    assert not any(s.startswith(("region.pool_in", "region.sim_")) for s in stages[False]), sorted(stages[False])
    assert "region.sim_gemm" in stages[True] and "region.pool_in" not in stages[True]


def test_butd_model_refuses_the_top_down_entry_points():
    opt, sd, W, inp, model = _tfm_case("butd_tfm_greedy_small_B3")
    nm = model._native_model()
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS), want_sim=False, beam=2)
    B, T = inp["segs_feat"].shape[:2]
    with pytest.raises(capi.GvdError, match="enable_BUTD"):
        nm.decode_greedy(B, T, dev["pnt_mask"])
    with pytest.raises(capi.GvdError, match="enable_BUTD"):
        nm.beam_decode(B, T, 2, dev["pnt_mask"])


@pytest.mark.parametrize("name", _names("tfm_train"))
def test_butd_training_step_against_oracle(name):
    """Every gradient of the BUTD step (NativeOps) against autograd over the oracle; loc_fc, vis_embed and the class bias get none."""
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    from make_golden_tfm_train import build_tfm_case
    from tfm_train_ref import tfm_train_step
    opt, sd, inp = build_tfm_case(CASES[name])
    with oracle_region_feats():
        lm, loss, grads, total_norm, new = tfm_train_step(oracle_weights(opt, sd), opt, inp)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    l2, loss2, g2, tn2, new2 = TrainStep(NativeOps()).step({k: v.cuda() for k, v in sd.items()}, opt, dev, host=inp)
    torch.cuda.synchronize()
    assert abs(float(loss2.cpu()) - float(loss)) <= TOL
    assert sorted(g2) == sorted(grads) and not any(k.startswith(("loc_fc.", "vis_embed.")) for k in g2)
    scale = float(total_norm)
    assert abs(tn2 - scale) <= 1e-4 * scale
    for k in grads:
        a, b = grads[k], g2[k].cpu().reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-6 * scale, k


def test_butd_trainer_three_steps():
    """Trainer over NativeOps for three steps against the torch mock; loc_fc, vis_embed and the class bias stay bit-identical (lr 0)."""
    from gvd_b200.train import Trainer
    from gvd_b200.train_ops import NativeOps
    from make_golden_tfm_train import build_tfm_case
    from tfm_train_ref import TfmRefOps
    opt, sd, inp = build_tfm_case(CASES["butd_tfm_train_small_B3"])
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    a, b = Trainer(NativeOps(), sd, opt), Trainer(TfmRefOps(), sd, opt)
    for it in range(3):
        la, lossa = a.step(dev, host=inp)
        lb, lossb = b.step(inp)
        torch.cuda.synchronize()
        assert abs(float(lossa.cpu()) - float(lossb)) <= 1e-4 * (1 + 9 * it), it
        for k in a.keys:
            assert float((a.weights[k].cpu() - b.weights[k]).abs().max()) <= 2 * 5e-4 * (it + 1), (it, k)
    untouched = [k for k in a.keys if k.startswith(("loc_fc.", "vis_embed.", "vis_classifiers_bias"))]
    assert untouched and set(untouched) <= set(a.idle)
    for k in untouched:
        assert torch.equal(a.weights[k].cpu(), sd[k]), k
