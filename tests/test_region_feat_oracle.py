"""transfer_mode 'none' and enable_BUTD on the CPU: the oracle (tests/region_feat_oracle.py) against the unmodified reference's outputs
(tests/golden/region_feat_cases.py, make_golden_region_feat.py), the training step's orchestration (gvd_b200/train.py over the torch mock of
its primitives) against autograd over the oracle, the state_dict against the reference's, and the option surface.  Same bars as
tests/test_oracle_golden.py."""
import warnings

import numpy as np
import pytest
import torch

import gvd_oracle as O
from cases import build_case, load_fixture, subsample
from gvd_b200 import capi
import gvd_b200.synth as synth
from region_attn_oracle import oracle_modes
from region_feat_cases import BUTD_KEYS_FIXTURE, NONE_KEYS_FIXTURE, REGION_FEAT_CASES as CASES
from region_feat_oracle import oracle_region_feats, oracle_weights

TOL = 1e-4


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol, np.max(np.abs(a - b))


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


def _case(name):
    opt, sd, inp = build_case(CASES[name])
    assert "vis_classifiers_bias" not in sd
    return opt, sd, oracle_weights(opt, sd), inp


@pytest.mark.parametrize("name", _names("greedy"))
def test_none_greedy_matches_reference(name):
    opt, sd, W, inp = _case(name)
    fx = load_fixture(name)
    with oracle_modes(opt):
        feats = O.prologue(W, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
        for k in ("fc_feats", "g_pool", "pool_embed", "p_pool_feats", "p_conv_feats"):
            _close(subsample(k, feats[k]).numpy(), fx[k])
        seq, logp, att2, sim = O.sample_greedy(W, opt, inp, feats=feats)
    assert fx["min_margin"] > TOL
    assert np.array_equal(seq.numpy(), fx["seq"])
    _close(logp.numpy(), fx["logp"])
    _close(att2.numpy(), fx["att2"])
    _close(subsample("sim_mat", sim).numpy(), fx["sim_mat"])


def test_none_changes_the_similarity():
    """The fixtures would also pass with the class bias of the 'cls' weights only if that bias did not change the similarity."""
    name = "none_greedy_small_B5"
    opt, sd, W, inp = _case(name)
    cls = dict(W, vis_classifiers_bias=synth.make_state_dict(synth.make_opt(**dict(CASES[name]["opt"], transfer_mode="cls")),
                                                             seed=CASES[name]["weight_seed"])["vis_classifiers_bias"])
    _, _, _, sim = O.sample_greedy(cls, opt, inp)
    assert np.max(np.abs(subsample("sim_mat", sim).numpy() - load_fixture(name)["sim_mat"])) > 1e-3


@pytest.mark.parametrize("name", _names("mle"))
def test_none_mle_losses_match_reference(name):
    opt, sd, W, inp = _case(name)
    losses = O.forward_teacher(W, opt, inp)
    _close(np.array([float(x) for x in losses]), load_fixture(name)["losses"])


@pytest.mark.parametrize("name", _names("grd"))
def test_none_grd_indices_match_reference(name):
    opt, sd, W, inp = _case(name)
    fx = load_fixture(name)
    cls_pred, att_idx, grd_idx = O.forward_teacher(W, opt, inp, eval_obj_ground=True)
    assert np.array_equal(cls_pred.numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.numpy(), fx["att_idx"]) and np.array_equal(grd_idx.numpy(), fx["grd_idx"])


@pytest.mark.parametrize("name", _names("beam"))
def test_none_beam_matches_repaired_reference(name):
    opt, sd, W, inp = _case(name)
    fx = load_fixture(name)
    seq, logp, att = O.sample_beam(W, opt, inp, CASES[name]["beam_size"])
    assert np.array_equal(seq.numpy(), fx["seq"]) and np.array_equal(att.numpy(), fx["att2_idx"])
    _close(logp.numpy(), fx["logp"])


@pytest.mark.parametrize("name", _names("train"))
def test_none_train_step_matches_reference(name):
    """Losses, the set of tensors that receive a gradient (no vis_classifiers_bias), gradient norms / leading entries, the first Adam update."""
    opt, sd, W, inp = _case(name)
    fx = load_fixture(name)
    losses, loss, grads, total_norm, new = O.train_step(W, opt, inp)
    _close(np.array([float(x) for x in losses]), fx["losses"])
    assert abs(float(loss) - float(fx["loss"])) <= TOL
    keys = [str(k) for k in fx["keys"]]
    assert sorted(grads.keys()) == keys and "vis_classifiers_bias" not in keys and "vis_embed.0.weight" in keys
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
def test_none_train_step_orchestration_matches_oracle(name):
    """gvd_b200/train.py's forward tape and explicit backward (on the CPU over the torch mock of its primitives) against autograd over the
    oracle: same gradient set, every gradient elementwise."""
    from gvd_b200.train import TrainStep
    from ops_ref import TorchRefOps
    opt, sd, W, inp = _case(name)
    losses, loss, grads, total_norm, new = O.train_step(W, opt, inp)
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


def test_none_trainer_flat_segments_follow_the_state_dict():
    """Trainer over the 'none' state_dict: one segment per float entry (no class bias), two steps move the trained tensors and leave the
    ones without a gradient (core.i2h_2 / h2h_2) bit-identical."""
    from gvd_b200.train import Trainer
    from ops_ref import TorchRefOps
    opt, sd, W, inp = _case("none_train_small_B5")
    tr = Trainer(TorchRefOps(), sd, opt)
    assert tr.keys == [k for k, v in sd.items() if v.is_floating_point() and "running_" not in k]
    for _ in range(2):
        tr.step(inp)
    assert tr.idle and all(k.startswith(("core.i2h_2", "core.h2h_2")) for k in tr.idle)
    for k in tr.idle:
        assert torch.equal(tr.weights[k], sd[k]), k
    assert not torch.equal(tr.weights["vis_embed.0.weight"], sd["vis_embed.0.weight"])


def test_none_state_dict_matches_reference_keys():
    """TopDownModel(opt) with transfer_mode 'none': the reference's keys, order and shapes (fixture from the unmodified reference), the
    synthetic state_dict alike, and the 'cls' list without its first entry, vis_classifiers_bias."""
    from gvd_b200.misc.AttModel import TopDownModel
    fx = load_fixture(NONE_KEYS_FIXTURE)
    ref = list(zip((str(k) for k in fx["keys"]), (str(s) for s in fx["shapes"])))
    opt = synth.make_opt(t_attn_size=10, transfer_mode="none")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    assert not hasattr(m, "vis_classifiers_bias")
    got = [(k, ",".join(str(n) for n in v.shape)) for k, v in m.state_dict().items()]
    assert got == ref
    sd = synth.make_state_dict(opt)
    assert [(k, ",".join(str(n) for n in v.shape)) for k, v in sd.items()] == ref
    m.load_state_dict(sd, strict=True)
    cls_sd = synth.make_state_dict(synth.make_opt(t_attn_size=10))
    assert list(cls_sd)[0] == "vis_classifiers_bias" and [k for k, _ in ref] == list(cls_sd)[1:]
    assert all(torch.equal(cls_sd[k], sd[k]) for k in sd)


def test_none_transfers_fc7_only(tmp_path, monkeypatch):
    """_init_from_detectron with transfer_mode 'none' copies fc7 into ctx2pool_grd and leaves vis_embed at its default init
    (model.py:172-178,214-215); 'cls' overwrites vis_embed with the matched detector classes."""
    import pickle
    from gvd_b200.misc.AttModel import TopDownModel
    kw = dict(vocab_size=301, detect_size=30, input_encoding_size=64, rnn_size=248, att_hid_size=96, seq_length=9, num_sampled_frm=4,
              num_prop_per_frm=13, t_attn_size=7, n_vg_cls=64)
    opt = synth.make_opt(transfer_mode="none", **kw)
    det = synth.make_detectron(opt)
    d = tmp_path / "data" / "detectron_weights"
    d.mkdir(parents=True)
    for k, v in det.items():
        with open(d / (k + ".pkl"), "wb") as f:
            pickle.dump(v, f)
    monkeypatch.chdir(tmp_path)
    torch.manual_seed(0)
    m = TopDownModel(opt)
    assert torch.equal(m.ctx2pool_grd[0].weight[:2048], torch.from_numpy(det["fc7_w"]))
    torch.manual_seed(0)
    c = TopDownModel(synth.make_opt(**kw))
    assert torch.equal(c.vis_embed[0].weight[0], torch.from_numpy(det["cls_score_w"][0]))
    assert not torch.equal(m.vis_embed[0].weight[0], torch.from_numpy(det["cls_score_w"][0]))


def test_transfer_mode_option_surface():
    """'none' is accepted for both captioners and every attention mode; 'glove' / 'both' and enable_BUTD raise with their reasons."""
    for extra in ({}, dict(att_input_mode="featmap"), dict(att_input_mode="dual_region"), dict(region_attn_mode="dp"),
                  dict(region_attn_mode="mix_mul"), dict(att_model="transformer"), dict(att_model="transformer", att_input_mode="region")):
        opt = synth.make_opt(transfer_mode="none", **extra)
        assert bytes(capi.dims_from_opt(opt)) == bytes(capi.dims_from_opt(synth.make_opt(**extra)))
        assert capi.transfer_mode_code(opt) == 1
    assert capi.transfer_mode_code(synth.make_opt()) == 0
    for bad, why in (("glove", "model.py:88-89,158,177"), ("both", "model.py:86-87,70,370"), ("x", "implemented")):
        with pytest.raises(NotImplementedError, match=why):
            capi.dims_from_opt(synth.make_opt(transfer_mode=bad))
    with pytest.raises(ValueError, match="model.py:66"):
        capi.dims_from_opt(synth.make_opt(enable_BUTD=True))
    with pytest.raises(ValueError, match="model.py:66"):
        capi.dims_from_opt(synth.make_opt(enable_BUTD=True, att_model="transformer", att_input_mode="featmap"))
    with pytest.raises(NotImplementedError, match="top-down captioner does not run"):
        capi.dims_from_opt(synth.make_opt(enable_BUTD=True, att_input_mode="region"))
    for mode in ("cls", "none"):
        opt = synth.make_opt(enable_BUTD=True, att_model="transformer", att_input_mode="region", transfer_mode=mode)
        assert bytes(capi.dims_from_opt(opt)) == bytes(capi.dims_from_opt(synth.make_opt(att_model="transformer", att_input_mode="region")))
        assert capi.att_input_mode_code(opt) == capi.ATT_INPUT_REGION == 3
    assert capi.att_input_mode_code(synth.make_opt(att_model="transformer", att_input_mode="region")) == 0
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(synth.make_opt(transfer_mode="none", t_attn_size=10))
    assert m._opt_view().transfer_mode == "none"


# ------------------------------------------------------------------------------------------------------------ enable_BUTD
@pytest.mark.parametrize("name", _names("tfm_greedy"))
def test_transformer_greedy_matches_reference(name):
    """The transformer captioner in 'none' and in 'region' + BUTD (with 'cls' and 'none'): ids bit-exact, the step logits within 1e-4."""
    opt, sd, W, inp = (lambda o, s, i: (o, s, oracle_weights(o, s), i))(*build_case(CASES[name]))
    fx = load_fixture(name)
    with oracle_region_feats():
        seq, _, _, trace = O.tfm_sample(W, opt, inp, return_trace=True)
    assert fx["min_margin"] > TOL
    assert np.array_equal(seq.numpy(), fx["seq"])
    _close(subsample("tfm_logits", torch.stack(trace[:opt.seq_length], 1)).numpy(), fx["tfm_logits"])


def test_butd_changes_the_region_features():
    """The BUTD fixture would also pass with the non-BUTD region embedding only if the region features did not reach the captions."""
    name = "butd_tfm_greedy_small_B3"
    opt, sd, inp = build_case(CASES[name])
    with oracle_region_feats():
        feats = O.prologue(sd, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    g = feats["g_pool"]
    assert torch.allclose(feats["pool_embed"], torch.relu(g @ sd["pool_embed.0.weight"].t() + sd["pool_embed.0.bias"]), atol=1e-6)
    assert tuple(sd["pool_embed.0.weight"].shape) == (opt.rnn_size, 2048)


@pytest.mark.parametrize("name", _names("tfm_mle"))
def test_butd_teacher_forced_loss_matches_reference(name):
    opt, sd, inp = build_case(CASES[name])
    with oracle_region_feats():
        lm = O.tfm_mle(oracle_weights(opt, sd), opt, inp)
    assert abs(float(lm) - float(load_fixture(name)["losses"][0])) <= TOL


@pytest.mark.parametrize("name", _names("tfm_train"))
def test_butd_train_specification_matches_reference(name):
    """tests/tfm_train_ref.tfm_train_step over the BUTD oracle against the reference's step: loss, norm, the gradient set (no loc_fc, vis_embed
    or class bias), gradients and the first Adam update."""
    from make_golden_tfm_train import build_tfm_case, sub
    from tfm_train_ref import tfm_train_step
    opt, sd, inp = build_tfm_case(CASES[name])
    fx = load_fixture(name)
    with oracle_region_feats():
        lm, loss, grads, total_norm, new = tfm_train_step(oracle_weights(opt, sd), opt, inp)
    assert abs(float(lm) - float(fx["lm"])) <= 1e-4
    assert abs(float(total_norm) - float(fx["total_norm"])) <= 1e-3 * float(fx["total_norm"])
    keys = [str(k) for k in fx["keys"]]
    assert sorted(grads) == keys
    assert not any(k.startswith(("loc_fc.", "vis_embed.", "vis_classifiers_bias")) for k in keys) and "pool_embed.0.weight" in keys
    for i, k in enumerate(keys):
        gmax = float(fx["grad_max"][i])
        assert abs(float(grads[k].abs().max()) - gmax) <= 1e-4 * gmax + 1e-12, k
        assert np.max(np.abs(sub(grads[k]).numpy() - fx["grad_sub"][i][:sub(grads[k]).numel()])) <= 1e-4 * gmax + 1e-12, k
        upd = sub(new[k] - sd[k]).numpy()
        ref = fx["update_sub"][i][:upd.size]
        assert np.linalg.norm(upd - ref) <= 5e-3 * np.linalg.norm(ref) + 1e-9 or gmax <= 1e-6 * float(fx["total_norm"]), k


@pytest.mark.parametrize("name", _names("tfm_train"))
def test_butd_train_orchestration_matches_specification(name):
    """gvd_b200/train.py's BUTD forward tape and backward (pool_embed straight into fc7's ReLU / Dropout) over the torch mock of its
    primitives against autograd over the oracle."""
    from gvd_b200.train import TrainStep
    from make_golden_tfm_train import build_tfm_case
    from tfm_train_ref import TfmRefOps, tfm_train_step
    opt, sd, inp = build_tfm_case(CASES[name])
    with oracle_region_feats():
        lm, loss, grads, total_norm, new = tfm_train_step(oracle_weights(opt, sd), opt, inp)
    losses, loss2, g2, tn2, new2 = TrainStep(TfmRefOps()).step(sd, opt, inp)
    assert abs(float(loss2) - float(loss)) <= 1e-5
    assert abs(tn2 - float(total_norm)) <= 1e-5 * float(total_norm)
    assert sorted(g2) == sorted(grads)
    scale = float(total_norm)
    for k in grads:
        a, b = grads[k], g2[k].reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 5e-5 * float(a.abs().max()) + 1e-7 * scale, k


def test_butd_state_dict_matches_reference_keys():
    """The transformer captioner with 'region' + BUTD: the reference's keys, order and shapes, pool_embed.0.weight [H, 2048], loc_fc.* kept;
    the synthetic state_dict alike; strict load."""
    from gvd_b200.misc.AttModel import TopDownModel
    fx = load_fixture(BUTD_KEYS_FIXTURE)
    ref = list(zip((str(k) for k in fx["keys"]), (str(s) for s in fx["shapes"])))
    opt = synth.make_opt(t_attn_size=10, att_model="transformer", att_input_mode="region", enable_BUTD=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    got = [(k, ",".join(str(n) for n in v.shape)) for k, v in m.state_dict().items()]
    assert got == ref
    assert dict(ref)["pool_embed.0.weight"] == "1024,2048" and "loc_fc.0.weight" in dict(ref)
    sd = synth.make_state_dict(opt)
    assert [(k, ",".join(str(n) for n in v.shape)) for k, v in sd.items()] == ref
    m.load_state_dict(sd, strict=True)
