"""region_attn_mode 'dp' and 'mix_mul' of the top-down captioner on the CPU: the oracle's steps (tests/region_attn_oracle.py) against the
unmodified reference's outputs (tests/golden/region_attn_cases.py, make_golden_region_attn.py), the training step's orchestration
(gvd_b200/train.py over the torch mock of its primitives) against the oracle, the state_dict key lists, the option surface, and an index
emulation of the new training kernels.  Same bars as tests/test_oracle_golden.py."""
import warnings

import numpy as np
import pytest
import torch

from cases import build_case, load_fixture, subsample
from gvd_b200 import capi
import gvd_b200.synth as synth
from region_attn_cases import DP_KEYS_FIXTURES, REGION_ATTN_CASES as CASES
from region_attn_oracle import RegionAttnRefOps, oracle_modes

TOL = 1e-4


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol, np.max(np.abs(a - b))


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


@pytest.mark.parametrize("name", _names("greedy"))
def test_region_attn_greedy_matches_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_modes(opt) as O:
        feats = O.prologue(sd, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
        for k in ("fc_feats", "p_pool_feats", "p_conv_feats"):
            if k in fx:                                   # (dual_region: the reference never computes p_conv_feats)
                _close(subsample(k, feats[k]).numpy(), fx[k])
        seq, logp, att2, sim = O.sample_greedy(sd, opt, inp, feats=feats)
    # the chosen token leads the runner-up by more than the parity tolerance at every step, so bit-exact ids are a fair demand on the GPU
    assert fx["min_margin"] > TOL, fx["min_margin"]
    assert np.array_equal(seq.numpy(), fx["seq"])
    _close(logp.numpy(), fx["logp"])
    _close(att2.numpy(), fx["att2"], tol=TOL * max(1.0, float(np.abs(fx["att2"][fx["att2"] > -1e7]).max())))
    _close(subsample("sim_mat", sim).numpy(), fx["sim_mat"])


@pytest.mark.parametrize("name", ["dp_greedy_small_B5", "mul_greedy_small_B5", "dp_dual_greedy_small_B5", "mul_dual_greedy_small_B5"])
def test_region_attn_changes_the_decode(name):
    """The fixtures would also pass with an oracle that ignored the form only if the form did not change the region logits: the same
    clips and weights ('mix' adds the region alpha_net) give other logits in 'mix'."""
    case = CASES[name]
    opt, sd, inp = build_case(dict(case, opt=dict(case["opt"], region_attn_mode="mix")))
    with oracle_modes(opt) as O:
        _, _, att2_mix, _ = O.sample_greedy(sd, opt, inp)
    assert np.max(np.abs(att2_mix.numpy() - load_fixture(name)["att2"])) > 1e-2


@pytest.mark.parametrize("name", _names("beam"))
def test_region_attn_beam_matches_repaired_reference(name):
    case = CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    with oracle_modes(opt) as O:
        seq, logp, att = O.sample_beam(sd, opt, inp, case["beam_size"])
    assert np.array_equal(seq.numpy(), fx["seq"]) and np.array_equal(att.numpy(), fx["att2_idx"])
    _close(logp.numpy(), fx["logp"])


@pytest.mark.parametrize("name", _names("beam"))
def test_region_attn_beam_keeps_a_margin(name):
    """At every core step of the beam search the returned region argmax (att2_idx) leads its runner-up by more than the parity tolerance,
    and so does each row's K-th best next word over its (K+1)-th, so the GPU must reproduce the ids exactly."""
    case = CASES[name]
    opt, sd, inp = build_case(case)
    K = case["beam_size"]
    zgaps, gaps = [], []
    with oracle_modes(opt) as O:
        step = O.core_step

        def tap(W, xt, feats, att_mask, pnt_mask, state):
            out = step(W, xt, feats, att_mask, pnt_mask, state)
            top = torch.topk(out[2], 2, dim=1).values
            zgaps.append(top[:, 0] - top[:, 1])
            v = torch.topk(torch.log_softmax(O._lin(out[0], W, "logit"), dim=1), K + 1, dim=1).values
            gaps.append(v[:, K - 1] - v[:, K])
            return out
        O.core_step = tap
        O.sample_beam(sd, opt, inp, K)
    assert float(torch.cat(zgaps).min()) > TOL
    assert float(torch.cat(gaps).min()) > TOL


@pytest.mark.parametrize("name", _names("mle"))
def test_region_attn_mle_losses_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    with oracle_modes(opt) as O:
        losses = O.forward_teacher(sd, opt, inp)
    _close(np.array([float(x) for x in losses]), load_fixture(name)["losses"])


@pytest.mark.parametrize("name", _names("grd"))
def test_region_attn_grd_indices_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_modes(opt) as O:
        cls_pred, att_idx, grd_idx = O.forward_teacher(sd, opt, inp, eval_obj_ground=True)
    assert np.array_equal(cls_pred.numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.numpy(), fx["att_idx"]) and np.array_equal(grd_idx.numpy(), fx["grd_idx"])


@pytest.mark.parametrize("name", _names("train"))
def test_region_attn_train_step_matches_reference(name):
    """Losses, the set of tensors that receive a gradient, per-tensor gradient norms / leading entries and the first Adam update."""
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    with oracle_modes(opt) as O:
        losses, loss, grads, total_norm, new = O.train_step(sd, opt, inp)
    _close(np.array([float(x) for x in losses]), fx["losses"])
    assert abs(float(loss) - float(fx["loss"])) <= TOL
    keys = [str(k) for k in fx["keys"]]
    assert sorted(grads.keys()) == keys
    if opt.region_attn_mode == "dp":
        assert not any("attention2" in k and "alpha_net" in k for k in sd)
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
def test_region_attn_train_step_orchestration_matches_oracle(name):
    """gvd_b200/train.py's forward tape and explicit backward (run on the CPU over the torch mock of its primitives) against autograd over
    the oracle: same gradient set, every gradient elementwise."""
    from gvd_b200.train import TrainStep
    opt, sd, inp = build_case(CASES[name])
    with oracle_modes(opt) as O:
        losses, loss, grads, total_norm, new = O.train_step(sd, opt, inp)
    l2, loss2, g2, tn2, new2 = TrainStep(RegionAttnRefOps()).step(sd, opt, inp)
    assert abs(float(loss2) - float(loss)) <= 1e-5
    for a, b in zip(losses, l2):
        assert abs(float(a) - float(b)) <= 1e-5
    assert sorted(g2.keys()) == sorted(grads.keys())
    scale = float(total_norm)
    assert abs(tn2 - scale) <= 1e-5 * scale
    for k in grads:
        a, b = grads[k], g2[k].reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max()) + 1e-7 * scale, k


def test_dp_trainer_steps_without_alpha_net():
    """Trainer needs no special case for 'dp': the state_dict has no region alpha_net, two steps run, and every other tensor trains."""
    from gvd_b200.train import Trainer
    opt, sd, inp = build_case(CASES["dp_train_small_B5"])
    tr = Trainer(RegionAttnRefOps(), sd, opt)
    for _ in range(2):
        tr.step(inp)
    assert not any("alpha_net" in k and "attention2" in k for k in tr.keys)
    for k in ("core.attention2.h2att.weight", "ctx2pool.weight", "core.attention.alpha_net.weight"):
        assert not torch.equal(tr.weights[k], sd[k]), k


@pytest.mark.parametrize("fixture", sorted(DP_KEYS_FIXTURES))
def test_dp_state_dict_matches_reference_keys(fixture):
    """TopDownModel(opt) in 'dp': the reference's keys, order and shapes (fixture from the unmodified reference), the synthetic state_dict
    alike, and the same tensors as the 'mix' state_dict minus the region alpha_net (byte-identical)."""
    from gvd_b200.misc.AttModel import TopDownModel
    fx = load_fixture(fixture)
    ref = list(zip((str(k) for k in fx["keys"]), (str(s) for s in fx["shapes"])))
    overrides = DP_KEYS_FIXTURES[fixture]
    opt = synth.make_opt(t_attn_size=10, **overrides)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    got = [(k, ",".join(str(n) for n in v.shape)) for k, v in m.state_dict().items()]
    assert got == ref
    sd = synth.make_state_dict(opt)
    assert [(k, ",".join(str(n) for n in v.shape)) for k, v in sd.items()] == ref
    m.load_state_dict(sd, strict=True)
    mix_sd = synth.make_state_dict(synth.make_opt(t_attn_size=10, **dict(overrides, region_attn_mode="mix")))
    absent = [k for k in mix_sd if k not in sd]
    assert absent and all(k.startswith(("core.attention2.alpha_net.", "core.attention2_dual.alpha_net.")) for k in absent)
    assert all(torch.equal(mix_sd[k], sd[k]) for k in sd)


def test_mix_mul_state_dict_is_mix():
    from gvd_b200.misc.AttModel import TopDownModel
    for extra in ({}, dict(att_input_mode="dual_region")):
        mix, mul = synth.make_opt(t_attn_size=10, **extra), synth.make_opt(t_attn_size=10, region_attn_mode="mix_mul", **extra)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            assert list(TopDownModel(mul).state_dict().keys()) == list(TopDownModel(mix).state_dict().keys())
        a, b = synth.make_state_dict(mix), synth.make_state_dict(mul)
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_option_surface():
    """'mix_mul' and 'dp' are accepted (top-down and transformer captioners); 'add' and 'cat' raise with the reason."""
    for mode, code in (("mix", 0), ("mix_mul", 1), ("dp", 2)):
        for extra in ({}, dict(att_input_mode="featmap"), dict(att_input_mode="dual_region"), dict(att_model="transformer")):
            opt = synth.make_opt(region_attn_mode=mode, **extra)
            assert bytes(capi.dims_from_opt(opt)) == bytes(capi.dims_from_opt(synth.make_opt(**extra)))
            assert capi.region_attn_mode_code(opt) == code
    for bad, why in (("add", "2048"), ("cat", "xt"), ("x", "implemented")):
        with pytest.raises(NotImplementedError, match=why):
            capi.dims_from_opt(synth.make_opt(region_attn_mode=bad))
        with pytest.raises(NotImplementedError):
            capi.region_attn_mode_code(synth.make_opt(region_attn_mode=bad))
    from gvd_b200.misc.AttModel import TopDownModel
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(synth.make_opt(region_attn_mode="dp"))
    assert m._opt_view().region_attn_mode == "dp" and m.opt_ns.region_attn_mode == "dp"


def test_att_scores_mul_kernels_index_emulation():
    """att_scores_mul_fwd (one warp per (b, n) row) and _bwd (flat over [B, N, A]) of csrc/gvd_train.cu, transliterated, against the
    primitive's definition (RegionAttnRefOps); dq and dw are then the colsum kernel's sums of the per-element terms."""
    rs = np.random.RandomState(0)
    f32 = lambda *s: rs.randn(*s).astype(np.float32)
    R_ = RegionAttnRefOps()
    Ba, Na, A = 2, 3, 40
    p, q, w, bias = f32(Ba, Na, A), f32(Ba, A), f32(A), f32(1)
    s = np.zeros(Ba * Na, np.float32)
    for row in range(Ba * Na):
        b = row // Na
        acc = 0.0
        for lane in range(32):
            for a_ in range(lane, A, 32):
                acc += w[a_] * np.tanh(p.ravel()[row * A + a_] * q.ravel()[b * A + a_])
        s[row] = acc + bias[0]
    assert np.allclose(s.reshape(Ba, Na), R_.att_scores_mul(*(torch.from_numpy(x) for x in (p, q, w, bias))).numpy(), atol=1e-5)
    ds = f32(Ba, Na)
    dp, dqt, dst = (np.zeros(Ba * Na * A, np.float32) for _ in range(3))
    for i in range(Ba * Na * A):
        a_ = i % A
        row = i // A
        b = row // Na
        pv, qv = p.ravel()[i], q.ravel()[b * A + a_]
        t = np.tanh(pv * qv)
        dpre = ds.ravel()[row] * w[a_] * (1 - t * t)
        dp[i], dqt[i], dst[i] = dpre * qv, dpre * pv, ds.ravel()[row] * t
    rp, rq, rw, rb = R_.att_scores_mul_bwd(*(torch.from_numpy(x) for x in (ds, p, q, w)))
    assert np.allclose(dp.reshape(Ba, Na, A), rp.numpy(), atol=1e-5)
    dq = np.zeros(Ba * A, np.float32)
    for z in range(Ba):                                  # colsum_kernel: out[z*N + n] = sum_m x[z*M*N + m*N + n]
        for n_ in range(A):
            dq[z * A + n_] = sum(dqt[z * Na * A + m * A + n_] for m in range(Na))
    assert np.allclose(dq.reshape(Ba, A), rq.numpy(), atol=1e-5) and np.allclose(dst.reshape(-1, A).sum(0), rw.numpy(), atol=1e-5)
    # the primitive against autograd
    pt, qt, wt, bt = (torch.from_numpy(x).double().requires_grad_() for x in (p, q, w, bias))
    (torch.from_numpy(ds).double() * (torch.tanh(pt * qt.unsqueeze(1)) @ wt + bt)).sum().backward()
    assert np.allclose(rp.numpy(), pt.grad.numpy(), atol=1e-5) and np.allclose(rq.numpy(), qt.grad.numpy(), atol=1e-5)
    assert np.allclose(rw.numpy(), wt.grad.numpy(), atol=1e-5) and np.allclose(rb.numpy(), bt.grad.numpy(), atol=1e-5)
