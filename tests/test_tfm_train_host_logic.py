"""The transformer captioner's training step (att_model = 'transformer') on the CPU: the specification (tests/tfm_train_ref.tfm_train_step)
against the fixtures made by the unmodified reference, and the product's orchestration (gvd_b200.train.TrainStep / Trainer) over the torch
mock of its primitives against the specification.  The native primitives are checked on the device in tests/test_gpu_tfm_train.py."""
import numpy as np
import pytest
import torch

import gvd_oracle as O
from make_golden_tfm_train import TFM_TRAIN_CASES, build_tfm_case, sub
from cases import CASES, build_case, load_fixture
from gvd_b200.train import DROP_SITES, TFM_DROP_SITES, TrainStep, Trainer
from gvd_b200 import capi
from tfm_train_ref import TfmRefOps, tfm_lm, tfm_train_step

SMALL_CASES = [n for n in TFM_TRAIN_CASES if "small" in n]


@pytest.mark.parametrize("name", list(TFM_TRAIN_CASES))
def test_specification_matches_reference_fixture(name):
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES[name])
    fx = load_fixture(name)
    lm, loss, grads, total_norm, new = tfm_train_step(sd, opt, inp)
    assert abs(float(lm) - float(fx["lm"])) <= 1e-4
    # the reference's clip_grad_norm_ takes fp32 norms of each tensor on the CPU; for the 5 M-entry out.weight gradient that norm is off by
    # ~1e-3 relative, so the bar on the norm is 1e-3 (the specification sums the squares in fp64)
    assert abs(float(total_norm) - float(fx["total_norm"])) <= 1e-3 * float(fx["total_norm"])
    keys = [str(k) for k in fx["keys"]]
    assert sorted(grads) == keys
    for i, k in enumerate(keys):
        gmax = float(fx["grad_max"][i])
        assert abs(float(grads[k].abs().max()) - gmax) <= 1e-4 * gmax + 1e-12, k
        assert np.max(np.abs(sub(grads[k]).numpy() - fx["grad_sub"][i][:sub(grads[k]).numel()])) <= 1e-4 * gmax + 1e-12, k
        upd = sub(new[k] - sd[k]).numpy()
        ref = fx["update_sub"][i][:upd.size]
        # Adam's g / (|g| + eps) turns rounding noise of a near-zero gradient into a full step: compare the updates as a whole
        assert np.linalg.norm(upd - ref) <= 5e-3 * np.linalg.norm(ref) + 1e-9 or gmax <= 1e-6 * float(fx["total_norm"]), k


def test_specification_decoder_is_the_eval_loss_without_dropout():
    """tfm_lm over the eval-mode prologue is the oracle's tfm_mle (the eval-mode loss pinned by tfm_mle_small_B5), bit for bit."""
    opt, sd, inp = build_case(CASES["tfm_mle_small_B5"])
    f = O.prologue(sd, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    assert torch.equal(tfm_lm(sd, opt, inp, f), O.tfm_mle(sd, opt, inp))


def _check_grads(grads, g2, total_norm, rel=5e-5, absn=1e-7):
    """(5e-5: the fp32 rounding of the deeper chain — prologue, encoder and two decoder layers — reaches 2.3e-5 of max|g| on a few tensors)"""
    assert sorted(g2) == sorted(grads)
    scale = float(total_norm)
    for k in grads:
        a, b = grads[k], g2[k].reshape(grads[k].shape)
        assert float((a - b).abs().max()) <= rel * float(a.abs().max()) + absn * scale, k


@pytest.mark.parametrize("name", SMALL_CASES + ["tfm_train_T10_B3"])
def test_orchestration_matches_specification(name):
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES[name])
    lm, loss, grads, total_norm, new = tfm_train_step(sd, opt, inp)
    losses, loss2, g2, tn2, new2 = TrainStep(TfmRefOps()).step(sd, opt, inp)
    assert abs(float(loss2) - float(loss)) <= 1e-5 and abs(float(losses[0]) - float(lm)) <= 1e-5
    assert all(float(x) == 0.0 for x in losses[1:])
    assert abs(tn2 - float(total_norm)) <= 1e-5 * float(total_norm)
    _check_grads(grads, g2, total_norm)
    for k in grads:
        if float(grads[k].norm()) > 1e-6 * float(total_norm):
            un, ur = float((new2[k] - sd[k]).norm()), float((new[k] - sd[k]).norm())
            assert abs(un - ur) <= 5e-3 * ur + 1e-9, k


def test_dropout_masks_forward_and_backward_are_consistent():
    """With the product's Philox masks injected into the specification's hook, autograd's gradients equal the explicit backward's at every
    site of the decoder and the prologue; the masks change the loss, and the next step draws new ones."""
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES["tfm_train_small_both"])
    ops = TfmRefOps()
    cfg = dict(seed=77, p_lm=0.5, p_interact=0.2, p_gru=0.2, p_loc=0.5, p_tfm=0.2)
    P = {"lm": 0.5, "interact": 0.2, "gru": 0.2, "loc": 0.5, "tfm": 0.2}
    ids = dict(DROP_SITES, **TFM_DROP_SITES)
    used = []

    def make_hook(it):
        def drop(x, kind, site, sub=0):
            used.append(site)
            return ops.dropout(x.contiguous(), P[kind], cfg["seed"], ids[site] * 4096 + sub, it)
        return drop
    ts = TrainStep(ops, dropout=cfg)
    base = tfm_train_step(sd, opt, inp)
    prev = None
    for it in range(2):
        lm, loss, grads, total_norm, _ = tfm_train_step(sd, opt, inp, drop=make_hook(it))
        losses, loss2, g2 = ts.forward_backward(sd, opt, inp)
        assert abs(float(loss2) - float(loss)) <= 2e-5
        assert abs(float(loss) - float(base[1])) > 1e-3
        _check_grads(grads, g2, total_norm)
        if prev is not None:
            assert abs(prev - float(loss)) > 1e-4
        prev = float(loss)
    assert set(TFM_DROP_SITES) <= set(used)
    assert min(TFM_DROP_SITES.values()) == len(DROP_SITES)                       # appended: the masks of the existing sites are unchanged


def test_input_checks():
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES["tfm_train_small_region"])
    ts = TrainStep(TfmRefOps())
    bad = dict(inp, gt_seq=inp["gt_seq"].clone())
    bad["gt_seq"][0, 0, 2] = opt.vocab_size
    with pytest.raises(IndexError):
        ts.forward(sd, opt, bad)
    bad["gt_seq"][0, 0, 2] = -1
    with pytest.raises(IndexError):
        ts.forward(sd, opt, bad)
    with pytest.raises(capi.GvdError):
        ts.forward(sd, opt, dict(inp, gt_seq=torch.zeros_like(inp["gt_seq"])))


@pytest.mark.parametrize("name,weight_decay", [("tfm_train_small_both", 0.0), ("tfm_train_small_region", 1e-4)])
def test_trainer_three_steps_match_torch_adam(name, weight_decay):
    """Trainer (flat buffers) against torch.optim.Adam + clip_grad_norm_ for three steps, both fed the Trainer's gradients (the gradients
    themselves are checked against the specification above): tensors without a gradient come out bit-identical, weight decay included, because
    Adam skips them; BatchNorm statistics move only when the frame branch ran."""
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES[name])
    tr = Trainer(TfmRefOps(), sd, opt, weight_decay=weight_decay)
    params = {k: torch.nn.Parameter(sd[k].clone()) for k in tr.keys}
    groups = [{"params": [p], "lr": 5e-4 * (0.1 if ("ctx2pool_grd" in k or "vis_embed" in k) else 1.0)} for k, p in params.items()]
    adam = torch.optim.Adam(groups, betas=(0.9, 0.999), eps=1e-8, weight_decay=weight_decay)
    for it in range(3):
        losses, loss = tr.forward_backward(inp)
        if it == 0:
            assert abs(float(loss) - float(tfm_train_step(sd, opt, inp)[1])) <= 1e-5
        for k, p in params.items():
            p.grad = None if k in tr.idle else tr.grad_view(k).clone()
        torch.nn.utils.clip_grad_norm_(list(params.values()), 0.1)
        adam.step()
        tr.apply()
        for k in tr.keys:
            a, b = params[k].detach(), tr.weights[k]
            if k in tr.idle:
                assert torch.equal(b, sd[k]) and torch.equal(a, sd[k]), k
            elif not weight_decay:
                assert float((a - b).abs().max()) <= 1e-3 * float((a - sd[k]).abs().max()) + 1e-7, (it, k)
            else:           # where g nearly cancels the decay term, Adam's normalised step depends on the last bits: bound it by the step size
                assert float((a - b).abs().max()) <= 2 * 5e-4 * (it + 1), (it, k)
    assert {"core.att_lstm.weight_ih", "embed.0.weight", "logit.weight", "ctx2pool.weight", "fc_embed.0.weight"} <= tr.idle
    region = opt.att_input_mode == "region"
    assert ("context_enc.weight_hh_l0" in tr.idle) == region
    for k in ("att_embed_aux.0.running_mean", "att_embed_aux.0.running_var"):
        assert torch.equal(tr.buffers[k], sd[k]) == region, k


def test_top_down_trainer_idle_set_is_the_never_set():
    """The top-down step's tensors without a gradient are exactly core.i2h_2 / h2h_2: its learning-rate table does not change."""
    opt, sd, inp = build_case(CASES["train_small_B5"])
    tr = Trainer(TfmRefOps(), sd, opt)
    before = tr.seg_lr.clone()
    tr.forward_backward(inp)
    assert all(k.startswith(tr.never) for k in tr.idle) and torch.equal(tr.seg_lr, before)


def test_apply_bumps_the_versions_of_adopted_parameters():
    """The flat Adam update bypasses torch's version counters; Trainer.apply bumps them so a module's cached native weights are refreshed."""
    from gvd_b200.misc.AttModel import TopDownModel
    import warnings
    opt, sd, inp = build_tfm_case(TFM_TRAIN_CASES["tfm_train_small_featmap"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    tr = Trainer(TfmRefOps(), sd, opt)
    tr.adopt_module(m)
    v0 = {k: p._version for k, p in m.named_parameters()}
    tr.step(inp)
    assert all(p._version > v0[k] for k, p in m.named_parameters() if k in tr.weights)
    assert torch.equal(dict(m.named_parameters())["cap_model.decoder.out.bias"].detach(), tr.weights["cap_model.decoder.out.bias"])
