"""The training loop's SGD and Adamax optimisers (main.py:671-677) and --disable_caption (main.py:243-246) on the CPU: gvd_b200.train.Trainer
over the torch mock of its primitives (tests/optim_ref.py) against torch.optim driven by the oracle's gradients, against the unmodified
reference's own steps (tests/golden/optim_cases.py, make_golden_optim.py), the per-tensor optimiser state, the module path, the refusals,
and the gradient all-reduce hook over gloo.  The native kernels are checked in tests/test_gpu_optim.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import gvd_oracle as O
from cases import CASES, build_case, load_fixture
from gvd_b200.dist import shard_range
from gvd_b200.train import TrainStep, Trainer
from optim_cases import OPTIM_CASES
from optim_ref import OptimRefOps

LR = 5e-4


def _lr(k, lr=LR):
    return lr * 0.1 if ("ctx2pool_grd" in k or "vis_embed" in k) else lr


def _torch_optim(optim, params, weight_decay):
    groups = [{"params": [p], "lr": _lr(k), "weight_decay": weight_decay, "betas": (0.9, 0.999)} for k, p in params.items()]
    return torch.optim.SGD(groups, momentum=0.9) if optim == "sgd" else torch.optim.Adamax(groups)     # main.py:673,677


def build_optim_case(name):
    case = OPTIM_CASES[name]
    opt, sd, inp = build_case(case)
    opt.disable_caption = case.get("disable_caption", False)
    return case, opt, sd, inp


@pytest.mark.parametrize("optim,weight_decay,decay", [("sgd", 0.0, False), ("sgd", 1e-2, True), ("adamax", 0.0, False), ("adamax", 1e-2, True)])
def test_trainer_three_steps_match_torch_optim_on_oracle_gradients(optim, weight_decay, decay):
    """Trainer(optim=...) (flat buffers, device-side clip coefficient, per-tensor step table) against torch.optim.SGD(momentum=0.9) /
    torch.optim.Adamax + clip_grad_norm_(0.1) driven by the oracle's autograd gradients, three steps on the same batch; `decay`: the
    learning rate is multiplied by 0.8 between the steps (utils.set_lr, main.py:680-684)."""
    opt, sd, inp = build_case(CASES["train_small_B5"])
    tr = Trainer(OptimRefOps(), sd, opt, weight_decay=weight_decay, optim=optim)
    params = {k: torch.nn.Parameter(sd[k].clone()) for k in tr.keys}
    ref_opt = _torch_optim(optim, params, weight_decay)
    for it in range(3):
        if decay and it:
            for g in ref_opt.param_groups:
                g["lr"] *= 0.8
            tr.set_lr(tr.lr * 0.8)
        W = {k: (params[k].detach() if k in params else v) for k, v in sd.items()}
        W.update({k: v for k, v in tr.buffers.items() if "running_" in k})
        losses, loss, grads, total_norm, _ = O.train_step(W, opt, inp)
        for k, p in params.items():
            p.grad = grads[k].clone() if k in grads else None
        torch.nn.utils.clip_grad_norm_(list(params.values()), 0.1)
        ref_opt.step()
        tr.step(inp)
        assert abs(float(tr.norm[0]) - float(total_norm)) <= 1e-3 * float(total_norm), it
        for k in tr.keys:
            a, b = params[k].detach(), tr.weights[k]
            upd = float((a - sd[k]).norm())
            if k not in grads:
                assert torch.equal(b, sd[k]), k                                       # idle: bit-identical
                continue
            assert float((a - b).abs().max()) <= 2 * LR * (it + 1), (it, k)
            if upd > 0 and float(grads[k].norm()) > 1e-6 * float(total_norm):
                # (plus fp32 rounding of the weights, one half-ulp per step: SGD's updates of small tensors come close to it)
                ulp = (it + 1) * 2.0 ** -23 * float(sd[k].norm())
                assert float((a - b).norm()) <= 2e-2 * upd + ulp, (it, k, float((a - b).norm()), upd)
    assert tr.seg_step.tolist() == [0 if k.startswith(("core.i2h_2", "core.h2h_2")) else 3 for k in tr.keys]


@pytest.mark.parametrize("optim", ["sgd", "adamax"])
def test_tensor_idle_on_step_one_starts_its_own_state(optim):
    """torch keeps the optimiser state per parameter: a tensor without a gradient on step 1 and with one on step 2 starts its momentum
    buffer (SGD: buf = d) / its bias correction (Adamax: t = 1) on step 2, and is left bit-identical on step 1."""
    opt, sd, _ = build_case(CASES["train_small_B5"])
    tr = Trainer(OptimRefOps(), sd, opt, optim=optim)
    keys = [k for k in tr.keys if not k.startswith(("core.i2h_2", "core.h2h_2"))]
    late = ["logit.weight", "core.att_lstm.bias_ih"]
    params = {k: torch.nn.Parameter(sd[k].clone()) for k in keys}
    ref_opt = _torch_optim(optim, params, 0.0)
    gen = torch.Generator().manual_seed(11)
    for it in range(2):
        idle = set(late) if it == 0 else set()
        grads = {k: torch.randn(sd[k].shape, generator=gen) * 1e-5 for k in keys if k not in idle}      # norm < 0.1: no clipping
        for k, p in params.items():
            p.grad = grads[k].clone() if k in grads else None
        torch.nn.utils.clip_grad_norm_(list(params.values()), 0.1)
        ref_opt.step()
        tr.flat_g.zero_()
        for k, g in grads.items():
            tr.grad_view(k).copy_(g)
        tr.idle = frozenset(k for k in tr.keys if k not in grads)
        tr.set_lr(tr.lr)
        tr.apply()
        for k in keys:
            if k in idle:
                assert torch.equal(tr.weights[k], sd[k]), k
            else:
                a, b = params[k].detach(), tr.weights[k]
                assert float((a - b).abs().max()) <= 1e-5 * float((a - sd[k]).abs().max()) + 2.0 ** -22 * float(sd[k].abs().max()), (it, k)
    steps = dict(zip(tr.keys, tr.seg_step.tolist()))
    assert steps["logit.weight"] == 1 and steps["core.att_lstm.bias_ih"] == 1 and steps["logit.bias"] == 2


@pytest.mark.parametrize("name", [n for n, c in OPTIM_CASES.items() if c["optim"] != "adam"])
def test_trainer_steps_match_reference(name):
    """Trainer(optim='sgd' / 'adamax') over the torch mock against the unmodified reference's own loss.backward() / clip_grad_norm_ /
    optim.SGD(momentum=0.9) / optim.Adamax, step by step (fixture)."""
    case, opt, sd, inp = build_optim_case(name)
    fx = load_fixture(name)
    keys = [str(k) for k in fx["keys"]]
    tr = Trainer(OptimRefOps(), sd, opt, optim=case["optim"])
    prev = {k: v.clone() for k, v in tr.weights.items()}
    for s in range(case["steps"]):
        losses, loss = tr.step(inp)
        assert abs(float(loss) - float(fx["loss"][s])) <= 1e-4, s
        assert np.max(np.abs(np.array([float(x) for x in losses]) - fx["losses"][s])) <= 1e-4, s
        assert abs(float(tr.norm[0]) - float(fx["total_norm"][s])) <= 1e-3 * float(fx["total_norm"][s]), s
        for i, k in enumerate(keys):
            un, ur = float((tr.weights[k] - prev[k]).norm()), float(fx["update_norm"][s][i])
            if fx["grad_norm"][i] <= 1e-6 * float(fx["total_norm"][0]):
                continue                                       # (zero-gradient tensors: the update is rounding noise)
            assert abs(un - ur) <= 5e-3 * ur + 1e-9, (s, k, un, ur)
        prev = {k: v.clone() for k, v in tr.weights.items()}


def test_disable_caption_matches_reference_and_oracle():
    """disable_caption (main.py:243-246): lm reported as 0, loss = (w_att2 att2 + w_grd grd + w_cls cls) / n, the reference's set of
    tensors with a gradient (all but the logit head and quirk Q10's i2h_2 / h2h_2), the gradients of the oracle's autograd over that loss,
    and the reference's Adam update (fixture)."""
    case, opt, sd, inp = build_optim_case("nocap_train_small_B5")
    fx = load_fixture("nocap_train_small_B5")
    keys = [str(k) for k in fx["keys"]]
    losses, loss, grads = TrainStep(OptimRefOps()).forward_backward(sd, opt, inp)
    assert float(losses[0]) == 0.0
    assert np.max(np.abs(np.array([float(x) for x in losses]) - fx["losses"][0])) <= 1e-4
    assert abs(float(loss) - float(fx["loss"][0])) <= 1e-4
    assert sorted(grads) == sorted(str(k) for k in fx["grad_keys"])
    assert not any(k.startswith("logit.") for k in grads)
    P = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running_" not in k else v) for k, v in sd.items()}
    _, att2, grd, cls = O.forward_teacher(P, opt, inp, train_bn=True)
    ks = [k for k in P if torch.is_tensor(P[k]) and P[k].requires_grad]
    ref = {k: g for k, g in zip(ks, torch.autograd.grad(opt.w_att2 * att2 + opt.w_grd * grd + opt.w_cls * cls, [P[k] for k in ks],
                                                        allow_unused=True)) if g is not None}
    assert sorted(ref) == sorted(grads)
    scale = float(torch.sqrt(sum((g.double() ** 2).sum() for g in ref.values())))
    for k in ref:
        assert float((ref[k] - grads[k].reshape(ref[k].shape)).abs().max()) <= 1e-5 * float(ref[k].abs().max()) + 1e-7 * scale, k
    # the language LSTM is reached only through the stacked decode state: exact zeros, as in the reference
    assert all(float(grads[k].abs().max()) == 0.0 for k in grads if k.startswith("core.lang_lstm."))
    tr = Trainer(OptimRefOps(), sd, opt)
    tr.step(inp)
    for i, k in enumerate(keys):
        un, ur = float((tr.weights[k] - sd[k]).norm()), float(fx["update_norm"][0][i])
        if fx["grad_norm"][i] > 1e-6 * float(fx["total_norm"][0]):
            assert abs(un - ur) <= 5e-3 * ur + 1e-9, (k, un, ur)


@pytest.mark.parametrize("optim", ["adam", "sgd", "adamax"])
def test_disable_caption_leaves_the_lm_head_bit_identical(optim):
    """Three Trainer steps with disable_caption: the logit head gets no gradient and is not touched by any of the three optimisers (lr 0:
    no update, no decay, no state), while the grounding tensors train."""
    opt, sd, inp = build_case(CASES["train_small_B5"])
    opt.disable_caption = True
    tr = Trainer(OptimRefOps(), sd, opt, weight_decay=1e-2, optim=optim)
    for _ in range(3):
        losses, _ = tr.step(inp)
        assert float(losses[0]) == 0.0
    for k in ("logit.weight", "logit.bias"):
        assert torch.equal(tr.weights[k], sd[k]) and k in tr.idle
        seg = slice(tr.offsets[k], tr.offsets[k] + sd[k].numel())
        assert not tr.flat_m[seg].any() and not tr.flat_v[seg].any()
    assert not torch.equal(tr.weights["core.attention2.h2att.weight"], sd["core.attention2.h2att.weight"])


def test_disable_caption_through_the_module_autograd_node():
    """The module path (train_autograd.MLEFunction, main.py:238-266): the reference driver's loss without lm — lm_loss.fill_(0) included —
    leaves the logit head's .grad None, and every other gradient equals the explicit backward's."""
    from gvd_b200.train_autograd import mle_losses
    opt, sd, inp = build_case(CASES["train_small_B5"])
    opt.disable_caption = True
    _, _, grads = TrainStep(OptimRefOps()).forward_backward(sd, opt, inp)
    params = [(k, v.clone().requires_grad_(True)) for k, v in sd.items() if v.is_floating_point() and "running_" not in k]
    lm, att2, grd, cls = mle_losses(TrainStep(OptimRefOps()), opt, inp, inp, params)
    loss = 0                                                                        # main.py:234-253, as written
    lm.fill_(0)
    loss += opt.w_att2 * att2.sum()
    loss += opt.w_grd * grd.sum()
    loss += opt.w_cls * cls.sum()
    (loss / lm.numel()).backward()
    for k, p in params:
        if k in grads:
            assert p.grad is not None and float((p.grad - grads[k].reshape(p.shape)).abs().max()) <= 1e-6 * float(grads[k].abs().max()) + 1e-9, k
        else:
            assert p.grad is None, k
    assert {k for k, p in params if p.grad is None} == {"logit.weight", "logit.bias", "core.i2h_2.weight", "core.i2h_2.bias", "core.h2h_2.weight",
                                                          "core.h2h_2.bias"}


def test_refusals():
    opt, sd, inp = build_case(CASES["train_small_B5"])
    with pytest.raises(ValueError, match="sgd.*adamax"):
        Trainer(OptimRefOps(), sd, opt, optim="rmsprop")
    opt.disable_caption = True
    opt.w_att2 = opt.w_grd = opt.w_cls = 0.0
    with pytest.raises(ValueError, match="empty"):
        Trainer(OptimRefOps(), sd, opt)
    with pytest.raises(ValueError, match="empty"):
        TrainStep(OptimRefOps()).forward_backward(sd, opt, inp)
    topt, tsd, _ = build_case(CASES["tfm_mle_small_B5"])
    topt.disable_caption = True
    with pytest.raises(ValueError, match="transformer"):
        Trainer(OptimRefOps(), tsd, topt)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _gloo_worker(rank, world, port, optim, q):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    for p_ in ("oracle", os.path.join("tests", "golden"), "tests"):
        sys.path.insert(0, os.path.join(root, p_))
    from cases import CASES, build_case
    from gvd_b200.dist import allreduce_flat
    from gvd_b200.train import Trainer
    from optim_ref import OptimRefOps
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    opt, sd, inp = build_case(CASES["train_small_B5"])
    lo, hi = shard_range(4, rank, world)
    shard = {k: v[lo:hi].contiguous() for k, v in inp.items()}
    calls = []

    def hook(flat):
        calls.append(flat.numel())
        return allreduce_flat(flat)
    tr = Trainer(OptimRefOps(), sd, opt, all_reduce=hook, n_replicas=world, optim=optim)
    for _ in range(2):
        tr.step(shard)
    q.put((rank, calls, tr.numel, tr.flat_w.double().norm().item(), tr.seg_step.tolist()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("optim", ["sgd", "adamax"])
def test_all_reduce_hook_once_per_step_over_gloo(optim):
    """Two gloo ranks: ONE all-reduce of the whole flat gradient buffer per step with each optimiser, and both ranks end in the same state."""
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, optim, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, calls, numel, wn, steps in results:
        assert calls == [numel, numel]
    assert results[0][3:] == results[1][3:]
