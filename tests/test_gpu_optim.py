"""The SGD and Adamax flat-buffer kernels (csrc/gvd_train.cu: gvd_tr_sgd_flat / gvd_tr_adamax_flat) against an fp64 restatement of
torch.optim's arithmetic, Trainer(optim=...) on the device against the CPU orchestration (tests/test_optim_host_logic.py checks that one
against torch.optim) and against the unmodified reference's steps (tests/golden/optim_cases.py), and disable_caption through Trainer and
through loss.backward() on the module."""
import numpy as np
import pytest
import torch

from cases import CASES, build_case, load_fixture
from optim_cases import OPTIM_CASES

pytestmark = pytest.mark.gpu


def _r(n, seed, scale=1.0):
    return (torch.randn(n, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale)


def _layout():
    """Ragged segments (lengths not multiples of 4 or of the block size), two idle ones, per-segment learning rates."""
    ends = np.cumsum([1, 4093, 3, 70001, 4, 256, 12345, 999999, 7]).tolist()
    lrs = [5e-4, 5e-5, 0.0, 5e-4, 5e-4, 0.0, 1e-3, 5e-4, 2e-4]
    return ends, lrs


def _fp64_step(optim, w, g, m, u, ends, lrs, steps, coef, wd, b1=0.9, b2=0.999, eps=1e-8, mu=0.9):
    """torch.optim.SGD(momentum=mu) / Adamax per segment in fp64; returns the new (w, g, m, u, steps) and d = g coef + wd w (0 where idle)."""
    w, g, m, u = w.clone(), g * coef, m.clone(), u.clone()
    dd = torch.zeros_like(w)
    lo = 0
    steps = list(steps)
    for s, (e, lr) in enumerate(zip(ends, lrs)):
        if lr > 0:
            d = g[lo:e] + wd * w[lo:e]
            dd[lo:e] = d
            if optim == "sgd":
                m[lo:e] = d if steps[s] == 0 else mu * m[lo:e] + d
                w[lo:e] -= lr * m[lo:e]
            else:
                m[lo:e] = b1 * m[lo:e] + (1 - b1) * d
                u[lo:e] = torch.maximum(b2 * u[lo:e], d.abs() + eps)
                w[lo:e] -= lr / (1 - b1 ** (steps[s] + 1)) * m[lo:e] / u[lo:e]
            steps[s] += 1
        lo = e
    return w, g, m, u, steps, dd


@pytest.mark.parametrize("optim,wd", [("sgd", 0.0), ("sgd", 1e-2), ("adamax", 0.0), ("adamax", 1e-2)])
def test_flat_kernels_match_fp64(optim, wd):
    """Three steps of the native kernel against fp64: clip coefficient < 1 read from the device, per-segment lr and step table (one segment
    idle on step 1 and live afterwards), idle segments bit-identical before and after, g clipped in place."""
    from gvd_b200.train_ops import NativeOps
    ops = NativeOps()
    ends, lrs = _layout()
    N = ends[-1]
    w64 = _r(N, 1, 0.1).float().double()
    m64, u64 = torch.zeros(N, dtype=torch.float64), torch.zeros(N, dtype=torch.float64)
    steps64 = [0] * len(ends)
    w, m, u = w64.float().cuda(), torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    seg_end = torch.tensor(ends, dtype=torch.int64, device="cuda")
    seg_step = torch.zeros(len(ends), dtype=torch.int32, device="cuda")
    w_before = w.clone()
    # Adamax's update lr d / (|d| + eps) is ill-conditioned where |d| ~ eps (the fp32 rounding of d = g coef + wd w is amplified up to
    # lr / eps): compare those elements to the step size only, the rest to fp64
    cond = torch.ones(N, dtype=torch.bool)
    for t in range(3):
        step_lrs = [0.0 if (t == 0 and s == 3) else lr for s, lr in enumerate(lrs)]          # segment 3: first gradient on step 2
        seg_lr = torch.tensor(step_lrs, dtype=torch.float32, device="cuda")
        g32 = _r(N, 10 + t, 1e-3).float()
        coef = 0.37 + 0.1 * t
        norm = torch.tensor([1.0, coef], dtype=torch.float32, device="cuda")
        g = g32.cuda()
        if optim == "sgd":
            ops.sgd_flat_(w, g, m, seg_end, seg_lr, seg_step, norm, 0.9, wd)
        else:
            ops.adamax_flat_(w, g, m, u, seg_end, seg_lr, seg_step, norm, 0.9, 0.999, 1e-8, wd)
        w64, g64, m64, u64, steps64, d64 = _fp64_step(optim, w64, g32.double(), m64, u64, ends, step_lrs, steps64, float(np.float32(coef)), wd)
        torch.cuda.synchronize()
        if optim == "adamax":
            lo = 0
            for s, e in enumerate(ends):
                if step_lrs[s] > 0:
                    cond[lo:e] &= d64[lo:e].abs() >= 1e-5
                lo = e
        dw = (w.cpu().double() - w64).abs()
        assert seg_step.cpu().tolist() == steps64, t
        assert float((g.cpu().double() - g64).abs().max()) <= 1e-7 * float(g64.abs().max())
        assert float(dw[cond].max()) <= 2.0 ** -22 * float(w64.abs().max()) + 1e-6 * 1e-3 * (t + 1), t
        assert float(dw.max()) <= 2e-3 * (t + 1) and float(cond.float().mean()) > 0.9, t
        assert float((m.cpu().double() - m64).abs().max()) <= 1e-5 * float(m64.abs().max()), t
        if optim == "adamax":
            assert float((u.cpu().double() - u64).abs().max()) <= 1e-5 * float(u64.abs().max()), t
    lo = 0
    for s, e in enumerate(ends):
        if lrs[s] <= 0:                                                             # idle throughout: weights and state untouched
            assert torch.equal(w[lo:e], w_before[lo:e]) and not m[lo:e].any() and not u[lo:e].any(), s
        lo = e
    assert seg_step.cpu().tolist() == [0 if lr <= 0 else (2 if s == 3 else 3) for s, lr in enumerate(lrs)]


def _trainers(opt, sd, optim, **kw):
    from gvd_b200.train import Trainer
    from gvd_b200.train_ops import NativeOps
    from optim_ref import OptimRefOps
    return Trainer(NativeOps(), sd, opt, optim=optim, **kw), Trainer(OptimRefOps(), sd, opt, optim=optim, **kw)


@pytest.mark.parametrize("optim", ["sgd", "adamax"])
def test_trainer_on_the_device_matches_the_cpu_orchestration(optim):
    """Trainer(optim=...) over NativeOps for three steps against the same Trainer over the torch mock (the bars of the Adam trajectory test
    in tests/test_gpu_zz_train.py)."""
    opt, sd, inp = build_case(CASES["train_small_B5"])
    dev = {k: v.cuda() for k, v in inp.items()}
    a, b = _trainers(opt, sd, optim, weight_decay=1e-4)
    for it in range(3):
        la, lossa = a.step(dev, host=inp)
        lb, lossb = b.step(inp)
        torch.cuda.synchronize()
        assert abs(float(lossa.cpu()) - float(lossb)) <= 1e-4 * (1 + 9 * it), it
        assert abs(float(a.norm[0].cpu()) - float(b.norm[0])) <= 2e-4 * (1 + 50 * it) * float(b.norm[0]), it
        for k in a.keys:
            wa, wb = a.weights[k].cpu(), b.weights[k]
            upd = float((wb - sd[k]).norm())
            assert float((wa - wb).abs().max()) <= 2 * 5e-4 * (it + 1), (it, k)
            if upd > 1e-7 and float(b.grad_view(k).norm()) > 1e-6 * float(b.norm[0]) * float(b.norm[1]):
                assert float((wa - wb).norm()) <= 5e-2 * upd + 2.0 ** -22 * float(sd[k].norm()), (it, k, float((wa - wb).norm()), upd)
    assert a.seg_step.cpu().tolist() == b.seg_step.tolist()


@pytest.mark.parametrize("name", list(OPTIM_CASES))
def test_trainer_on_the_device_matches_reference(name):
    """Trainer over NativeOps against the unmodified reference's own steps (fixture): loss, norm and every tensor's update, step by step."""
    case = OPTIM_CASES[name]
    opt, sd, inp = build_case(case)
    opt.disable_caption = case.get("disable_caption", False)
    fx = load_fixture(name)
    keys = [str(k) for k in fx["keys"]]
    dev = {k: v.cuda() for k, v in inp.items()}
    tr, _ = _trainers(opt, sd, case["optim"])
    prev = {k: v.cpu() for k, v in tr.weights.items()}
    for s in range(case["steps"]):
        losses, loss = tr.step(dev, host=inp)
        torch.cuda.synchronize()
        assert abs(float(loss.cpu()) - float(fx["loss"][s])) <= 1e-4 * (1 + 9 * s), s
        assert np.max(np.abs(np.array([float(x.cpu()) for x in losses]) - fx["losses"][s])) <= 1e-4 * (1 + 9 * s), s
        assert abs(float(tr.norm[0].cpu()) - float(fx["total_norm"][s])) <= 2e-4 * (1 + 50 * s) * float(fx["total_norm"][s]), s
        now = {k: v.cpu() for k, v in tr.weights.items()}
        for i, k in enumerate(keys):
            if fx["grad_norm"][i] <= 1e-6 * float(fx["total_norm"][0]):
                continue
            un, ur = float((now[k] - prev[k]).norm()), float(fx["update_norm"][s][i])
            assert abs(un - ur) <= 5e-2 * ur + 2.0 ** -22 * float(sd[k].norm()), (s, k, un, ur)
        prev = now
    if opt.disable_caption:
        for k in ("logit.weight", "logit.bias"):
            assert torch.equal(tr.weights[k].cpu(), sd[k])


@pytest.mark.parametrize("optim", ["adam", "sgd", "adamax"])
def test_disable_caption_through_trainer_keeps_the_lm_head(optim):
    opt, sd, inp = build_case(CASES["train_small_B5"])
    opt.disable_caption = True
    dev = {k: v.cuda() for k, v in inp.items()}
    a, b = _trainers(opt, sd, optim)
    for _ in range(3):
        la, _ = a.step(dev, host=inp)
        b.step(inp)
        assert float(la[0].cpu()) == 0.0
    torch.cuda.synchronize()
    assert a.idle == b.idle and {"logit.weight", "logit.bias"} <= a.idle
    for k in ("logit.weight", "logit.bias"):
        assert torch.equal(a.weights[k].cpu(), sd[k])


def test_disable_caption_through_the_module():
    """model.train(); losses = model(..., 'MLE'); the loss of main.py:234-253 with disable_caption (lm_loss.fill_(0), no lm term);
    loss.backward(): the logit head's .grad stays None, every other gradient equals the CPU orchestration's."""
    from gvd_b200.train import TrainStep
    from optim_ref import OptimRefOps
    from test_gpu_parity import _model
    opt, sd, inp = build_case(CASES["train_small_B5"])
    opt.disable_caption = True
    _, _, grads = TrainStep(OptimRefOps()).forward_backward(sd, opt, inp)
    model = _model(opt, sd)
    model.train()
    model.train_dropout = False
    dev = {k: v.cuda() for k, v in inp.items()}
    lm, att2, grd, cls = model(dev["segs_feat"], dev["input_seq"], dev["gt_seq"], dev["num"], dev["ppls"], dev["gt_boxes"], dev["mask_boxes"],
                               dev["ppls_feat"], dev["frm_mask"], dev["sample_idx"], dev["pnt_mask"], "MLE")
    loss = 0
    lm.fill_(0)
    loss += opt.w_att2 * att2.sum()
    loss += opt.w_grd * grd.sum()
    loss += opt.w_cls * cls.sum()
    (loss / lm.numel()).backward()
    scale = float(torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())))
    for k, p in model.named_parameters():
        if k in grads:
            assert float((p.grad.cpu() - grads[k].reshape(p.shape)).abs().max()) <= 1e-4 * float(grads[k].abs().max()) + 1e-6 * scale, k
        else:
            assert p.grad is None, k
    assert model.logit.weight.grad is None and model.logit.bias.grad is None
