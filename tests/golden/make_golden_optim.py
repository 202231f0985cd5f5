"""Generate the optimiser / disable_caption golden fixtures (optim_cases.py) by running the UNMODIFIED reference on CPU, like make_golden.py.

The loop body is main.py:235-266 with the optimiser of main.py:660-677: one param group per tensor (lr x 0.1 for ctx2pool_grd / vis_embed,
weight_decay, betas = (optim_alpha, optim_beta)), optim.SGD(params, momentum=0.9) / optim.Adam(params) / optim.Adamax(params), every Dropout
off and BatchNorm in train mode (ref_harness.ref_train_step's deterministic set-up), `steps` steps on the same batch.

Run in the build container only:  ``python tests/golden/make_golden_optim.py [case ...]``"""
import os
import sys
import time

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import gvd_b200.synth as synth  # noqa: E402
import ref_harness as rh  # noqa: E402
from cases import build_case  # noqa: E402
from optim_cases import OPTIM_CASES  # noqa: E402


def ref_train_steps(model, inp, opt, optim, steps, disable_caption, lr=5e-4, grad_clip=0.1):
    for m in model.modules():
        if isinstance(m, nn.Dropout):
            m.p = 0.0
    model.core.drop_prob_lm = 0.0
    model.context_enc.dropout = 0.0
    model.train()
    params = []
    for key, value in dict(model.named_parameters()).items():
        if value.requires_grad:
            step_lr = lr * 0.1 if ("ctx2pool_grd" in key) or ("vis_embed" in key) else lr
            params += [{"params": [value], "lr": step_lr, "weight_decay": 0, "betas": (0.9, 0.999)}]
    optimizer = {"sgd": lambda: torch.optim.SGD(params, momentum=0.9), "adam": lambda: torch.optim.Adam(params),
                 "adamax": lambda: torch.optim.Adamax(params)}[optim]()
    out = dict(losses=[], loss=[], total_norm=[], update_norm=[], update_head=[])
    for _ in range(steps):
        before = {k: v.detach().clone() for k, v in model.named_parameters()}
        loss = 0
        lm_loss, att2_loss, ground_loss, cls_loss = rh.ref_mle(model, inp, train_mode=True)
        raw = [att2_loss, ground_loss, cls_loss]
        att2_loss = opt.w_att2 * att2_loss.sum()
        ground_loss = opt.w_grd * ground_loss.sum()
        cls_loss = opt.w_cls * cls_loss.sum()
        if not disable_caption:                                          # main.py:243-246
            loss += lm_loss.sum()
        else:
            lm_loss.fill_(0)
        if opt.w_att2:
            loss += att2_loss
        if opt.w_grd:
            loss += ground_loss
        if opt.w_cls:
            loss += cls_loss
        loss = loss / lm_loss.numel()
        model.zero_grad()
        loss.backward()
        grads = {k: v.grad.detach().clone() for k, v in model.named_parameters() if v.grad is not None}
        total_norm = nn.utils.clip_grad_norm_(model.parameters(), grad_clip)
        optimizer.step()
        after = {k: v.detach().clone() for k, v in model.named_parameters()}
        keys = sorted(before)
        out["losses"].append([float(x.detach()) for x in [lm_loss] + raw])          # (lm_loss after the fill)
        out["loss"].append(float(loss))
        out["total_norm"].append(float(total_norm))
        out["update_norm"].append([float((after[k] - before[k]).norm()) for k in keys])
        out["update_head"].append(np.stack([np.resize((after[k] - before[k]).flatten()[:8].numpy(), 8) for k in keys]))
        if "keys" not in out:
            out["keys"] = np.array(keys)
            out["grad_keys"] = np.array(sorted(grads))
            out["grad_norm"] = np.array([float(grads[k].norm()) if k in grads else 0.0 for k in keys], dtype=np.float32)
    return {k: (v if isinstance(v, np.ndarray) else np.asarray(v, dtype=np.float32)) for k, v in out.items()}


def run_case(case):
    opt, sd, inp = build_case(case)
    model = rh.build_reference_model(opt, synth.make_detectron(opt))
    model.load_state_dict(sd, strict=True)
    return ref_train_steps(model, inp, opt, case["optim"], case["steps"], case.get("disable_caption", False))


def main():
    only = sys.argv[1:]
    for name, case in OPTIM_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %6.1fs %8.1f KB" % (name, time.time() - t0, os.path.getsize(path) / 1024), flush=True)


if __name__ == "__main__":
    main()
