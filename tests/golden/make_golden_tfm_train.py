"""Generate the transformer-captioner training-step fixtures by running the UNMODIFIED reference (read-only checkout, see ref_harness).

Run in the build container only:  ``python tests/golden/make_golden_tfm_train.py``
One optimisation step of att_model = 'transformer' as main.py:235-266 would take it if its driver could unpack this branch's six return values
(misc/model.py:418-419 against main.py:235): the model in train mode with every nn.Dropout at p = 0 and context_enc.dropout = 0 (the masks
come from torch's RNG, so only p = 0 is reproducible), loss = out[0].sum() / out[0].numel(), loss.backward(), clip_grad_norm_(0.1) and
torch.optim.Adam with one group per tensor (main.py:660-677).  ``ref_harness.ref_train_step`` cannot be reused: it unpacks four losses.
The case list lives here (not in cases.py::CASES) so the existing fixture parametrizations stay as they are.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from cases import SMALL  # noqa: E402

TFM = dict(att_model="transformer")
TFM_TRAIN_CASES = {
    "tfm_train_small_both":    dict(B=5, opt=dict(SMALL, **TFM), weight_seed=3, input_seed=5),
    "tfm_train_small_region":  dict(B=3, opt=dict(SMALL, att_input_mode="region", **TFM), weight_seed=4, input_seed=6),
    "tfm_train_small_featmap": dict(B=3, opt=dict(SMALL, att_input_mode="featmap", obj_interact=False, **TFM), weight_seed=5, input_seed=7),
    "tfm_train_T10_B3":        dict(B=3, opt=dict(t_attn_size=10, **TFM)),
}
N_SUB = 64                                                   # entries kept per tensor (every n-th element)


def build_tfm_case(case):
    import gvd_b200.synth as synth
    opt = synth.make_opt(**case["opt"])
    sd = synth.make_state_dict(opt, seed=case.get("weight_seed", 0))
    inp = synth.make_inputs(opt, case["B"], seed=case.get("input_seed", 1234), masked=True, train=True)
    return opt, sd, inp


def sub(t):
    """Every n-th element of the flattened tensor, at most N_SUB of them."""
    f = t.reshape(-1)
    return f[::max(1, f.numel() // N_SUB)][:N_SUB]


def pack(keys, grads, before, after, lm, total_norm):
    """Fixture arrays: the loss, the total norm, the sorted gradient keys, per key max|g| and the sub-sampled gradient / update."""
    return dict(lm=np.float32(lm), total_norm=np.float32(total_norm), keys=np.array(keys),
                grad_max=np.array([float(grads[k].abs().max()) for k in keys], dtype=np.float32),
                grad_sub=np.stack([np.resize(sub(grads[k]).numpy(), N_SUB) for k in keys]).astype(np.float32),
                update_sub=np.stack([np.resize(sub(after[k] - before[k]).numpy(), N_SUB) for k in keys]).astype(np.float32))


def run_case(case, lr=5e-4, grad_clip=0.1):
    import torch.nn as nn
    import gvd_b200.synth as synth
    import ref_harness as rh
    opt, sd, inp = build_tfm_case(case)
    model = rh.build_reference_model(opt, synth.make_detectron(opt))
    model.load_state_dict(sd, strict=True)
    for m in model.modules():
        if isinstance(m, nn.Dropout):
            m.p = 0.0
    model.context_enc.dropout = 0.0
    model.train()
    params = []
    for key, value in dict(model.named_parameters()).items():
        if value.requires_grad:
            step_lr = lr * 0.1 if ("ctx2pool_grd" in key) or ("vis_embed" in key) else lr
            params += [{"params": [value], "lr": step_lr, "weight_decay": 0, "betas": (0.9, 0.999)}]
    optimizer = torch.optim.Adam(params)
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    out = model(inp["segs_feat"], inp["input_seq"], inp["gt_seq"], inp["num"], inp["ppls"], inp["gt_boxes"], inp["mask_boxes"], inp["ppls_feat"],
                inp["frm_mask"], inp["sample_idx"], inp["pnt_mask"], "MLE")
    assert len(out) == 6
    loss = out[0].sum() / out[0].numel()
    model.zero_grad()
    loss.backward()
    grads = {k: v.grad.detach().clone() for k, v in model.named_parameters() if v.grad is not None}
    total_norm = nn.utils.clip_grad_norm_(model.parameters(), grad_clip)
    optimizer.step()
    after = {k: v.detach().clone() for k, v in model.named_parameters()}
    return pack(sorted(grads), grads, before, after, float(loss.detach()), float(total_norm))


def main():
    only = sys.argv[1:]
    for name, case in TFM_TRAIN_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %6.1fs %8.1f KB lm=%.6f norm=%.4f keys=%d" % (name, time.time() - t0, os.path.getsize(path) / 1024, out["lm"],
                                                                   out["total_norm"], len(out["keys"])))


if __name__ == "__main__":
    main()
