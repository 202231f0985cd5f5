"""Measurement aid: the three flat optimiser updates of gvd_b200.train.Trainer (gvd_tr_adam_flat / gvd_tr_sgd_flat / gvd_tr_adamax_flat) on the
real layout — every trainable tensor of the full-dims top-down captioner in one flat fp32 buffer, one segment per tensor, 16-byte aligned,
one idle segment pair (core.i2h_2 / h2h_2) like the product's.

Per optimiser: CUDA events around one update call (the clip coefficient already on the device), median and minimum of --reps calls after
--warmup, alternating the three optimisers call by call.  Bytes are what the update has to move: SGD reads and writes w, g and the momentum
buffer (6 x 4 bytes per element), Adam and Adamax read and write w, g and two moments (8 x 4 bytes per element).  Prints the card name and
power limit with the numbers, one JSON line per optimiser."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=5)
args = ap.parse_args()
assert args.reps >= 20, "the medians want at least 20 calls"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from gvd_b200 import synth  # noqa: E402
from gvd_b200.train_ops import NativeOps  # noqa: E402

assert torch.cuda.is_available(), "optim_bench measures on a CUDA device"
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

opt = synth.make_opt()
sd = synth.make_state_dict(opt)
keys = [k for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point() and "running_" not in k]
ends, o = [], 0
for k in keys:
    o += (sd[k].numel() + 3) // 4 * 4
    ends.append(o)
n = o
lrs = [0.0 if k.startswith(("core.i2h_2", "core.h2h_2")) else (5e-5 if ("ctx2pool_grd" in k or "vis_embed" in k) else 5e-4) for k in keys]
ops = NativeOps()
g = torch.Generator().manual_seed(0)
w = (torch.randn(n, generator=g) * 0.05).cuda()
grad0 = (torch.randn(n, generator=g) * 1e-3).cuda()
grad = grad0.clone()
m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
seg_end = torch.tensor(ends, dtype=torch.int64, device="cuda")
seg_lr = torch.tensor(lrs, dtype=torch.float32, device="cuda")
seg_step = torch.zeros(len(keys), dtype=torch.int32, device="cuda")
norm = torch.tensor([1.0, 1.0], device="cuda")            # clip coefficient 1: g stays the same call after call
ts = {"adam": 0}


def adam():
    ts["adam"] += 1
    ops.adam_flat_(w, grad, m, v, seg_end, seg_lr, norm, 0.9, 0.999, 1e-8, 0.0, ts["adam"])


UPDATES = {
    "adam": (adam, 8),
    "sgd": (lambda: ops.sgd_flat_(w, grad, m, seg_end, seg_lr, seg_step, norm, 0.9, 0.0), 6),
    "adamax": (lambda: ops.adamax_flat_(w, grad, m, v, seg_end, seg_lr, seg_step, norm, 0.9, 0.999, 1e-8, 0.0), 8),
}
for fn, _ in UPDATES.values():
    for _ in range(args.warmup):
        fn()
torch.cuda.synchronize()
ms = {name: [] for name in UPDATES}
for _ in range(args.reps):
    for name, (fn, _) in UPDATES.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms[name].append(e0.elapsed_time(e1))
assert bool(torch.isfinite(w).all())
print("card: %s   elements: %d (%d tensors)" % (card, n, len(keys)))
for name, (fn, words) in UPDATES.items():
    t = sorted(ms[name])
    med = t[len(t) // 2]
    nbytes = words * 4 * n
    print(json.dumps({"optim": name, "elements": n, "bytes": nbytes, "median_ms": round(med, 4), "min_ms": round(t[0], 4),
                      "achieved_GBps": round(nbytes / (med * 1e-3) / 1e9, 1), "reps": args.reps, "card": card}))
