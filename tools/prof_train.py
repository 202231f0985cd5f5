"""Profiling aid: one training step (B=100, T=10, dropout off) (for use under a profiler); argv[1] = number of steps after one warm-up."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import synth
from gvd_b200.train import Trainer
from gvd_b200.train_ops import NativeOps
B, T = 100, 10
opt = synth.make_opt(t_attn_size=T)
opt.w_att2, opt.w_grd, opt.w_cls = 0.1, 0.0, 0.1
sd = synth.make_state_dict(opt)
inp = synth.make_inputs(opt, B, seed=4321, masked=True, train=True)
dev = {k: v.cuda() for k, v in inp.items()}
host = {k: inp[k] for k in ("gt_seq", "input_seq", "sample_idx")}
tr = Trainer(NativeOps(), sd, opt)
import time
for i in range(1 + (int(sys.argv[1]) if len(sys.argv) > 1 else 1)):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    losses, loss = tr.step(dev, host)
    torch.cuda.synchronize(); print("step %d: %.1f ms  loss %.4f" % (i, (time.perf_counter() - t0) * 1e3, float(loss)), flush=True)
