"""Profiling aid: B=100 prologue (+ optional decode) once per iteration; argv: backend, T, iterations."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import capi, synth
be = int(sys.argv[1]) if len(sys.argv) > 1 else 27
T = int(sys.argv[2]) if len(sys.argv) > 2 else 10
it = int(sys.argv[3]) if len(sys.argv) > 3 else 2
B = 100
opt = synth.make_opt(t_attn_size=T); sd = synth.make_state_dict(opt)
nm = capi.NativeModel(opt); nm.load_state_dict(sd)
capi.set_backend(be)
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
for _ in range(it):
    nm.prologue(*(dev[k] for k in keys))
torch.cuda.synchronize()
print("done", capi.kernel_launches())
