"""Profiling aid: B=100, T=10 prologue once, then the greedy loop a few times (kernel-by-kernel with GVD_NO_GRAPH=1).  argv[1] = backend flags."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import capi, synth
be = int(sys.argv[1]) if len(sys.argv) > 1 else 3
B, T = 100, 10
opt = synth.make_opt(t_attn_size=T); sd = synth.make_state_dict(opt)
nm = capi.NativeModel(opt); nm.load_state_dict(sd)
capi.set_backend(be)
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
nm.prologue(*(dev[k] for k in keys))
for _ in range(int(sys.argv[2]) if len(sys.argv) > 2 else 3):
    nm.decode_greedy(B, T, dev["pnt_mask"])
torch.cuda.synchronize()
print("done", capi.kernel_launches())
