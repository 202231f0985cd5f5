"""Measurement aid: the 20-step greedy loop alone (gvd_decode_greedy, graph replay) at B=100, default backend; argv[1] = T (default 10)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import capi, synth
B, T = 100, int(sys.argv[1]) if len(sys.argv) > 1 else 10
opt = synth.make_opt(t_attn_size=T); sd = synth.make_state_dict(opt)
nm = capi.NativeModel(opt); nm.load_state_dict(sd)
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for _ in range(2): nm.prologue(*(dev[k] for k in keys))
torch.cuda.synchronize(); e0.record()
for _ in range(5): nm.prologue(*(dev[k] for k in keys))
e1.record(); torch.cuda.synchronize()
pro = e0.elapsed_time(e1) / 5
for _ in range(3): out = nm.decode_greedy(B, T, dev["pnt_mask"])
torch.cuda.synchronize(); e0.record()
for _ in range(10): out = nm.decode_greedy(B, T, dev["pnt_mask"])
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 10
print("T=%d: prologue %.3f ms  loop %.3f ms (%.1f us/step)  tokens checksum %d" % (T, pro, ms, ms / 20 * 1e3, int(out[0].sum())), flush=True)
