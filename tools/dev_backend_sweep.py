"""Step time and stage times of the B=100, T=10 greedy decode under the backend switches
(+8 = operand-swapped split-K decode products), plus token equality with
the default.  Usage: python tools/dev_backend_sweep.py 3 11 923"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import capi, synth
import os
B, T = 100, int(os.environ.get("GVD_SWEEP_T", "10"))
opt = synth.make_opt(t_attn_size=T); sd = synth.make_state_dict(opt)
nm = capi.NativeModel(opt); nm.load_state_dict(sd)
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
def devstep():
    nm.prologue(*(dev[k] for k in keys)); return nm.decode_greedy(B, T, dev["pnt_mask"])
ref = None
for be in [int(a) for a in sys.argv[1:]] or [3]:
    capi.set_backend(be)
    try:
        out = devstep(); devstep(); torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(4): devstep()
        torch.cuda.synchronize(); ms = (time.perf_counter() - t0) / 4 * 1e3
        capi.profile_enable(1); capi.profile_reset(); devstep(); torch.cuda.synchronize()
        pr = capi.profile_read(); capi.profile_enable(0)
    except Exception as e:
        print("backend", be, "FAILED:", e, flush=True); continue
    if ref is None: ref = out
    loop = sum(v[0] for k, v in pr.items() if k.startswith("decode.") and k != "decode.pre_att")
    print("backend %2d  step %.2f ms  decode loop %.2f ms  seq==default %s  att2 maxdiff %.2e" % (be, ms, loop, torch.equal(out[0], ref[0]), float((out[2] - ref[2]).abs().max())), flush=True)
    for k, v in sorted(pr.items(), key=lambda kv: -kv[1][0])[:14]: print("      %-24s %8.3f ms %5d" % (k, v[0], v[1]))
