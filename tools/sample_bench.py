"""Measurement aid: the decode loop alone with greedy picking (gvd_decode_greedy) and with multinomial sampling at temperature 1.0
(gvd_decode_sample), both through their captured graphs, at B = 100 clips, T = 10 frames, default backend, after one prologue.
The two modes alternate so that both see the same state of a shared GPU; CUDA events bracket the loop call only.  Greedy token ids must be
identical across all alternations (the sampling graph shares the workspace with the greedy one).  Prints the card and its power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B, T, ROUNDS = 100, 10, 20
assert torch.cuda.is_available(), "sample_bench measures on a CUDA device"
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
opt = synth.make_opt(t_attn_size=T)
nm = capi.NativeModel(opt)
nm.load_state_dict(synth.make_state_dict(opt))
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
nm.prologue(*(dev[k] for k in keys))
L = opt.seq_length
modes = {"greedy": lambda i: nm.decode_greedy(B, T, dev["pnt_mask"]),
         "sample": lambda i: nm.decode_sample(B, T, dev["pnt_mask"], 1000 + i, 1.0)}
for fn in modes.values():                                   # capture both graphs, warm up
    for i in range(3):
        fn(i)
torch.cuda.synchronize()
ms = {m: [] for m in modes}
greedy_tokens, distinct = None, set()
for i in range(ROUNDS):
    for m, fn in modes.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        seq, _, _ = fn(i)
        e1.record()
        torch.cuda.synchronize()
        ms[m].append(e0.elapsed_time(e1))
        if m == "greedy":
            if greedy_tokens is None:
                greedy_tokens = seq.clone()
            assert torch.equal(seq, greedy_tokens), "greedy tokens changed between alternations"
        else:
            distinct.add(int(seq.sum()))
print("card, power limit: %s" % card)
for m, v in ms.items():
    v = sorted(v)
    print("%-6s B=%d T=%d L=%d: loop median %.3f ms (min %.3f, max %.3f) = %.1f us per decode step over %d calls" % (
        m, B, T, L, v[len(v) // 2], v[0], v[-1], v[len(v) // 2] / L * 1e3, len(v)))
print("greedy tokens identical across %d alternations; %d distinct sampled token checksums over %d seeds" % (ROUNDS, len(distinct), ROUNDS))
