"""Measurement aid: the cost of grounding beam-search captions.  The beam loop alone (gvd_beam_decode) against the grounded beam loop
(gvd_beam_decode_att2: every step's region logits written into the history, parents kept, one backtrack gather at the end) at B = 100 clips,
T = 10 and 480 frames, beam 3 and 5, default backend, after one prologue per (T, beam).  The two calls alternate so that both see the same
state of a shared GPU; CUDA events bracket the decode call only.  Tokens and log-probabilities must be bit-identical between the two.
Prints the card and its power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B, ROUNDS = 100, 15
assert torch.cuda.is_available(), "beam_att2_bench measures on a CUDA device"
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card, power limit: %s" % card)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
for T in (10, 480):
    opt = synth.make_opt(t_attn_size=T)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(synth.make_state_dict(opt))
    inp = synth.make_inputs(opt, B, masked=False)
    dev = {k: inp[k].cuda() for k in keys}
    L, R = opt.seq_length, nm.R
    for K in (3, 5):
        nm.prologue(*(dev[k] for k in keys), beam=K, att2=True)
        calls = {"plain": lambda: nm.beam_decode(B, T, K, dev["pnt_mask"]),
                 "att2": lambda: nm.beam_decode_att2(B, T, K, dev["pnt_mask"])}
        for fn in calls.values():                       # warm up
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        ms = {m: [] for m in calls}
        ref = None
        for _ in range(ROUNDS):
            for m, fn in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[m].append(e0.elapsed_time(e1))
                if ref is None:
                    ref = (out[0].clone(), out[1].clone())
                assert torch.equal(out[0], ref[0]) and torch.equal(out[1], ref[1]), "tokens / log-probs differ between the two calls"
        med = {m: sorted(v)[len(v) // 2] for m, v in ms.items()}
        hist_mb = L * B * K * R * 4 / 1e6
        for m, v in ms.items():
            v = sorted(v)
            print("B=%d T=%d K=%d %-5s: beam loop median %.3f ms (min %.3f, max %.3f) over %d calls" % (B, T, K, m, med[m], v[0], v[-1], len(v)))
        print("B=%d T=%d K=%d: grounding costs %+.3f ms (%+.2f%%); logit history %.1f MB" % (
            B, T, K, med["att2"] - med["plain"], 100.0 * (med["att2"] / med["plain"] - 1.0), hist_mb))
    del nm
    torch.cuda.empty_cache()
