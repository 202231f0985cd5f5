"""Measurement aid: decoding at growing vocabularies.  B = 100 clips, T = 10 frames, the full model dims, default backend.

Per vocabulary size V (4905, 6144: the register tails; 6145 and up: the sliced tail gvd_vocab_tail):
  * the 20-step greedy loop (gvd_decode_greedy) and the multinomial loop (gvd_decode_sample), both through their captured graphs, alternating,
    CUDA events around the loop call only;
  * with --profile, in a separate pass: the vocabulary head's launches alone (the split-K product of the logit weights and the tail on the
    same shapes as in the loop) under torch.profiler, their per-call kernel times, the head's algorithmic bytes per step
    (V (H + 1) 4 for the weights and bias + the partial planes written and read) and the achieved bandwidth.
--root DIR imports gvd_b200 from another checkout (a parent build, for an A/B comparison in alternating processes).
Prints the card name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--vocabs", type=int, nargs="+", default=[4905, 6144, 6145, 8192, 16384, 32000])
ap.add_argument("--rounds", type=int, default=10)
ap.add_argument("--greedy-only", action="store_true")
ap.add_argument("--profile", action="store_true")
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B, T = 100, 10
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
assert torch.cuda.is_available(), "vocab_bench measures on a CUDA device"
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def loops(V):
    opt = synth.make_opt(t_attn_size=T, vocab_size=V)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(synth.make_state_dict(opt))
    inp = synth.make_inputs(opt, B, masked=False)
    dev = {k: inp[k].cuda() for k in KEYS}
    nm.prologue(*(dev[k] for k in KEYS))
    modes = {"greedy": lambda i: nm.decode_greedy(B, T, dev["pnt_mask"])}
    if not args.greedy_only:
        modes["sample"] = lambda i: nm.decode_sample(B, T, dev["pnt_mask"], 1000 + i, 1.0)
    for fn in modes.values():
        for i in range(3):
            fn(i)
    torch.cuda.synchronize()
    ms = {m: [] for m in modes}
    tokens = None
    for i in range(args.rounds):
        for m, fn in modes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            seq = fn(i)[0]
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1))
            if m == "greedy":
                tokens = seq.clone() if tokens is None else tokens
                assert torch.equal(seq, tokens), "greedy tokens changed between calls"
    out = {m + "_loop_ms": sorted(v)[len(v) // 2] for m, v in ms.items()}
    out.update({m + "_loop_ms_min": min(v) for m, v in ms.items()})
    out["greedy_token_checksum"] = int(tokens.sum())
    del nm
    torch.cuda.empty_cache()
    return out, opt


def head(V, opt):
    """The head's product and tail on the loop's shapes, kernel times from torch.profiler (one call = one decode step's head)."""
    H = opt.rnn_size
    g = torch.Generator().manual_seed(V)
    W = (torch.randn(V, H, generator=g) * 0.03).cuda()
    bias = torch.randn(V, generator=g).cuda()
    X = torch.randn(B, H, generator=g).cuda()
    ldp = (V + 3) // 4 * 4
    it = torch.zeros(B, dtype=torch.int64, device="cuda")
    S = int(capi.lib().gvd_plan_skinny_splits(V, H, B))

    def step():
        part = capi.op_skinny_partials(W, X, S=S, f16_images=1, ldp=ldp) if S > 0 else None
        if part is None:
            return 0
        if V <= 6144:
            capi.op_reduce_pick(part, bias, V, V - 1, it)
        else:
            capi.op_reduce_pick_split(part, bias, V, capi.VOCAB_GREEDY, it, unk=V - 1)
        return part.shape[0]

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    n = 20
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type is not None and "CUDA" in str(e.device_type) and e.count > 0:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            kern[e.key[:80]] = round(us / n, 2)
    prod = sum(v for k, v in kern.items() if "skinny" in k or "gemm" in k.lower())
    tail = sum(v for k, v in kern.items() if "reduce_pick" in k or "vocab_tail" in k)
    Vp = (V + 3) // 4 * 4
    nbytes = V * (H + 1) * 4 + 2 * S * B * Vp * 4
    return dict(splits=S, kernels_us_per_call=kern, product_us=round(prod, 2), tail_us=round(tail, 2),
                head_bytes_per_step=nbytes, head_TBps=round(nbytes / ((prod + tail) * 1e-6) / 1e12, 3) if prod + tail > 0 else None)


print("card, power limit: %s" % card)
print("gvd_b200 from %s" % os.path.abspath(args.root))
for V in args.vocabs:
    res, opt = loops(V)
    res["V"] = V
    if args.profile:
        res["head"] = head(V, opt)
    print(json.dumps(res), flush=True)
