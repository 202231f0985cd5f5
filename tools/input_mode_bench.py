"""Measurement aid: the top-down captioner's att_input_mode 'both', 'featmap' and 'dual_region' at B=100 clips, T=10 and T=480 frames.

For each (T, mode) it times the prologue (gvd_prologue_fwd) and the 20-step greedy loop (gvd_decode_greedy, graph replay) with CUDA events,
and prints the loop's tokens/s and the feature bytes the decode attention reads per clip and step (from the shapes, fp32 features only,
no state or weights: 'both' reads p_pool, pool_feats, p_conv and conv_feats; 'featmap' skips pool_feats; 'dual_region' reads p_pool and
pool_feats once for both of its attentions and no frame features).  The modes alternate inside each round so that drift of the shared machine
hits both alike.  Prints the card's name and power limit with the numbers.
Usage: python tools/input_mode_bench.py [rounds (default 3)]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B = 100
MODES = ("both", "featmap", "dual_region")
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


def attn_bytes(opt, T, mode):
    """fp32 feature bytes the decode attention streams per clip and step."""
    R, A, H = opt.num_sampled_frm * opt.num_prop_per_frm, opt.att_hid_size, opt.rnn_size
    region = R * (A + (0 if mode == "featmap" else H))
    return 4 * (region + (0 if mode == "dual_region" else T * (A + H)))


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, out


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    if not torch.cuda.is_available():
        raise SystemExit("input_mode_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip().splitlines()[0] if q.stdout else "n/a"), flush=True)
    for T in (10, 480):
        setups = {}
        for mode in MODES:
            opt = synth.make_opt(t_attn_size=T, att_input_mode=mode)
            nm = capi.NativeModel(opt)
            nm.load_state_dict(synth.make_state_dict(opt))
            inp = synth.make_inputs(opt, B, masked=False)
            dev = {k: inp[k].cuda() for k in KEYS}
            setups[mode] = (opt, nm, dev)
        res = {m: dict(pro=[], loop=[]) for m in MODES}
        for r in range(rounds + 1):                          # round 0 warms every shape up
            for mode in MODES:
                opt, nm, dev = setups[mode]
                pro, _ = timed(lambda: nm.prologue(*(dev[k] for k in KEYS)), 5)
                loop, out = timed(lambda: nm.decode_greedy(B, T, dev["pnt_mask"]), 10)
                if r:
                    res[mode]["pro"].append(pro)
                    res[mode]["loop"].append(loop)
        for mode in MODES:
            opt = setups[mode][0]
            pro, loop = min(res[mode]["pro"]), min(res[mode]["loop"])
            spread = max(res[mode]["loop"]) / loop - 1
            toks = B * opt.seq_length / (loop * 1e-3)
            print("T=%3d %-8s prologue %7.3f ms  loop %7.3f ms (%5.1f us/step, spread %.1f%%)  %8.0f tok/s  attention reads %.3f MB/clip-step"
                  % (T, mode, pro, loop, loop / opt.seq_length * 1e3, 100 * spread, toks, attn_bytes(opt, T, mode) / 1e6), flush=True)


if __name__ == "__main__":
    main()
