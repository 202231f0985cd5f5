"""Measurement aid: the top-down captioner's att_input_mode 'both', 'featmap' and 'dual_region' (or, with the axis region_attn_mode, the
region attention's score 'mix', 'mix_mul' and 'dp' in att_input_mode 'both') at B=100 clips, T=10 and T=480 frames.

For each (T, mode) it times the prologue (gvd_prologue_fwd) and the 20-step greedy loop (gvd_decode_greedy, graph replay) with CUDA events,
and prints the loop's tokens/s and the feature bytes the decode attention reads per clip and step (from the shapes, fp32 features only,
no state or weights: 'both' reads p_pool, pool_feats, p_conv and conv_feats; 'featmap' skips pool_feats; 'dual_region' reads p_pool and
pool_feats once for both of its attentions and no frame features).  The modes alternate inside each round so that drift of the shared machine
hits both alike.  The region_attn_mode axis also times the decode attention launch on its own (gvd_op_attention_form at the decode step's
shapes and chunking, random features and queries, 50 launches per sample): the three forms read the same bytes, so what differs is the
phase-A arithmetic.  Prints the card's name and power limit with the numbers.
Usage: python tools/input_mode_bench.py [rounds (default 3)] [att_input_mode (default) | region_attn_mode]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B = 100
MODES = ("both", "featmap", "dual_region")
FORMS = ("mix", "mix_mul", "dp")
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


def attn_launch(opt, T, form):
    """A closure that launches the decode attention alone on the step's shapes (B rows, R proposals, T frames, the decode's chunking)."""
    R, A, H = opt.num_sampled_frm * opt.num_prop_per_frm, opt.att_hid_size, opt.rnn_size
    pick = lambda n: min(128, max(16, (-(-n // max(1, -(-592 // B))) + 7) // 8 * 8))      # attn_chunking (csrc/gvd_api.cu)
    RC, TC = pick(R), pick(T)
    g = torch.Generator().manual_seed(T)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.5).cuda()
    p_pool, pool, p_conv, conv, q = r(B, R, A), r(B, R, H), r(B, T, A), r(B, T, H), r(B, 2 * A)
    w1, b1, w2, b2 = r(A), r(1), r(A), r(1)
    mask = torch.zeros(B, R + 1, dtype=torch.uint8, device="cuda")
    z, x = torch.empty(B, R, device="cuda"), torch.empty(B, H, device="cuda")
    part = torch.empty(B, -(-R // RC) + -(-T // TC), H + 4, device="cuda")
    ticket = torch.zeros(B, dtype=torch.int32, device="cuda")
    dp = form == "dp"
    return lambda: capi.op_attention(p_pool, pool, p_conv, conv, w1, b1, None if dp else w2, None if dp else b2, mask, mask, z, part, x, RC, TC,
                                     q=q, ticket=ticket, region_attn_mode=form)


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    axis = sys.argv[2] if len(sys.argv) > 2 else "att_input_mode"
    if axis not in ("att_input_mode", "region_attn_mode"):
        raise SystemExit("axis: att_input_mode or region_attn_mode")
    if not torch.cuda.is_available():
        raise SystemExit("input_mode_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip().splitlines()[0] if q.stdout else "n/a"), flush=True)
    region = axis == "region_attn_mode"
    modes = FORMS if region else MODES
    for T in (10, 480):
        setups = {}
        for mode in modes:
            opt = synth.make_opt(t_attn_size=T, **({"region_attn_mode": mode} if region else {"att_input_mode": mode}))
            nm = capi.NativeModel(opt)
            nm.load_state_dict(synth.make_state_dict(opt))
            inp = synth.make_inputs(opt, B, masked=False)
            dev = {k: inp[k].cuda() for k in KEYS}
            setups[mode] = (opt, nm, dev, attn_launch(opt, T, mode) if region else None)
        res = {m: dict(pro=[], loop=[], attn=[]) for m in modes}
        for r in range(rounds + 1):                          # round 0 warms every shape up
            for mode in modes:
                opt, nm, dev, attn = setups[mode]
                pro, _ = timed(lambda: nm.prologue(*(dev[k] for k in KEYS)), 5)
                loop, out = timed(lambda: nm.decode_greedy(B, T, dev["pnt_mask"]), 10)
                if r:
                    res[mode]["pro"].append(pro)
                    res[mode]["loop"].append(loop)
                if attn is not None:
                    a, _ = timed(attn, 50)
                    if r:
                        res[mode]["attn"].append(a)
        for mode in modes:
            opt = setups[mode][0]
            pro, loop = min(res[mode]["pro"]), min(res[mode]["loop"])
            spread = max(res[mode]["loop"]) / loop - 1
            toks = B * opt.seq_length / (loop * 1e-3)
            nbytes = attn_bytes(opt, T, "both" if region else mode)
            line = ("T=%3d %-8s prologue %7.3f ms  loop %7.3f ms (%5.1f us/step, spread %.1f%%)  %8.0f tok/s  attention reads %.3f MB/clip-step"
                    % (T, mode, pro, loop, loop / opt.seq_length * 1e3, 100 * spread, toks, nbytes / 1e6))
            if region:
                a = min(res[mode]["attn"])
                line += "  attention launch %6.1f us (%.2f TB/s)" % (a * 1e3, B * nbytes / (a * 1e-3) / 1e12)
            print(line, flush=True)


if __name__ == "__main__":
    main()
