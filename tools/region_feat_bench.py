"""Measurement aid: the top-down captioner with transfer_mode 'cls' and 'none' at B=100 clips, T=10 and T=480 frames, full model dims.

'none' only drops the class bias: the similarity GEMM's epilogue adds no bias row and the grounding adds no per-class term, so the expected
difference is nil (it saves R (D+1) adds per clip in the similarity, 43.2 M per batch of 100 at D = 431, R = 1000, of a 1.7 KB bias vector
that stays in cache).  For each (T, mode) it times the prologue (gvd_prologue_fwd, with the similarity matrix returned) and the 20-step
greedy loop (gvd_decode_greedy, graph replay) with CUDA events, alternating the modes inside each round so that drift of the shared machine
hits both alike.  Then the transformer captioner with att_input_mode 'region', without and with enable_BUTD: the prologue (no similarity
requested, as the captioner calls it) and the 20-step greedy decoder loop.  BUTD removes, per clip at R = 1000, D = 431, H = 1024: the
region-embedding row kernel (reads 2048 + 432 floats, writes the 2784-wide operand image per region), the similarity GEMM (2 R 2048 432 =
1.77 GFLOP) and its softmax, and shrinks pool_embed's K from 2784 (its operand image) to 2048 (2 R 1024 736 = 1.51 GFLOP fewer, and 736
fewer image columns per region to stream).  Prints the card's name and power limit with the numbers.
Usage: python tools/region_feat_bench.py [rounds (default 3)]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B = 100
MODES = ("cls", "none")
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


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
        raise SystemExit("region_feat_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip().splitlines()[0] if q.stdout else "n/a"), flush=True)
    for T in (10, 480):
        setups = {}
        for mode in MODES:
            opt = synth.make_opt(t_attn_size=T, transfer_mode=mode)
            nm = capi.NativeModel(opt)
            sd = synth.make_state_dict(opt)
            nm.load_state_dict(sd)
            inp = synth.make_inputs(opt, B, masked=False)
            setups[mode] = (nm, {k: inp[k].cuda() for k in KEYS})
        res = {m: dict(pro=[], loop=[]) for m in MODES}
        for r in range(rounds + 1):                          # round 0 warms every shape up
            for mode in MODES:
                nm, dev = setups[mode]
                pro, _ = timed(lambda: nm.prologue(*(dev[k] for k in KEYS)), 5)
                loop, _ = timed(lambda: nm.decode_greedy(B, T, dev["pnt_mask"]), 10)
                if r:
                    res[mode]["pro"].append(pro)
                    res[mode]["loop"].append(loop)
        for mode in MODES:
            p, l = res[mode]["pro"], res[mode]["loop"]
            print("T=%3d %-4s prologue %7.2f ms (min %7.2f, max %7.2f) | greedy loop %6.2f ms (min %6.2f, max %6.2f) | %.0f tokens/s"
                  % (T, mode, sum(p) / len(p), min(p), max(p), sum(l) / len(l), min(l), max(l), B * 20 / (min(l) / 1e3)), flush=True)
    transformer_region(rounds)


def transformer_region(rounds):
    for T in (10, 480):
        setups = {}
        for butd in (False, True):
            opt = synth.make_opt(t_attn_size=T, att_model="transformer", att_input_mode="region", enable_BUTD=butd)
            from gvd_b200.misc.AttModel import TopDownModel
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                m = TopDownModel(opt)
            m.load_state_dict(synth.make_state_dict(opt))
            m.cuda().eval()
            inp = synth.make_inputs(opt, B, masked=False)
            setups[butd] = (m, {k: inp[k].cuda() for k in KEYS})
        res = {b: dict(pro=[], loop=[]) for b in setups}
        for r in range(rounds + 1):
            for butd, (m, dev) in setups.items():
                nm = m._native_model()
                pro, _ = timed(lambda: nm.prologue(*(dev[k] for k in KEYS), want_sim=False), 5)
                enc = m._tfm_encodings(nm, B, T)
                loop, _ = timed(lambda: m._tfm.decode_greedy(*enc), 10)
                if r:
                    res[butd]["pro"].append(pro)
                    res[butd]["loop"].append(loop)
        for butd in setups:
            p, l = res[butd]["pro"], res[butd]["loop"]
            print("T=%3d transformer 'region' %-8s prologue %7.2f ms (min %7.2f, max %7.2f) | greedy loop %6.2f ms (min %6.2f, max %6.2f)"
                  % (T, "BUTD" if butd else "non-BUTD", sum(p) / len(p), min(p), max(p), sum(l) / len(l), min(l), max(l)), flush=True)


if __name__ == "__main__":
    main()
