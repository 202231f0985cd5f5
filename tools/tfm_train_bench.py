"""One optimisation step of the transformer captioner (att_model = 'transformer', att_input_mode 'both', obj_interact on, full dims, T = 10)
at B = 100 on one GPU: the device step (TrainStep over NativeOps) with dropout off and on, the same step in eager PyTorch fp32 (the
specification tests/tfm_train_ref.tfm_train_step, TF32 off) as the baseline, and the decoder attention kernels (gvd_tr_mha_fwd / _bwd)
from a separate torch.profiler run, as achieved bytes/s against the bytes their shapes require.

    python tools/tfm_train_bench.py [--B 100] [--steps 7] [--warmup 2]

Prints the card and its power limit, then one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

import torch  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), ms


def mha_bytes(B, L, H, n_enc):
    """Algorithmic bytes of one step's decoder attention: per call the forward reads q, k, v and writes o (+ lse), the backward reads q, k,
    v, o, dO (+ lse) and writes dq, dk, dv; 2 layers x (self-attention over L keys, cross-attention over n_enc[l] keys)."""
    nh = 6
    fwd = bwd = 0
    for N in (L, n_enc[0], L, n_enc[1]):
        fwd += 4 * (2 * B * L * H + 2 * B * N * H + B * nh * L)
        bwd += 4 * (4 * B * L * H + 4 * B * N * H + B * nh * L)
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=100)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tfm_train_bench needs a CUDA device")
    import gvd_b200.synth as synth
    from gvd_b200.train import TrainStep
    from gvd_b200.train_ops import NativeOps
    from tfm_train_ref import tfm_train_step

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    print("card:", card)

    opt = synth.make_opt(t_attn_size=10, att_model="transformer")
    sd = synth.make_state_dict(opt, seed=0)
    inp = synth.make_inputs(opt, args.B, seed=11, masked=True, train=True)
    W = {k: v.cuda() for k, v in sd.items()}
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in inp.items()}
    ops = NativeOps()
    res = dict(workload="tfm_train_step", B=args.B, T=opt.t_attn_size, R=opt.num_sampled_frm * opt.num_prop_per_frm, L=opt.seq_length,
               H=opt.rnn_size, card=card)
    for name, drop in (("p0", None), ("dropout", dict(seed=1, p_lm=0.5, p_interact=0.2, p_gru=0.2, p_loc=0.5, p_tfm=0.2))):
        ts = TrainStep(ops, dropout=drop)
        med, ms = timed(lambda: ts.step(W, opt, dev, host=inp), args.steps, args.warmup)
        res["step_ms_" + name] = round(med, 2)
        res["step_ms_all_" + name] = [round(x, 2) for x in ms]
        print("device step (%s): median %.2f ms over %d steps" % (name, med, args.steps))

    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        med, ms = timed(lambda: tfm_train_step(W, opt, dev), max(5, args.steps // 2), 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    res["eager_fp32_step_ms"] = round(med, 2)
    print("eager PyTorch fp32 step (TF32 off): median %.2f ms" % med)

    ts = TrainStep(ops)
    ts.step(W, opt, dev, host=inp)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ts.step(W, opt, dev, host=inp)
        torch.cuda.synchronize()
    t = {"fwd": 0.0, "bwd": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "mha_fwd_kernel" in e.key:
            t["fwd"] += us
        elif "mha_bwd_kernel" in e.key:
            t["bwd"] += us
    fb, bb = mha_bytes(args.B, opt.seq_length, opt.rnn_size, (opt.t_attn_size, opt.num_sampled_frm * opt.num_prop_per_frm))
    for k, nbytes in (("fwd", fb), ("bwd", bb)):
        res["mha_%s_us" % k] = round(t[k], 1)
        res["mha_%s_GBps" % k] = round(nbytes / (t[k] * 1e-6) / 1e9, 1) if t[k] else None
        print("gvd_tr_mha_%s: %.1f us per step (4 launches), %.1f MB algorithmic, %s GB/s" % (k, t[k], nbytes / 1e6, res["mha_%s_GBps" % k]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
