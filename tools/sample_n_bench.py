"""n sampled captions per clip (gvd_decode_sample_n) against the batch repeated n times (gvd_decode_sample on repeat_interleave(n)), the
two decode attention kernels on shared clip features, and the beam loop; full model dims, default backend.

  --part sample   prologue + loop, CUDA events, the two forms alternating, median of --reps, at (B clips, n) x T; also whether the outputs
                  are bit-identical (the prologue at n times the clips may differ in the last bits)
  --part profile  the decode attention launches alone under torch.profiler (a run of its own): time per launch, and the feature bytes
                  of the distinct clips it attends over (sample_n: B clips, read by their n rows; repeated: B * n clip copies)
  --part paths    the decode attention launch alone through gvd_op_attention_path: per-row kernel (path 0, what the decode runs) against
                  the row-grouped kernel (path 1) on the same clip features, n rows per clip, the decode's chunking; CUDA events around 20
                  launches, paths alternating, median of --reps
  --part beam     gvd_beam_decode at B = 100, K = 3 / 5 (median loop time of --reps); --dump DIR stores seq, log-probs, region indices and
                  the att2 logits of gvd_beam_decode_att2 at K = 3.  Calls only entry points older than gvd_decode_sample_n, so --root can
                  point at a build of another tree (e.g. the parent commit) for an output and timing comparison.
Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))


def _card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _model(T, seed=1):
    from gvd_b200 import synth
    from gvd_b200.misc.AttModel import TopDownModel
    opt = synth.make_opt(t_attn_size=T)
    sd = synth.make_state_dict(opt, seed=seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    m.load_state_dict(sd)
    return opt, m.cuda().eval()


KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


def _inputs(opt, B, seed=7):
    from gvd_b200 import synth
    return {k: v.cuda() for k, v in synth.make_inputs(opt, B, seed=seed).items()}


def _time(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _median(x):
    x = sorted(x)
    return x[len(x) // 2]


def part_sample(args, card):
    import torch
    for T in args.T:
        opt, model = _model(T)
        nm = model._native_model()
        for B, n in args.Bn:
            inp = _inputs(opt, B)
            rep = {k: v.repeat_interleave(n, 0).contiguous() for k, v in inp.items()}

            def grouped():
                nm.prologue(*(inp[k] for k in KEYS), rows=n)
                return nm.decode_sample_n(B, T, n, inp["pnt_mask"], 11, 1.0)

            def repeated():
                nm.prologue(*(rep[k] for k in KEYS))
                return nm.decode_sample(B * n, T, rep["pnt_mask"], 11, 1.0)

            out = {}
            for name, fn in (("sample_n", grouped), ("repeated", repeated)):
                for _ in range(args.warmup):
                    fn()
                out[name] = [o.cpu() for o in fn()]
            same = all(torch.equal(x, y) for x, y in zip(out["sample_n"], out["repeated"]))
            ts = {"sample_n": [], "repeated": []}
            for _ in range(args.reps):
                for name, fn in (("sample_n", grouped), ("repeated", repeated)):
                    ts[name].append(_time(fn))
            print(json.dumps(dict(part="sample", B=B, n=n, T=T, rows=B * n, ms_sample_n=round(_median(ts["sample_n"]), 3),
                                  ms_repeated=round(_median(ts["repeated"]), 3), bit_identical=same, reps=args.reps, **card)), flush=True)
        del model, nm
        torch.cuda.empty_cache()


def _feature_bytes(opt, clips, reads_per_clip, T):
    R = opt.num_sampled_frm * opt.num_prop_per_frm
    A, H = opt.att_hid_size, opt.rnn_size
    return clips * reads_per_clip * (R + T) * (A + H) * 4


def part_profile(args, card):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for T in args.T:
        opt, model = _model(T)
        nm = model._native_model()
        for B, n in args.Bn:
            inp = _inputs(opt, B)
            rep = {k: v.repeat_interleave(n, 0).contiguous() for k, v in inp.items()}
            runs = (("sample_n", lambda: (nm.prologue(*(inp[k] for k in KEYS), rows=n), lambda: nm.decode_sample_n(B, T, n, inp["pnt_mask"], 3, 1.0))),
                    ("repeated", lambda: (nm.prologue(*(rep[k] for k in KEYS)), lambda: nm.decode_sample(B * n, T, rep["pnt_mask"], 3, 1.0))))
            for name, setup in runs:
                _, loop = setup()
                loop()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.reps):
                        loop()
                    torch.cuda.synchronize()
                us, calls = 0.0, 0
                for e in prof.key_averages():
                    if "attn_partial_kernel" in e.key:
                        us += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                        calls += e.count
                per = us / max(calls, 1)
                nbytes = _feature_bytes(opt, B, 1 if name == "sample_n" else n, T)
                print(json.dumps(dict(part="profile", kind=name, B=B, n=n, T=T, attn_launches=calls, attn_us_per_launch=round(per, 2),
                                      distinct_feature_bytes=nbytes, **card)), flush=True)
        del model, nm
        torch.cuda.empty_cache()


def part_paths(args, card):
    import torch
    from gvd_b200 import capi
    A, H, R = 512, 1024, 1000
    g = torch.Generator().manual_seed(0)
    for T in args.T:
        for clips, n in args.Bn:
            rows = clips * n
            target = max(1, -(-592 // rows))                  # attn_chunking of the decode at `rows` rows
            pick = lambda N: min(128, max(16, (-(-N // target) + 7) // 8 * 8))
            RC, TC = pick(R), pick(T)
            c = lambda t: t.cuda().contiguous()
            p_pool, pool = c(torch.randn(clips, R, A, generator=g)), c(torch.randn(clips, R, H, generator=g))
            p_conv, conv = c(torch.randn(clips, T, A, generator=g)), c(torch.randn(clips, T, H, generator=g))
            w = c(torch.randn(A, generator=g) / A ** 0.5)
            b = c(torch.zeros(1))
            mask = c(torch.zeros(clips, R + 1, dtype=torch.uint8))
            q = c(torch.randn(rows, 2 * A, generator=g))
            z, x = c(torch.empty(rows, R)), c(torch.empty(rows, H))
            part = c(torch.empty(rows, -(-R // RC) + -(-T // TC), H + 4))
            ticket = c(torch.zeros(rows, dtype=torch.int32))

            def launch(path, k=20):
                for _ in range(k):
                    capi.op_attention(p_pool, pool, p_conv, conv, w, b, w, b, mask, mask, z, part, x, RC, TC, q=q, ticket=ticket,
                                      feat_div=n, att_input_mode="both", region_attn_mode="mix", path=path)

            for p in (0, 1):
                launch(p, 3)
            ts = {0: [], 1: []}
            for _ in range(args.reps):
                for p in (0, 1):
                    ts[p].append(_time(lambda: launch(p)) / 20 * 1e3)
            print(json.dumps(dict(part="paths", clips=clips, n=n, rows=rows, T=T, RC=RC, TC=TC, us_per_row=round(_median(ts[0]), 1),
                                  us_row_groups=round(_median(ts[1]), 1), spread_per_row=[round(min(ts[0]), 1), round(max(ts[0]), 1)],
                                  spread_row_groups=[round(min(ts[1]), 1), round(max(ts[1]), 1)], reps=args.reps, **card)), flush=True)


def part_beam(args, card):
    import numpy as np
    import torch
    B = 100
    for T in args.T:
        opt, model = _model(T)
        nm = model._native_model()
        inp = _inputs(opt, B)
        for K in (3, 5):
            nm.prologue(*(inp[k] for k in KEYS), beam=K, att2=K == 3)
            for _ in range(args.warmup):
                nm.beam_decode(B, T, K, inp["pnt_mask"])
            ts = [_time(lambda: nm.beam_decode(B, T, K, inp["pnt_mask"])) for _ in range(args.reps)]
            if K == 3 and args.dump:
                seq, logp, att, att2 = nm.beam_decode_att2(B, T, K, inp["pnt_mask"])
                os.makedirs(args.dump, exist_ok=True)
                np.savez(os.path.join(args.dump, "beam_K3_T%d.npz" % T), seq=seq.cpu().numpy(), logp=logp.cpu().numpy(), att=att.cpu().numpy(),
                         att2=att2.cpu().numpy())
            print(json.dumps(dict(part="beam", B=B, K=K, T=T, ms_beam_loop=round(_median(ts), 3), reps=args.reps, root=args.root, **card)),
                  flush=True)
        del model, nm
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--part", choices=["sample", "profile", "paths", "beam"], required=True)
    ap.add_argument("--root", default=os.path.dirname(HERE), help="tree whose gvd_b200 package and built library are loaded")
    ap.add_argument("--dump", default=None, help="beam part: directory for the K = 3 outputs")
    ap.add_argument("--T", type=int, nargs="+", default=[10, 480])
    ap.add_argument("--Bn", type=lambda s: tuple(int(v) for v in s.split(",")), nargs="+", default=[(20, 5), (100, 3)],
                    help="B,n pairs")
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    if not torch.cuda.is_available():
        sys.exit("sample_n_bench needs a CUDA device")
    card = _card()
    {"sample": part_sample, "profile": part_profile, "paths": part_paths, "beam": part_beam}[args.part](args, card)


if __name__ == "__main__":
    main()
