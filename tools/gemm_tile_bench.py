"""Per-GEMM timing of the prologue's conversion-free fp16x3 GEMMs (ss_gemm_kernel) at B=100, T=10.

Runs the prologue a few times under torch.profiler (CUDA activities only, a run of its own), picks the ss_gemm_kernel launches whose
grid covers all B*R region rows, attributes them to the twelve operand-image GEMMs of one prologue
by launch order and prints per GEMM: kernel time (median over the profiled prologues), algorithmic TFLOP/s (2 M N K), issued fp16
TFLOP/s (three fp16 products per element pair, padded to whole 128 x 128 x 32 tiles) and the operand bytes every CTA streams from L2
((128 + 128) rows x 128 B per 32-wide K slice) over the kernel time.  The issued rate is
also given as a fraction of the data-sheet dense fp16 peak and of a ceiling measured in the same run: torch.matmul in fp16 (cuBLAS) at
the fc7 shape [100 000 x 2048] . [2048 x 2048]^T.  The card's name, power limit and max SM clock are printed in the same run.
argv: backend (default 923), profiled prologues (default 3)."""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

BM, BN, BK = 128, 128, 32
PEAK_F16 = 989e12           # H100 SXM data sheet, dense fp16 / bf16 at 700 W


def cdiv(a, b):
    return (a + b - 1) // b


def gemm_list(opt, B):
    """(name, M, N, K) of the operand-image GEMMs of one prologue, in launch order (gvd_api.cu: region_fwd / obj_interact_fwd)."""
    H, A, D = opt.rnn_size, opt.att_hid_size, opt.detect_size
    R = opt.num_sampled_frm * opt.num_prop_per_frm
    rup4 = lambda x: cdiv(x, 4) * 4
    HP = rup4(cdiv(H, 6)) * len(range(0, H, cdiv(H, 6)))
    M = B * R
    g = [("region.fc7", M, 2048, opt.att_feat_size), ("region.sim_gemm", M, D + 1, 2048),
         ("region.pool_embed", M, H, rup4(opt.att_feat_size + 300 + D + 1))]
    for l in range(2):
        g += [("interact.qkv_proj.%d" % l, M, 3 * HP, H), ("interact.wo.%d" % l, M, H, HP),
              ("interact.ffn1.%d" % l, M, H // 2, H), ("interact.ffn2.%d" % l, M, H, H // 2)]
    g.append(("region.ctx2pool", M, A, H))
    return g


def counts(M, N, K):
    """algorithmic FLOP, issued fp16 MMA FLOP, operand bytes L2 -> SM of one launch"""
    gx, gy, nk = cdiv(N, BN), cdiv(M, BM), cdiv(K, BK)
    return 2.0 * M * N * K, 3 * 2.0 * (gy * BM) * (gx * BN) * (nk * BK), gy * gx * nk * (BM + BN) * 128.0


def cublas_ceiling(M=100000, N=2048, K=2048, reps=20):
    """dense fp16 TFLOP/s of torch.matmul (cuBLAS, fp32 accumulation) at the fc7 shape, CUDA events over reps launches"""
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(M, K, device="cuda", dtype=torch.float16, generator=g)
    w = torch.randn(N, K, device="cuda", dtype=torch.float16, generator=g)
    for _ in range(3):
        torch.matmul(a, w.t())
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        torch.matmul(a, w.t())
    t1.record()
    torch.cuda.synchronize()
    return 2.0 * M * N * K * reps / (t0.elapsed_time(t1) * 1e-3)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "nvidia-smi unavailable"
    return "%s (power limit, max SM clock: %s)" % (name, pl)


def main():
    be = int(sys.argv[1]) if len(sys.argv) > 1 else 923
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    assert torch.cuda.is_available(), "gemm_tile_bench needs a CUDA device"
    B, T = 100, 10
    opt = synth.make_opt(t_attn_size=T)
    sd = synth.make_state_dict(opt)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    capi.set_backend(be)
    inp = synth.make_inputs(opt, B, masked=False)
    keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
    dev = {k: inp[k].cuda() for k in keys}
    for _ in range(2):
        nm.prologue(*(dev[k] for k in keys))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            nm.prologue(*(dev[k] for k in keys))
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]

    gemms = gemm_list(opt, B)
    M = gemms[0][1]
    launches = sorted((e for e in events if e.get("cat") == "kernel" and "ss_gemm_kernel" in e.get("name", "")
                       and list(e.get("args", {}).get("grid", [0, 0, 0]))[1:] == [cdiv(M, BM), 1]), key=lambda e: e["ts"])
    if len(launches) != len(gemms) * iters:
        raise SystemExit("expected %d full-height ss_gemm_kernel launches, found %d" % (len(gemms) * iters, len(launches)))
    ceil = cublas_ceiling()
    print("card:", card())
    print("backend %d, B=%d T=%d, %d profiled prologues, median kernel time per GEMM" % (be, B, T, iters))
    print("ceiling: torch.matmul fp16 (cuBLAS) [100000 x 2048] . [2048 x 2048]^T: %.1f TFLOP/s (%.2f of the %.0f TFLOP/s data sheet)"
          % (ceil * 1e-12, ceil / PEAK_F16, PEAK_F16 * 1e-12))
    print("%-20s %7s %5s %5s %9s %9s %9s %6s %6s %9s" % ("gemm", "M", "N", "K", "time_ms", "alg_TF/s", "f16_TF/s", "/ceil", "/sheet",
                                                        "L2_GB/s"))
    tot_t = tot_alg = tot_iss = tot_b = 0.0
    for j, (name, m, n, k) in enumerate(gemms):
        ev = [launches[i * len(gemms) + j] for i in range(iters)]
        gx = ev[0]["args"]["grid"][0]
        if gx != cdiv(n, BN):
            raise SystemExit("launch %d (%s): grid.x = %d, expected %d" % (j, name, gx, cdiv(n, BN)))
        t = sorted(e["dur"] for e in ev)[iters // 2] * 1e-6      # us -> s
        alg, iss, byt = counts(m, n, k)
        tot_t += t; tot_alg += alg; tot_iss += iss; tot_b += byt
        print("%-20s %7d %5d %5d %9.3f %9.1f %9.1f %6.2f %6.2f %9.0f" % (name, m, n, k, t * 1e3, alg / t * 1e-12, iss / t * 1e-12,
                                                                      iss / t / ceil, iss / t / PEAK_F16, byt / t * 1e-9))
    print("%-20s %26s %9.3f %9.1f %9.1f %6.2f %6.2f %9.0f" % ("all twelve", "", tot_t * 1e3, tot_alg / tot_t * 1e-12, tot_iss / tot_t * 1e-12,
                                                            tot_iss / tot_t / ceil, tot_iss / tot_t / PEAK_F16, tot_b / tot_t * 1e-9))
    print("totals: %.2f TFLOP algorithmic, %.2f TFLOP issued fp16, %.1f GB operands L2 -> SM" % (tot_alg * 1e-12, tot_iss * 1e-12, tot_b * 1e-9))


if __name__ == "__main__":
    main()
