"""Per-launch timing of the region encoder's fused self-attention kernel (self_attn_fused_kernel, csrc/gvd_attn.cu) at B=100, T=10.

Runs the prologue a few times under torch.profiler (CUDA activities only, a run of its own), takes every self_attn_fused_kernel launch
(two per prologue: one per encoder layer) and prints the kernel time per launch (median) with its rate: algorithmic TFLOP/s (Q K^T and
P.V at the real head sizes, 4 R^2 (nh hs) per clip) and issued fp16 TFLOP/s (three fp16 products per element pair over whole 128-row query
tiles, 32-key blocks, 176 head-dimension columns and the n176 P.V product).  The card's name and power limit are printed in the same run.
argv: profiled prologues (default 3)."""
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from gemm_tile_bench import card, cdiv  # noqa: E402
from gvd_b200 import capi, synth  # noqa: E402


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    assert torch.cuda.is_available(), "attn_kernel_bench needs a CUDA device"
    B, T = 100, 10
    opt = synth.make_opt(t_attn_size=T)
    sd = synth.make_state_dict(opt)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(sd)
    capi.set_backend(923)
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
    us = [e.device_time for e in prof.events() if "self_attn_fused_kernel" in e.name]
    assert len(us) == 2 * iters, "expected two launches per prologue, found %d" % len(us)
    H, R, nh = opt.rnn_size, opt.num_sampled_frm * opt.num_prop_per_frm, 6
    algo = B * 4.0 * R * R * H                                    # Q K^T + P.V over the 1024 real head columns
    issued = B * nh * 2 * 3 * 2.0 * (cdiv(R, 128) * 128) * (cdiv(R, 32) * 32) * 176
    ms = statistics.median(us) / 1e3
    print("card: %s" % card())
    print("self_attn_fused_kernel: %d launches, median %.3f ms per launch (min %.3f, max %.3f); %.1f TFLOP/s algorithmic, %.1f TFLOP/s issued fp16"
          % (len(us), ms, min(us) / 1e3, max(us) / 1e3, algo / (ms / 1e3) / 1e12, issued / (ms / 1e3) / 1e12))


if __name__ == "__main__":
    main()
