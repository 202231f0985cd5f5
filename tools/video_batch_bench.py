"""Measurement aid: a video-indexed batch (frame features once per video, eval_opt['video_idx']) against the per-clip batch that carries a
copy of its video's frames per event, at the reference's inference shape: B = 100 events, T = 480 frames (opts.py:50), full model dims.

For V = 100 videos (one event each: nothing is shared) and V = 28 (~3.5 events per video, as in ActivityNet Captions) it times, with CUDA
events, the prologue (gvd_prologue_fwd vs gvd_prologue_fwd_video), the 20-step greedy loop (graph replay) and the host-buffer entry point end
to end (pinned inputs: H2D, prologue, loop, D2H).  The two paths alternate inside each round so that drift of the shared machine hits both
alike; the minimum over the rounds is printed with the spread.  It also prints, from the shapes and windows, the frame bytes that cross PCIe
and the frame-feature bytes the decode attention streams per step (p_conv + conv rows, fp32), and the card's name and power limit.
Usage: python tools/video_batch_bench.py [rounds (default 3)]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gvd_b200 import capi, synth  # noqa: E402

B, T = 100, 480
KEYS = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")


def frame_h2d_bytes(B, V, T, F):
    """Frame-feature bytes the host-buffer entry point copies: one [T, F] fp32 block per video (V), or per clip (V = None)."""
    return (V if V else B) * T * F * 4


def temporal_attn_bytes(win, T, A, H, video):
    """fp32 frame-feature bytes (p_conv and conv rows) the decode attention streams per step for clips with windows win [B, 2]: every row of
    every clip's copy, or only the rows inside each window of the video's features."""
    if not video:
        return win.shape[0] * T * (A + H) * 4
    n_in = (torch.clamp(win[:, 1], max=T) - torch.clamp(win[:, 0], min=0)).clamp(min=0)
    return int(n_in.sum()) * (A + H) * 4


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
        raise SystemExit("video_batch_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q.stdout.strip().splitlines()[0] if q.stdout else "n/a"), flush=True)
    opt = synth.make_opt(t_attn_size=T)
    nm = capi.NativeModel(opt)
    nm.load_state_dict(synth.make_state_dict(opt))
    for V in (100, 28):
        inp = synth.make_video_inputs(opt, B, V, masked=False)
        clip = dict(inp, segs_feat=inp["segs_feat"][inp["video_idx"]].contiguous())
        dev = {"video": {k: v.cuda() for k, v in inp.items()}, "clip": {k: v.cuda() for k, v in clip.items()}}
        host = {"video": {k: v.pin_memory() for k, v in inp.items()}, "clip": {k: v.pin_memory() for k, v in clip.items()}}
        vid = {"video": dev["video"]["video_idx"], "clip": None}
        hvid = {"video": host["video"]["video_idx"], "clip": None}
        res = {p: dict(pro=[], loop=[], host=[]) for p in ("clip", "video")}
        outs = {}
        for r in range(rounds + 1):                          # round 0 warms every shape up
            for p in ("clip", "video"):
                d = dev[p]
                pro, _ = timed(lambda: nm.prologue(*(d[k] for k in KEYS), video_idx=vid[p]), 3)
                loop, out = timed(lambda: nm.decode_greedy(B, T, d["pnt_mask"]), 5)
                e2e, _ = timed(lambda: nm.sample_greedy_host(*(host[p][k] for k in KEYS), video_idx=hvid[p]), 2)
                outs[p] = out[0].cpu()
                if r:
                    res[p]["pro"].append(pro)
                    res[p]["loop"].append(loop)
                    res[p]["host"].append(e2e)
        same = torch.equal(outs["clip"], outs["video"])
        print("B=%d events, V=%d videos, T=%d: greedy tokens of the two paths equal: %s" % (B, V, T, same), flush=True)
        for p in ("clip", "video"):
            h2d = frame_h2d_bytes(B, V if p == "video" else None, T, opt.fc_feat_size)
            att = temporal_attn_bytes(inp["sample_idx"], T, opt.att_hid_size, opt.rnn_size, p == "video")
            line = "  %-5s" % p
            for k, name in (("pro", "prologue"), ("loop", "greedy loop"), ("host", "host-buffer e2e")):
                v = res[p][k]
                line += "  %s %8.3f ms (spread %4.1f%%)" % (name, min(v), 100 * (max(v) / min(v) - 1))
            print(line + "  | frame H2D %.1f MB, temporal attention %.1f MB/step" % (h2d / 1e6, att / 1e6), flush=True)


if __name__ == "__main__":
    main()
