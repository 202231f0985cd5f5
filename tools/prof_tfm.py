"""Profiling aid: B=100, T=10 prologue once, then the transformer captioner's greedy decode (gvd_tfm_decode_greedy) argv[1] times."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gvd_b200 import capi, synth
B, T = 100, 10
opt = synth.make_opt(t_attn_size=T, att_model="transformer"); sd = synth.make_state_dict(opt)
nm = capi.NativeModel(opt); nm.load_state_dict(sd)
cap = capi.TransformerCaptioner(opt.rnn_size, opt.vocab_size, opt.seq_length); cap.load_state_dict(sd)
inp = synth.make_inputs(opt, B, masked=False)
keys = ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")
dev = {k: inp[k].cuda() for k in keys}
nm.prologue(*(dev[k] for k in keys))
e0 = nm.workspace_tensor(B, T, "conv_feats", (B, T, opt.rnn_size)); e1 = nm.workspace_tensor(B, T, "pool_feats", (B, nm.R, opt.rnn_size))
for _ in range(int(sys.argv[1]) if len(sys.argv) > 1 else 2):
    cap.decode_greedy(e0, e1)
torch.cuda.synchronize()
print("done", capi.kernel_launches())
