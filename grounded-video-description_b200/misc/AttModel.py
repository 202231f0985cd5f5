"""``TopDownModel`` / ``TopDownCore`` (reference: misc/AttModel.py:22-176).

TopDownCore here only owns the decode-step parameters under the reference's key names
(``core.att_lstm.weight_ih`` ...); one decode step is the native sequence
lstm_step -> h2att GEMM -> attn_partial (TMA-fed) -> attn_combine -> lstm_step (csrc/gvd_decode.cu).
"""
import torch.nn as nn

try:
    from .model import AttModel
except ImportError:
    from misc.model import AttModel


class _AttentionParams(nn.Module):
    """h2att + alpha_net of Attention / Attention2 (AttModel.py:22-31, 56-68).  alpha_net=False: Attention2 in region_attn_mode 'dp' (a
    plain dot product p . q, AttModel.py:62-65,95-96), which has no alpha_net."""

    def __init__(self, opt, alpha_net=True):
        super().__init__()
        self.h2att = nn.Linear(opt.rnn_size, opt.att_hid_size)
        if alpha_net:
            self.alpha_net = nn.Linear(opt.att_hid_size, 1)


class TopDownCore(nn.Module):
    def __init__(self, opt, use_maxout=False):
        super().__init__()
        self.att_lstm = nn.LSTMCell(opt.input_encoding_size + opt.rnn_size, opt.rnn_size)
        self.lang_lstm = nn.LSTMCell(opt.rnn_size * 2, opt.rnn_size)
        self.attention = _AttentionParams(opt)
        region_alpha = getattr(opt, "region_attn_mode", "mix") != "dp"
        self.attention2 = _AttentionParams(opt, region_alpha)
        if opt.att_input_mode == "dual_region":                 # AttModel.py:126-128
            self.attention2_dual = _AttentionParams(opt, region_alpha)
            self.dual_pointer = nn.Sequential(nn.Linear(opt.rnn_size, 1), nn.Sigmoid())
        # present in every reference checkpoint, never used by forward (AttModel.py:130-131)
        self.i2h_2 = nn.Linear(opt.rnn_size * 2, opt.rnn_size)
        self.h2h_2 = nn.Linear(opt.rnn_size, opt.rnn_size)

    def forward(self, *args):
        raise RuntimeError("TopDownCore has no stand-alone torch path; use gvd_decode_step_fwd via the model")


class TopDownModel(AttModel):
    def __init__(self, opt):
        super().__init__(opt)
        self.num_layers = 2
        self.core = TopDownCore(opt)
