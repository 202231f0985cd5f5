"""The CPU oracle (oracle/gvd_oracle.py) for the top-down captioner's region_attn_mode 'mix_mul' and 'dp' (AttModel.py:56-108).

The mode changes one line of Attention2.forward, the score of proposal r against the query q = h2att(h_att):
    'mix'     z_r = w . tanh(p_r + q) + b          (oracle/gvd_oracle.py, tests/input_mode_oracle.py)
    'mix_mul' z_r = w . tanh(p_r * q) + b          (same parameters)
    'dp'      z_r = p_r . q                        (Attention2 has no alpha_net)
It applies to attention2 and, in att_input_mode 'dual_region', to attention2_dual.  The temporal attention is additive in every mode and the
grounding is unchanged.

Every loop of the oracle (greedy, beam, teacher-forced, training step) reaches the decode step through the module attribute
``gvd_oracle.core_step``; ``oracle_modes(opt)`` puts the step of (opt.att_input_mode, opt.region_attn_mode) there for the duration of a call,
so that ``O.train_step`` (autograd over the oracle) is the training reference.  ``RegionAttnRefOps`` adds the torch definition of the new
training primitive (att_scores_mul / att_scores_mul_bwd) to the primitive mock of tests/ops_ref.py."""
import contextlib

import torch

import gvd_oracle as O
from ops_ref import TorchRefOps


def region_scores(W, prefix, p, q, form):
    """Attention2's scores (AttModel.py:79-96) of the projected rows p [B, N, A] against q [B, A], before masking."""
    if form == "dp":
        return torch.matmul(p, q.unsqueeze(2)).squeeze(2)
    x = p * q.unsqueeze(1) if form == "mix_mul" else p + q.unsqueeze(1)
    return torch.tanh(x) @ W[prefix + ".alpha_net.weight"].view(-1) + W[prefix + ".alpha_net.bias"]


def _region_attention(W, prefix, h_att, feats, att_mask, form):
    q = O._lin(h_att, W, prefix + ".h2att")
    z = region_scores(W, prefix, feats["p_pool_feats"], q, form)
    z = z.masked_fill(att_mask[:, 1:].bool(), O.MIN_VALUE)
    return torch.einsum("br,brh->bh", torch.softmax(z, dim=1), feats["pool_feats"]), z, q


def _temporal_attention(W, h_att, feats):
    q1 = O._lin(h_att, W, "core.attention.h2att")
    s = torch.tanh(feats["p_conv_feats"] + q1.unsqueeze(1)) @ W["core.attention.alpha_net.weight"].view(-1) + W["core.attention.alpha_net.bias"]
    return torch.einsum("bt,bth->bh", torch.softmax(s, dim=1), feats["conv_feats"])


def make_core_step(att_input_mode, form):
    """TopDownCore.forward (AttModel.py:134-164) for one (att_input_mode, region_attn_mode) pair."""
    def core_step(W, xt, feats, att_mask, pnt_mask, state):
        h, c = state
        h_att, c_att = O._lstm_cell(torch.cat((feats["fc_feats"], xt), dim=1), h[0], c[0], W, "core.att_lstm")
        att2, z, q2 = _region_attention(W, "core.attention2", h_att, feats, att_mask, form)
        if att_input_mode == "dual_region":
            att2_dual, _, _ = _region_attention(W, "core.attention2_dual", h_att, feats, att_mask, form)
            g = torch.sigmoid(O._lin(h_att, W, "core.dual_pointer.0"))
            x = g * att2 + (1 - g) * att2_dual
        else:
            att = _temporal_attention(W, h_att, feats)
            x = att if att_input_mode == "featmap" else att + att2
        z_out = z.masked_fill(pnt_mask[:, 1:].bool(), O.MIN_VALUE)
        h_lang, c_lang = O._lstm_cell(torch.cat((x, h_att), dim=1), h[1], c[1], W, "core.lang_lstm")
        return h_lang, (torch.stack((h_att, h_lang)), torch.stack((c_att, c_lang))), z_out, q2
    return core_step


STEPS = {(m, f): make_core_step(m, f) for m in ("both", "featmap", "dual_region") for f in ("mix", "mix_mul", "dp")}


@contextlib.contextmanager
def oracle_modes(opt):
    orig = O.core_step
    O.core_step = STEPS[(getattr(opt, "att_input_mode", "both"), getattr(opt, "region_attn_mode", "mix"))]
    try:
        yield O
    finally:
        O.core_step = orig


class RegionAttnRefOps(TorchRefOps):
    """tests/ops_ref.py's primitive mock plus the multiplicative scores of 'mix_mul'."""

    def att_scores_mul(self, p, q, w, b):
        assert p.dim() == 3 and q.shape == (p.shape[0], p.shape[2]) and w.numel() == p.shape[2] and b.numel() == 1
        return torch.tanh(p * q.unsqueeze(1)) @ w.reshape(-1) + b.reshape(())

    def att_scores_mul_bwd(self, ds, p, q, w):
        t = torch.tanh(p * q.unsqueeze(1))
        dpre = ds.unsqueeze(2) * w.reshape(1, 1, -1) * (1 - t * t)
        return dpre * q.unsqueeze(1), (dpre * p).sum(1), torch.einsum("bn,bna->a", ds, t), ds.sum().reshape(1)
