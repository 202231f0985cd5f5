"""The CPU oracle (oracle/gvd_oracle.py) for the top-down captioner's att_input_mode 'featmap' and 'dual_region' (AttModel.py:126-156).

'featmap' changes one line of TopDownCore.forward: the language LSTM reads cat(att, h_att) instead of cat(att + att2, h_att).  The region
attention still runs for its masked logits (att2_weight: the returned attention weights, the grounding, the attention / grounding losses);
its weighted sum is discarded.  The prologue and the state_dict are those of 'both'.
'dual_region' has no temporal attention: a second region attention (attention2_dual) over the same features and masks, and the language LSTM
reads cat(g att2 + (1 - g) att2_dual, h_att) with g = sigmoid(dual_pointer(h_att)).  The oracle's prologue still computes the frame branch;
the step never reads it, so its parameters get no gradient, as in the reference.

Every loop of the oracle (greedy, beam, teacher-forced, training step) reaches the decode step through the module attribute
``gvd_oracle.core_step``; ``oracle_mode(opt)`` puts the step of ``opt.att_input_mode`` there for the duration of a call."""
import contextlib

import torch

import gvd_oracle as O


def core_step_featmap(W, xt, feats, att_mask, pnt_mask, state):
    h, c = state
    h_att, c_att = O._lstm_cell(torch.cat((feats["fc_feats"], xt), dim=1), h[0], c[0], W, "core.att_lstm")
    q1 = O._lin(h_att, W, "core.attention.h2att")
    s = torch.tanh(feats["p_conv_feats"] + q1.unsqueeze(1)) @ W["core.attention.alpha_net.weight"].view(-1) \
        + W["core.attention.alpha_net.bias"]
    att = torch.einsum("bt,bth->bh", torch.softmax(s, dim=1), feats["conv_feats"])
    q2 = O._lin(h_att, W, "core.attention2.h2att")
    z = torch.tanh(feats["p_pool_feats"] + q2.unsqueeze(1)) @ W["core.attention2.alpha_net.weight"].view(-1) \
        + W["core.attention2.alpha_net.bias"]
    z = z.masked_fill(att_mask[:, 1:].bool(), O.MIN_VALUE)
    z_out = z.masked_fill(pnt_mask[:, 1:].bool(), O.MIN_VALUE)
    h_lang, c_lang = O._lstm_cell(torch.cat((att, h_att), dim=1), h[1], c[1], W, "core.lang_lstm")
    return h_lang, (torch.stack((h_att, h_lang)), torch.stack((c_att, c_lang))), z_out, q2


def _region_attention(W, p, h_att, feats, att_mask):
    q = O._lin(h_att, W, p + ".h2att")
    z = torch.tanh(feats["p_pool_feats"] + q.unsqueeze(1)) @ W[p + ".alpha_net.weight"].view(-1) + W[p + ".alpha_net.bias"]
    z = z.masked_fill(att_mask[:, 1:].bool(), O.MIN_VALUE)
    return torch.einsum("br,brh->bh", torch.softmax(z, dim=1), feats["pool_feats"]), z, q


def core_step_dual_region(W, xt, feats, att_mask, pnt_mask, state):
    h, c = state
    h_att, c_att = O._lstm_cell(torch.cat((feats["fc_feats"], xt), dim=1), h[0], c[0], W, "core.att_lstm")
    att2, z, q2 = _region_attention(W, "core.attention2", h_att, feats, att_mask)
    att2_dual, _, _ = _region_attention(W, "core.attention2_dual", h_att, feats, att_mask)
    g = torch.sigmoid(O._lin(h_att, W, "core.dual_pointer.0"))
    z_out = z.masked_fill(pnt_mask[:, 1:].bool(), O.MIN_VALUE)
    h_lang, c_lang = O._lstm_cell(torch.cat((g * att2 + (1 - g) * att2_dual, h_att), dim=1), h[1], c[1], W, "core.lang_lstm")
    return h_lang, (torch.stack((h_att, h_lang)), torch.stack((c_att, c_lang))), z_out, q2


STEPS = {"both": O.core_step, "featmap": core_step_featmap, "dual_region": core_step_dual_region}


@contextlib.contextmanager
def oracle_mode(opt):
    orig = O.core_step
    O.core_step = STEPS[getattr(opt, "att_input_mode", "both")]
    try:
        yield O
    finally:
        O.core_step = orig
