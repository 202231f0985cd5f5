"""References for the grounded beam search (gvd_beam_decode_att2, forward(..., 'sample') with eval_opt['att2_weights']): the region-attention
logits of each returned caption, row t being the logit row the caption's own beam used to pick word t, zeros after its last word.

These references carry every beam's rows along with the beam, the way the bookkeeping carries its words (a finished beam records a copy),
instead of walking parent pointers back at the end as the device does: two constructions of the same rows.

  sample_beam_att2   oracle/gvd_oracle.py::sample_beam with that per-beam history; its seq / logps / indices are the oracle's own
  teacher_att2       the teacher-forced region logits of given captions (the contract: the attention a caption used is the attention
                     teacher forcing gives it)
  scripted_att2      beam_ref.scripted_search with the same history, on a script (gvd_op_beam_att2_scripted)

The oracle's decode step is read through the module attribute ``gvd_oracle.core_step``, so the mode contexts of input_mode_oracle.py /
region_attn_oracle.py apply."""
import numpy as np
import torch

import gvd_oracle as O
from beam_ref import ClipBeams, beam_step, step_topk
from cases import CASES, build_case
from input_mode_cases import INPUT_MODE_CASES
from region_attn_cases import REGION_ATTN_CASES
from region_feat_cases import REGION_FEAT_CASES
from region_feat_oracle import oracle_weights
from vocab_cases import VOCAB_CASES

FEAT_KEYS = ("fc_feats", "conv_feats", "p_conv_feats", "pool_feats", "p_pool_feats")

# every beam case with a fixture of the reference (tests/golden/*beam*.npz)
BEAM_CASES = {n: c for d in (CASES, INPUT_MODE_CASES, REGION_ATTN_CASES, REGION_FEAT_CASES, VOCAB_CASES) for n, c in d.items()
              if c["kind"] == "beam"}


def beam_case(name):
    """(case, opt, state_dict, oracle weights, inputs) of a beam case; run the oracle inside region_attn_oracle.oracle_modes(opt)."""
    case = BEAM_CASES[name]
    opt, sd, inp = build_case(case)
    return case, opt, sd, oracle_weights(opt, sd), inp


def _feats(W, opt, inp, feats):
    if feats is None:
        feats = O.prologue(W, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    return feats


def sample_beam_att2(W, opt, inp, beam_size, feats=None):
    """O.sample_beam's search, line for line, plus beam_z [L, K, R]: the logit rows each live beam used.  Returns seq, logps, att2 index
    (as O.sample_beam) and att2 [B, L, R]."""
    feats = _feats(W, opt, inp, feats)
    B = inp["ppls"].shape[0]
    H, L = opt.rnn_size, opt.seq_length
    K = beam_size
    seq_out = torch.zeros(B, L, dtype=torch.long)
    lp_out = torch.zeros(B, L)
    att_out = torch.full((B, L), -1, dtype=torch.long)
    att2_out = None
    for b in range(B):
        fb = {k: feats[k][b:b + 1].expand(K, *feats[k].shape[1:]) for k in FEAT_KEYS}
        mask = inp["pnt_mask"][b:b + 1].expand(K, -1)
        state = (torch.zeros(2, K, H), torch.zeros(2, K, H))
        out, state, z, _ = O.core_step(W, O.embed_tokens(W, torch.zeros(K, dtype=torch.long)), fb, mask, mask, state)
        if att2_out is None:
            att2_out = torch.zeros(B, L, z.shape[1])
        att_out[b, 0] = int(z[0].argmax())
        beam_seq = torch.zeros(L, K, dtype=torch.long)
        beam_lp = torch.zeros(L, K)
        beam_att = torch.full((L, K), -1, dtype=torch.long)
        beam_z = torch.zeros(L, K, z.shape[1])
        att_ind = torch.full((K,), -1, dtype=torch.long)
        sums = torch.zeros(K)
        done = []
        for t in range(L):
            logp = torch.log_softmax(O._lin(out, W, "logit"), dim=1)
            ys, ix = torch.sort(logp, 1, descending=True)
            rows = 1 if t == 0 else K
            cands = []
            for cpos in range(min(K, ys.shape[1])):
                for q in range(rows):
                    cands.append((float(sums[q] + ys[q, cpos]), int(ix[q, cpos]), q, float(ys[q, cpos]), int(att_ind[q])))
            cands.sort(key=lambda x: -x[0])
            prev_seq, prev_lp, prev_att, prev_z = beam_seq[:t].clone(), beam_lp[:t].clone(), beam_att[:t].clone(), beam_z[:t].clone()
            new_h, new_c, new_out = state[0].clone(), state[1].clone(), out.clone()
            for v in range(K):
                p, tok, q, r, w = cands[v]
                if t >= 1:
                    beam_seq[:t, v], beam_lp[:t, v], beam_att[:t, v], beam_z[:t, v] = prev_seq[:, q], prev_lp[:, q], prev_att[:, q], prev_z[:, q]
                new_h[:, v], new_c[:, v], new_out[v] = state[0][:, q], state[1][:, q], out[q]
                beam_seq[t, v], beam_lp[t, v] = tok, r
                beam_z[t, v] = z[q]                                   # the logits that picked word t: those of the beam it continues
                if t >= 1:
                    beam_att[t, v] = w
                sums[v] = torch.tensor(p, dtype=torch.float32)
            state, out = (new_h, new_c), new_out
            for v in range(K):
                if int(beam_seq[t, v]) == 0 or t == L - 1:
                    zs = beam_z[:, v].clone()
                    zs[t + 1:] = 0
                    done.append(dict(seq=beam_seq[:, v].clone(), logps=beam_lp[:, v].clone(), slot=v, z=zs))
                    sums[v] = -1000.0
            out, state, z, _ = O.core_step(W, O.embed_tokens(W, beam_seq[t]), fb, mask, mask, state)
            att_ind = z.argmax(dim=1)
        done.sort(key=lambda d: -float(sums[d["slot"]]))
        best = done[0]
        seq_out[b], lp_out[b], att2_out[b] = best["seq"], best["logps"], best["z"]
        att_out[b, 1:] = beam_att[1:, best["slot"]]
    return seq_out, lp_out, att_out, att2_out


def caption_length(seq):
    """Words of each caption up to and including its first token 0 (the step at which its beam finished), the whole length without one."""
    L = seq.shape[1]
    n = []
    for row in np.asarray(seq):
        z = np.flatnonzero(row == 0)
        n.append(int(z[0]) + 1 if z.size else L)
    return n


def teacher_att2(W, opt, inp, seq, feats=None):
    """The region logits [B, L, R] of the teacher-forced pass on captions seq [B, L]: step t feeds <bos> (t = 0) or word t - 1, as
    O.forward_teacher's 'GRD' pass does (both masks the proposal mask)."""
    feats = _feats(W, opt, inp, feats)
    B, L, H = seq.shape[0], seq.shape[1], opt.rnn_size
    state = (torch.zeros(2, B, H), torch.zeros(2, B, H))
    tokens = torch.cat((torch.zeros(B, 1, dtype=torch.long), torch.as_tensor(seq, dtype=torch.long)[:, :L - 1]), dim=1)
    fb = {k: feats[k] for k in FEAT_KEYS}
    zs = []
    for t in range(L):
        _, state, z, _ = O.core_step(W, O.embed_tokens(W, tokens[:, t]), fb, inp["pnt_mask"], inp["pnt_mask"], state)
        zs.append(z)
    return torch.stack(zs, 1)


def scripted_att2(logits, z, K, L, topk=None):
    """beam_ref.scripted_search on a script (logits [L, B*K, V], region scores z [L+1, B*K, R]) with each beam's rows of z carried along;
    topk as scripted_search takes it.  Returns seq [B, L], logp [B, L], att2 index [B, L], parents [L, B*K] and att2 [B, L, R]."""
    logits = np.asarray(logits, np.float32)
    z = np.asarray(z, np.float32)
    BK, R = logits.shape[1], z.shape[2]
    B = BK // K
    seq = np.zeros((B, L), np.int64)
    lp = np.zeros((B, L), np.float32)
    att = np.full((B, L), -1, np.int64)
    parents = np.zeros((L, BK), np.int64)
    att2 = np.zeros((B, L, R), np.float32)
    for b in range(B):
        rs = slice(b * K, (b + 1) * K)
        cb = ClipBeams(K, L)
        bz = np.zeros((L, K, R), np.float32)
        done_z = []
        att[b, 0] = int(np.argmax(z[0, b * K]))
        for t in range(L):
            ys, ix = step_topk(logits[t, rs], K) if topk is None else (topk[0][t, rs], topk[1][t, rs])
            n_done = len(cb.done)
            parents[t, rs], _ = beam_step(cb, ys, ix, t)
            par = parents[t, rs]
            bz[:t] = bz[:t, par].copy()
            bz[t] = z[t, rs][par]
            for _, _, v in cb.done[n_done:]:
                zs = bz[:, v].copy()
                zs[t + 1:] = 0
                done_z.append(zs)
            cb.att_ind = np.argmax(z[t + 1, rs], axis=1) if t + 1 < z.shape[0] else cb.att_ind
        order = sorted(range(len(cb.done)), key=lambda i: -float(cb.sums[cb.done[i][2]]))
        best_seq, best_lp, slot = cb.done[order[0]]
        seq[b], lp[b] = best_seq, best_lp
        att[b, 1:] = cb.att[1:, slot]
        att2[b] = done_z[order[0]]
    return seq, lp, att, parents, att2
