"""The beam search's bookkeeping (oracle/gvd_oracle.py::sample_beam, lines 603-629) in numpy, one step at a time, and a whole search on a
script: logits and region scores given per step instead of computed by the model.

test_beam_emulation.py pins `scripted_search` to the oracle (whose model calls are replaced by the same script); test_gpu_attn_beam_ops.py
compares gvd_op_beam_search_scripted (beam_topk, beam_update, beam_gather_rows, row_argmax, beam_finish) with it bit for bit."""
import numpy as np
import torch


class ClipBeams:
    """The bookkeeping of one clip's K beams over L steps (sample_beam's beam_seq, beam_lp, beam_att, att_ind, sums, done)."""

    def __init__(self, K, L):
        self.K, self.L = K, L
        self.seq = np.zeros((L, K), np.int64)
        self.lp = np.zeros((L, K), np.float32)
        self.att = np.full((L, K), -1, np.int64)
        self.att_ind = np.full(K, -1, np.int64)
        self.sums = np.zeros(K, np.float32)
        self.done = []                                    # (seq, logps) cloned when a beam finishes, and its slot


def beam_step(cb, ys, ix, t):
    """Step t given each current beam's words by descending log-probability, ys / ix [K, >= K] (float32 / int): candidates in c-major /
    q-minor order (one row at t = 0), a stable sort by -(sums[q] + ys[q, c]) in fp32, the first K continue (new beam v forks old beam q),
    finishing beams (token 0 or the last step) are recorded in push order and their running sum set to -1000.
    Returns (parent [K], number of exactly tied candidate pairs among the first K + 1 of the sorted list)."""
    K = cb.K
    rows = 1 if t == 0 else K
    cands = []
    for c in range(min(K, ys.shape[1])):
        for q in range(rows):
            cands.append((np.float32(cb.sums[q]) + np.float32(ys[q, c]), int(ix[q, c]), q, np.float32(ys[q, c]), int(cb.att_ind[q])))
    cands.sort(key=lambda x: -float(x[0]))                 # list.sort is stable
    head = [float(c[0]) for c in cands[:K + 1]]
    ties = sum(head[i] == head[i + 1] for i in range(len(head) - 1))
    prev_seq, prev_lp, prev_att = cb.seq[:t].copy(), cb.lp[:t].copy(), cb.att[:t].copy()
    parent = np.zeros(K, np.int64)
    for v in range(K):
        p, tok, q, r, w = cands[v]
        if t >= 1:
            cb.seq[:t, v], cb.lp[:t, v], cb.att[:t, v] = prev_seq[:, q], prev_lp[:, q], prev_att[:, q]
        cb.seq[t, v], cb.lp[t, v] = tok, r
        if t >= 1:
            cb.att[t, v] = w
        cb.sums[v] = p
        parent[v] = q
    for v in range(K):
        if cb.seq[t, v] == 0 or t == cb.L - 1:
            cb.done.append((cb.seq[:, v].copy(), cb.lp[:, v].copy(), v))
            cb.sums[v] = np.float32(-1000.0)
    return parent, ties


def step_topk(logits, K):
    """ys / ix [rows, K] as sample_beam takes them: fp32 log_softmax (torch, like the oracle), words by descending value, ties to the lower
    index."""
    lp = torch.log_softmax(torch.from_numpy(np.ascontiguousarray(logits, np.float32)), dim=-1).numpy()
    ix = np.argsort(-lp, axis=1, kind="stable")[:, :K]
    return np.take_along_axis(lp, ix, axis=1), ix


def scripted_search(logits, z, K, L, topk=None):
    """The whole search on a script: logits [L, B*K, V] (step t's vocabulary logits), z [L+1, B*K, R] (region scores of core step t, t = 0
    the <bos> step).  topk: optional (ys, ix) [L, B*K, K] replacing step_topk (the device's own beam_topk output).
    Returns seq [B, L] int64, logp [B, L] float32, att2 index [B, L] int64, parents [L, B*K] int64 and the number of tied candidate pairs
    that the stable sort ordered."""
    logits = np.asarray(logits, np.float32)
    z = np.asarray(z, np.float32)
    BK = logits.shape[1]
    B = BK // K
    seq = np.zeros((B, L), np.int64)
    lp = np.zeros((B, L), np.float32)
    att = np.full((B, L), -1, np.int64)
    parents = np.zeros((L, BK), np.int64)
    ties = 0
    for b in range(B):
        rs = slice(b * K, (b + 1) * K)
        cb = ClipBeams(K, L)
        att[b, 0] = int(np.argmax(z[0, b * K]))           # first index of the maximum, like torch.argmax
        for t in range(L):
            ys, ix = step_topk(logits[t, rs], K) if topk is None else (topk[0][t, rs], topk[1][t, rs])
            parents[t, rs], n = beam_step(cb, ys, ix, t)
            ties += n
            cb.att_ind = np.argmax(z[t + 1, rs], axis=1) if t + 1 < z.shape[0] else cb.att_ind
        order = sorted(range(len(cb.done)), key=lambda i: -float(cb.sums[cb.done[i][2]]))   # keys read after the search
        best_seq, best_lp, slot = cb.done[order[0]]
        seq[b], lp[b] = best_seq, best_lp
        att[b, 1:] = cb.att[1:, slot]
    return seq, lp, att, parents, ties


def make_script(B, K, L, V, R, seed, ties=False, eos_at=None, no_eos=False):
    """logits [L, B*K, V] and region scores [L+1, B*K, R].  The words of a row have distinct values (the reference's torch.sort does not
    promise an order for equal words; beam_topk's lower-index rule is tested on its own) on a dyadic grid just below 100, so that the
    log-probabilities x - lse are exact fp32 differences and sums of them coincide exactly whenever they coincide on the grid.
    ties: all rows of a step equal, so that joint scores sums[q] + ys[q, c] of different beams collide and the
    stable c-major / q-minor order decides; region scores from a three-value set (first-index argmax).  eos_at: at that step token 0 is
    the best word of every row (several beams finish at once).  no_eos: token 0 is the worst word everywhere, no beam finishes early (a
    finished beam's sum of -1000 would also keep it out of ties)."""
    rs = np.random.RandomState(seed)
    step = 2.0 ** -max(2, int(np.ceil(np.log2(V / 16.0))))

    def rows(n):                                          # no_eos: word 0 below the grid, the other words a permutation of it
        r = 100.0 - step * (1 + np.stack([rs.permutation(V - no_eos) for _ in range(n)]))
        return np.concatenate((np.full((n, 1), 100.0 - step * (V + 8)), r), axis=1) if no_eos else r

    if ties:
        logits = np.stack([np.repeat(rows(1), B * K, axis=0) for _ in range(L)])
        z = rs.randint(-2, 1, size=(L + 1, B * K, R)) * 0.25
    else:
        logits = np.stack([rows(B * K) for _ in range(L)])
        z = rs.randint(-40, 41, size=(L + 1, B * K, R)) * 0.25
    if eos_at is not None:
        logits[eos_at, :, 0] = 100.0
    return logits.astype(np.float32), z.astype(np.float32)
