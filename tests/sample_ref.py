"""Definition of the multinomial sampler (sample_max = 0) — TEST INFRASTRUCTURE.

The reference draws with torch.multinomial on torch's global RNG (misc/model.py:595-603), so no implementation can match its draws.
Like dropout (tests/ops_ref.py::TorchRefOps.dropout), the sampler uses counter-based noise instead, and the checkers take that noise as an
injected input:

  u_i = ((w >> 9) + 0.5) * 2^-23,  w = word (i & 3) of Philox4x32-10(counter = (i >> 2, b, t, 0), key = (seed_lo, seed_hi))
  g_i = -log(-log(u_i))                                   (Gumbel noise; b = the row in the decode call, t = the decode step)
  it  = argmax_i (logit_i / temperature + g_i)            (ties -> lower index; the Gumbel-max trick: it ~ softmax(logit / temperature))
  logp = log_softmax(logit)[it]                           (untempered, model.py:602)

``sample_multinomial`` restates the reference's decode loop (model.py:586-624) on the functional oracle with that draw."""
import numpy as np
import torch

import gvd_oracle as O

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays holding 32-bit values (counter c0..c3, key k0, k1): the round function of csrc/gvd_common.cuh."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _M32 for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _M32, p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def noise_words(seed, rows, t, V):
    """The 32-bit words [len(rows), V] behind the noise of decode step t for the batch rows `rows` (their indices in the decode call)."""
    rows = np.asarray(rows, dtype=np.uint64).reshape(-1, 1)
    q = np.arange((V + 3) // 4, dtype=np.uint64).reshape(1, -1)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    c0, c1 = np.broadcast_arrays(q, rows)
    words = philox4x32_10(c0, c1, np.full(c0.shape, t & 0xFFFFFFFF, np.uint64), np.zeros(c0.shape, np.uint64), seed & 0xFFFFFFFF, seed >> 32)
    return np.stack(words, axis=2).reshape(len(rows), -1)[:, :V]


def uniforms(words):
    """u = ((w >> 9) + 0.5) * 2^-23 in float32 (exact): 23-bit uniforms strictly inside (0, 1)."""
    w = np.asarray(words, dtype=np.uint64)
    return ((w >> np.uint64(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)


def gumbel_noise(seed, rows, t, V):
    """g [len(rows), V] float64 = -log(-log(u)) of the float32 uniforms."""
    u = uniforms(noise_words(seed, rows, t, V)).astype(np.float64)
    return -np.log(-np.log(u))


def noise_fn(seed, rows, V):
    """noise(t) -> [len(rows), V] float64 tensor: the hook ``sample_multinomial`` and the reference run take."""
    return lambda t: torch.from_numpy(gumbel_noise(seed, rows, t, V))


def sample_multinomial(W, opt, inp, temperature, noise, feats=None):
    """``_sample`` with sample_max = 0, beam_size = 1 (model.py:492-624) with the draw argmax(logprobs / temperature + noise(t)).
    Returns (seq [B,L], logp [B,L], att2 [B,L,R], sim_mat, min_gap [L]): min_gap[t] = the smallest top-2 key gap over the rows at step t
    (a token comparison is exact where that gap is well above the rounding of the keys)."""
    if feats is None:
        feats = O.prologue(W, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
    B = inp["ppls"].shape[0]
    H, L = opt.rnn_size, opt.seq_length
    state = (torch.zeros(2, B, H), torch.zeros(2, B, H))
    it = torch.zeros(B, dtype=torch.long)
    seq, lps, att2, gaps = [], [], [], []
    for t in range(L):
        h_lang, state, z, _ = O.core_step(W, O.embed_tokens(W, it), feats, inp["pnt_mask"], inp["pnt_mask"], state)
        logprobs = torch.log_softmax(O._lin(h_lang, W, "logit"), dim=1)
        key = logprobs.double() / temperature + noise(t)
        it = key.argmax(dim=1)                                      # first maximal index
        top2 = torch.topk(key, 2, dim=1).values
        gaps.append(float((top2[:, 0] - top2[:, 1]).min()))
        seq.append(it)
        lps.append(logprobs.gather(1, it.unsqueeze(1)).squeeze(1))
        att2.append(z)
    return torch.stack(seq, 1), torch.stack(lps, 1), torch.stack(att2, 1), feats["sim_mat"], np.array(gaps)
