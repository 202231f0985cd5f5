"""beam_ref.scripted_search against the oracle's sample_beam (no GPU): the oracle's model calls (core_step, the vocabulary head, the token
embedding) are replaced by stubs that serve a scripted sequence of logits and region scores, so what is compared is the bookkeeping alone.
test_gpu_attn_beam_ops.py holds the device kernels to the same reference."""
import types

import numpy as np
import pytest
import torch

import gvd_oracle as O
from beam_ref import make_script, scripted_search


def oracle_search(monkeypatch, logits, z, K, L):
    """O.sample_beam with the model replaced by the script: core call i of clip b returns z[i] and tags its output with i, and the
    vocabulary head maps that tag back to logits[i]."""
    BK = logits.shape[1]
    B = BK // K
    calls = [0]

    def core_step(W, xt, feats, att_mask, pnt_mask, state):
        i = calls[0]
        calls[0] += 1
        b, t = divmod(i, L + 1)
        assert xt.shape[0] == K
        return torch.full((K, 1), float(i)), state, torch.from_numpy(z[t, b * K:(b + 1) * K].copy()), None

    def lin(x, W, name, relu=False):
        assert name == "logit"
        b, t = divmod(int(x[0, 0]), L + 1)
        assert bool((x == x[0, 0]).all())
        return torch.from_numpy(logits[t, b * K:(b + 1) * K].copy())

    monkeypatch.setattr(O, "core_step", core_step)
    monkeypatch.setattr(O, "_lin", lin)
    monkeypatch.setattr(O, "embed_tokens", lambda W, it: torch.zeros(it.shape[0], 1))
    opt = types.SimpleNamespace(rnn_size=4, seq_length=L)
    feats = {k: torch.zeros(B, 1) for k in ("fc_feats", "conv_feats", "p_conv_feats", "pool_feats", "p_pool_feats")}
    inp = {"ppls": torch.zeros(B, 1, 7), "pnt_mask": torch.zeros(B, 2, dtype=torch.uint8)}
    seq, lp, att = O.sample_beam({}, opt, inp, K, feats=feats)
    assert calls[0] == B * (L + 1)
    return seq.numpy(), lp.numpy(), att.numpy()


_CASES = [  # B, K, L, V, R
    (1, 2, 1, 9, 13), (3, 2, 2, 9, 13), (3, 3, 20, 257, 52), (2, 5, 20, 9, 7), (2, 8, 20, 255, 13), (1, 8, 64, 8, 5), (2, 3, 64, 4905, 13),
    (4, 2, 20, 2, 3)]


@pytest.mark.parametrize("kind", ["random", "ties", "eos", "no_eos"])
@pytest.mark.parametrize("B,K,L,V,R", _CASES)
def test_scripted_search_matches_oracle(monkeypatch, B, K, L, V, R, kind):
    """seq, log-probabilities and attention indices bit for bit."""
    logits, z = make_script(B, K, L, V, R, seed=B * 1000 + K * 100 + L + V, ties=kind == "ties", eos_at=L // 2 if kind == "eos" else None,
                            no_eos=kind in ("ties", "no_eos"))
    seq, lp, att, parents, ties = scripted_search(logits, z, K, L)
    oseq, olp, oatt = oracle_search(monkeypatch, logits, z, K, L)
    assert np.array_equal(seq, oseq)
    assert np.array_equal(lp.view(np.int32), olp.view(np.int32))
    assert np.array_equal(att, oatt)
    assert parents.min() >= 0 and parents.max() < K
    if kind == "ties" and L > 1 and K < V:
        assert ties > 0                                   # the script does exercise the stable order
    if kind == "no_eos" and K < V:
        assert not (seq[:, :-1] == 0).any()


def test_scripted_search_first_pushed_beam_wins(monkeypatch):
    """All three beams of a clip emit token 0 at step 1: the first one pushed (slot 0, the continuation of the best beam) is the result."""
    K, L, V, R = 3, 4, 6, 5
    logits = np.full((L, K, V), -8.0, np.float32)
    logits[0, 0, 1:4] = [2.0, 1.0, 0.0]                   # step 0: beams of words 1, 2, 3
    logits[1, :, 0] = 4.0                                 # step 1: token 0 best for every beam
    z = np.random.RandomState(0).randint(-4, 5, size=(L + 1, K, R)).astype(np.float32)
    seq, lp, att, parents, _ = scripted_search(logits, z, K, L)
    assert seq.tolist() == [[1, 0, 0, 0]] and parents[1].tolist() == [0, 1, 2]
    oseq, olp, oatt = oracle_search(monkeypatch, logits, z, K, L)
    assert np.array_equal(seq, oseq) and np.array_equal(lp, olp) and np.array_equal(att, oatt)
