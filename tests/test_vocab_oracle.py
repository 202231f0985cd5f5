"""Vocabularies above 6144 words on the CPU: the oracle against the unmodified reference's outputs at V = 9001, 13001 and 40000
(tests/golden/vocab_cases.py, make_golden_vocab.py), and an emulation of the sliced vocabulary tail's indexing (vocab_tail_kernel in
csrc/gvd_skinny.cu): every word is read by exactly one thread of one slice, the four words of a thread are those of one Philox counter, and
the merge visits every record once in an order that does not depend on which CTA finishes last."""
import numpy as np
import pytest

import gvd_oracle as O
import sampler_ref
from cases import build_case, load_fixture, subsample
from vocab_cases import VOCAB_CASES as CASES

TOL = 1e-4
SLICE, NT = 1024, 256            # VOCAB_SLICE and the threads of one CTA (4 words each)


def _names(kind):
    return [n for n, c in CASES.items() if c["kind"] == kind]


def _close(a, b, tol=TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.max(np.abs(a - b)) <= tol, np.max(np.abs(a - b))


@pytest.mark.parametrize("name", _names("greedy"))
def test_wide_vocab_greedy_matches_reference(name):
    opt, sd, inp = build_case(CASES[name])
    assert opt.vocab_size > 6144
    fx = load_fixture(name)
    seq, logp, att2, sim = O.sample_greedy(sd, opt, inp)
    assert fx["min_margin"] > TOL and fx["unk_top1_steps"] > 0            # the UNK rule decides some steps
    assert np.array_equal(seq.numpy(), fx["seq"])
    _close(logp.numpy(), fx["logp"])
    _close(att2.numpy(), fx["att2"])
    _close(subsample("sim_mat", sim).numpy(), fx["sim_mat"])


@pytest.mark.parametrize("name", _names("beam"))
def test_wide_vocab_beam_matches_repaired_reference(name):
    case = CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    seq, logp, att = O.sample_beam(sd, opt, inp, case["beam_size"])
    assert np.array_equal(seq.numpy(), fx["seq"]) and np.array_equal(att.numpy(), fx["att2_idx"])
    _close(logp.numpy(), fx["logp"])


@pytest.mark.parametrize("name", _names("mle"))
def test_wide_vocab_mle_losses_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    _close(np.array([float(x) for x in O.forward_teacher(sd, opt, inp)]), load_fixture(name)["losses"])


@pytest.mark.parametrize("name", _names("grd"))
def test_wide_vocab_grd_indices_match_reference(name):
    opt, sd, inp = build_case(CASES[name])
    fx = load_fixture(name)
    cls_pred, att_idx, grd_idx = O.forward_teacher(sd, opt, inp, eval_obj_ground=True)
    assert np.array_equal(cls_pred.numpy(), fx["cls_pred"])
    assert np.array_equal(att_idx.numpy(), fx["att_idx"]) and np.array_equal(grd_idx.numpy(), fx["grd_idx"])


@pytest.mark.parametrize("name", _names("tfm_greedy"))
def test_wide_vocab_transformer_greedy_matches_reference(name):
    opt, sd, inp = build_case(CASES[name])
    assert opt.vocab_size > 12000                                         # above the transformer head's shared-memory row
    fx = load_fixture(name)
    seq, _, _, trace = O.tfm_sample(sd, opt, inp, return_trace=True)
    assert fx["min_margin"] > TOL and np.array_equal(seq.numpy(), fx["seq"])
    import torch
    _close(subsample("tfm_logits", torch.stack(trace, 1)).numpy(), fx["tfm_logits"])


# ------------------------------------------------------------------------------------------------------------ index emulation
def _slice_words(V, j, x):
    """Words thread x of slice j reads (the float4 group 4x .. 4x + 3 of the slice, cut at V) and its Philox counter."""
    i0 = j * SLICE + 4 * x
    return [i for i in range(i0, i0 + 4) if i < V], i0 >> 2


def _merge_order(nsl):
    """(lane, slices in the order that lane merges them) of warp 0 in the merging CTA."""
    return [(lane, list(range(lane, nsl, 32))) for lane in range(32)]


@pytest.mark.parametrize("V", [2, 1023, 1024, 1025, 6145, 8192, 8193, 12001, 40000, 65536])
def test_every_word_read_once_and_every_record_merged_once(V):
    nsl = -(-V // SLICE)
    seen = np.zeros(V, np.int64)
    for j in range(nsl):
        for x in range(NT):
            words, ctr = _slice_words(V, j, x)
            for k, i in enumerate(words):
                assert i >> 2 == ctr and (i & 3) == k          # word i takes output (i & 3) of counter (i >> 2): the noise of reduce_sample
            seen[words] += 1
    assert (seen == 1).all()
    # the last group is read as one float4 inside the row pitch (ldp >= V, ldp % 4 == 0)
    ldp = -(-V // 4) * 4
    assert max(j * SLICE + 4 * x + 3 for j in range(nsl) for x in range(NT) if j * SLICE + 4 * x < V) < ldp
    merged = sorted(s for _, ss in _merge_order(nsl) for s in ss)
    assert merged == list(range(nsl))
    assert all(ss == sorted(ss) for _, ss in _merge_order(nsl))


def _emulate_tail(x, unk, arrival):
    """The greedy tail on float32 logits x [V] with the slices finishing in the order `arrival`: per-slice records (top-2, max, sum of
    exp), the merge of the last arrival; returns (token, logp)."""
    V = x.shape[0]
    nsl = -(-V // SLICE)
    rec = {}
    for j in arrival:                                          # records land in any order ...
        w = x[j * SLICE:(j + 1) * SLICE]
        order = np.argsort(-w, kind="stable")[:2]
        m = np.float32(w[order[0]])
        s = np.float32(np.exp(w.astype(np.float64) - m).sum())
        v2, i2 = (w[order[1]], j * SLICE + order[1]) if len(w) > 1 else (-np.inf, 2 ** 31 - 1)
        rec[j] = (m, s, w[order[0]], j * SLICE + order[0], v2, i2)
    cand = []
    M = -np.inf
    for lane, ss in _merge_order(nsl):                         # ... and are read in a fixed order
        for j in ss:
            m, s, v1, i1, v2, i2 = rec[j]
            M = max(M, m)
            cand += [(v1, i1), (v2, i2)]
    S = sum(float(rec[j][1]) * np.exp(float(rec[j][0]) - M) for _, ss in _merge_order(nsl) for j in ss)
    cand.sort(key=lambda c: (-c[0], c[1]))
    (v1, i1), (v2, i2) = cand[0], cand[1]
    tok, val = (i1, v1) if i1 != unk else (i2, v2)
    return tok, float(val) - (M + np.log(S))


@pytest.mark.parametrize("V,unk", [(6145, 6144), (9001, 4500), (12001, 0)])
def test_emulated_tail_matches_the_greedy_rule_on_tie_and_unk_rows(V, unk):
    """The record / merge scheme gives sampler_ref's token on every special row (ties within and across slices, UNK on top), whatever the
    order in which the slices finish."""
    x, kinds = sampler_ref.special_rows(len(sampler_ref.KINDS), V, unk, seed=V + unk)
    want_tok, want_lp = sampler_ref.pick_reference(x, unk)
    nsl = -(-V // SLICE)
    rs = np.random.RandomState(V)
    for b in range(x.shape[0]):
        for arrival in (list(range(nsl)), list(rs.permutation(nsl))):
            tok, lp = _emulate_tail(x[b].astype(np.float32), unk, arrival)
            assert tok == want_tok[b], (kinds[b], tok, want_tok[b])
            assert abs(lp - want_lp[b]) <= 1e-5, kinds[b]
