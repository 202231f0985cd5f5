"""The grounded beam search on the CPU (tests/beam_att2_ref.py): the region-attention logits of each returned caption, on every beam case of
the reference's fixtures and on scripts.  The search itself is unchanged (seq / logps / indices equal the oracle's and the fixtures'); the
logit rows up to the caption's end equal the teacher-forced pass on the caption; the rows after it are 0."""
import warnings

import numpy as np
import pytest
import torch

from beam_att2_ref import BEAM_CASES, beam_case, caption_length, sample_beam_att2, scripted_att2, teacher_att2
from beam_ref import make_script, scripted_search
from cases import CASES, build_case, load_fixture
from region_attn_oracle import oracle_modes


@pytest.mark.parametrize("name", sorted(BEAM_CASES))
def test_grounded_beam_keeps_the_search_and_returns_the_teacher_forced_logits(name):
    case, opt, sd, W, inp = beam_case(name)
    fx = load_fixture(name)
    K = case["beam_size"]
    with oracle_modes(opt) as O:
        feats = O.prologue(W, opt, inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"])
        oseq, olp, oatt = O.sample_beam(W, opt, inp, K, feats=feats)
        seq, lp, att, att2 = sample_beam_att2(W, opt, inp, K, feats=feats)
        tf = teacher_att2(W, opt, inp, seq, feats=feats)
    assert torch.equal(seq, oseq) and torch.equal(lp, olp) and torch.equal(att, oatt)
    assert np.array_equal(seq.numpy(), fx["seq"]) and np.array_equal(att.numpy(), fx["att2_idx"])
    B, L = seq.shape
    assert att2.shape == (B, L, inp["pnt_mask"].shape[1] - 1) and att2.dtype == torch.float32
    for b, n in enumerate(caption_length(seq)):
        assert float((att2[b, :n] - tf[b, :n]).abs().max()) <= 1e-5, (b, n)
        assert not att2[b, n:].any()
        # the masked columns carry the mask value, as in greedy decoding's logits
        assert bool((att2[b, :n][:, inp["pnt_mask"][b, 1:].bool()] == O.MIN_VALUE).all())
    # a caption's logits select the region the search reported for its first word (the <bos> step's own argmax)
    assert torch.equal(att2[:, 0].argmax(dim=1), att[:, 0])


def test_grounded_beam_cases_end_early_and_late():
    """The fixtures hold captions that end before the last step (tail rows zero) and captions that run to it."""
    ends = [n for name in BEAM_CASES for n in caption_length(load_fixture(name)["seq"])]
    L = {beam_case(name)[1].seq_length for name in BEAM_CASES}
    assert min(ends) < min(L) and max(ends) == max(L)


SCRIPTS = [  # B, K, L, V, R, script kwargs
    (3, 3, 6, 40, 24, dict(seed=1)),
    (4, 2, 5, 33, 17, dict(seed=2, ties=True)),
    (3, 3, 6, 40, 20, dict(seed=3, eos_at=0)),
    (2, 4, 7, 50, 16, dict(seed=4, no_eos=True)),
    (2, 3, 64, 300, 36, dict(seed=5)),
]


@pytest.mark.parametrize("B,K,L,V,R,kw", SCRIPTS)
def test_scripted_att2_reference_keeps_the_search(B, K, L, V, R, kw):
    """scripted_att2 runs beam_ref's bookkeeping: its search equals scripted_search's, and its rows are rows of the script's z of the
    right step, zero after the end."""
    logits, z = make_script(B, K, L, V, R, **kw)
    seq, lp, att, parents, att2 = scripted_att2(logits, z, K, L)
    s_seq, s_lp, s_att, s_parents, _ = scripted_search(logits, z, K, L)
    assert np.array_equal(seq, s_seq) and np.array_equal(lp, s_lp) and np.array_equal(att, s_att) and np.array_equal(parents, s_parents)
    for b, n in enumerate(caption_length(seq)):
        for t in range(L):
            if t < n:
                assert any(np.array_equal(att2[b, t], z[t, b * K + q]) for q in range(K))
            else:
                assert not att2[b, t].any()
    if kw.get("eos_at") == 0:
        assert caption_length(seq) == [1] * B
    if kw.get("no_eos"):
        assert caption_length(seq) == [L] * B


def test_att2_weights_refused_by_the_transformer_captioner():
    """The transformer captioner has no region attention to return: the key raises, as beam_size > 1 does there (before any device work)."""
    from gvd_b200.misc.AttModel import TopDownModel
    opt, sd, inp = build_case(CASES["tfm_greedy_small_B5"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = TopDownModel(opt).eval()
    args = [inp[k] for k in ("segs_feat", "ppls", "num", "ppls_feat", "sample_idx", "pnt_mask")]
    for eo in ({"beam_size": 1, "att2_weights": True}, {"beam_size": 3, "att2_weights": True}):
        with pytest.raises(NotImplementedError, match="att2_weights"):
            model._sample(*args, eo)
