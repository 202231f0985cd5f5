"""CPU checks of the multinomial sampler's definition (tests/sample_ref.py): the oracle with the counter-based noise reproduces the
unmodified reference run with the same noise (fixtures tests/golden/multinomial_*.npz, make_golden_sample.py), and the noise itself is
well formed — uniforms strictly inside (0, 1), one independent word per (row, step, word index), the Philox rounds of the dropout masks."""
import numpy as np
import pytest
import torch

import sample_ref as SR
from cases import build_case, load_fixture
from make_golden_sample import SAMPLE_CASES
from ops_ref import TorchRefOps

TOL = 1e-4


@pytest.mark.parametrize("name", list(SAMPLE_CASES))
def test_oracle_reproduces_reference_draws(name):
    case = SAMPLE_CASES[name]
    opt, sd, inp = build_case(case)
    fx = load_fixture(name)
    B = inp["ppls"].shape[0]
    assert float(fx["min_gap"]) > 1e-3                       # no near-tie of the keys: the token comparison is exact
    seq, logp, att2, _, gaps = SR.sample_multinomial(sd, opt, inp, case["temperature"], SR.noise_fn(case["noise_seed"], np.arange(B), opt.vocab_size))
    assert gaps.min() > 1e-3
    assert np.array_equal(seq.numpy(), fx["seq"])
    assert float(np.abs(logp.numpy() - fx["logp"]).max()) <= TOL
    assert float(np.abs(att2.numpy() - fx["att2"]).max()) <= TOL
    assert len(np.unique(fx["seq"])) > opt.seq_length       # a draw, not a constant caption


def test_uniforms_strictly_inside_the_unit_interval():
    w = np.array([0, 1, 511, 512, 0x7FFFFFFF, 0x80000000, 0xFFFFFE00, 0xFFFFFFFF], dtype=np.uint64)
    u = SR.uniforms(w)
    assert u.dtype == np.float32
    assert bool((u > 0).all()) and bool((u < 1).all())
    assert u[0] == np.float32(2.0 ** -24) and u[-1] == np.float32(1 - 2.0 ** -24)
    assert float(u[-1].astype(np.float64)) == 1 - 2.0 ** -24   # exact in fp32: 23 bits + the half
    g = -np.log(-np.log(u.astype(np.float64)))
    assert np.isfinite(g).all() and -2.9 < g.min() and g.max() < 16.7


def test_noise_words_depend_on_row_step_and_index():
    V = 4905
    base = SR.noise_words(11, [3], 4, V)[0]
    assert len(np.unique(base)) == V                          # every word index its own word (4 words per Philox call)
    for other in (SR.noise_words(11, [4], 4, V)[0], SR.noise_words(11, [3], 5, V)[0], SR.noise_words(12, [3], 4, V)[0],
                  SR.noise_words(11 + (1 << 32), [3], 4, V)[0]):
        assert (other != base).mean() > 0.999                 # another row, step, seed (low and high half)
    rows = SR.noise_words(11, [0, 3, 9], 4, V)                # a row's words do not depend on the other rows of the call
    assert np.array_equal(rows[1], base)
    assert np.array_equal(SR.noise_words(11, [3], 4, 2049)[0], base[:2049])


def test_noise_statistics():
    g = SR.gumbel_noise(5, np.arange(64), 0, 4096).ravel()
    assert abs(g.mean() - 0.5772156649) < 0.01 and abs(g.var() - np.pi ** 2 / 6) < 0.03


def test_philox_rounds_are_the_dropout_masks():
    """The noise and train-mode dropout share one Philox definition: the helper reproduces ops_ref's dropout masks bit for bit."""
    n, p, seed, site, step = 1031, 0.3, 0x123456789AB, 5, (7 << 32) + 9
    x = torch.ones(n)
    y = TorchRefOps().dropout(x, p, seed, site, step)
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    words = SR.philox4x32_10(q, np.full_like(q, site), (step & 0xFFFFFFFF) ^ (q >> np.uint64(32)), np.full_like(q, step >> 32), seed & 0xFFFFFFFF,
                             seed >> 32)
    u = (np.stack(words, axis=1).reshape(-1)[:n] >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    assert np.array_equal((y != 0).numpy(), u >= np.float32(p))
