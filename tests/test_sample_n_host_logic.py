"""n sampled captions per clip, on the CPU: the eval_opt['sample_n'] validation and refusals, and an emulation of the row-grouped decode
attention's grid and ticket arithmetic (attn_group_kernel in csrc/gvd_decode.cu)."""
import warnings

import numpy as np
import pytest
import torch

from cases import CASES
from gvd_b200 import synth
from gvd_b200.misc.model import check_sample_n


# ------------------------------------------------------------------------------------------------------------ eval_opt['sample_n']
@pytest.mark.parametrize("n", [1, 2, 7, 100, np.int64(3), torch.tensor(4)])
def test_valid_sample_n(n):
    assert check_sample_n(n) == int(n)


@pytest.mark.parametrize("n", [0, -1, 2.0, 2.5, "3", None, True, False, [2]])
def test_invalid_sample_n(n):
    with pytest.raises(ValueError):
        check_sample_n(n)


def _cpu_model(**over):
    from gvd_b200.misc.AttModel import TopDownModel
    opt = synth.make_opt(**dict(CASES["greedy_small_B5"]["opt"], **over))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = TopDownModel(opt)
    return m.eval(), opt


@pytest.mark.parametrize("eval_opt,exc", [
    ({"sample_max": 1, "sample_n": 2}, ValueError),                 # n identical greedy captions
    ({"sample_n": 3}, ValueError),                                  # sample_max defaults to 1
    ({"sample_max": 0, "sample_n": 2, "beam_size": 3}, ValueError),
    ({"sample_max": 0, "sample_n": 0}, ValueError),
    ({"sample_max": 0, "sample_n": 1.5}, ValueError),
])
def test_refusals_before_any_device_work(eval_opt, exc):
    """The refusals come before the prologue: no device is needed to see them."""
    m, opt = _cpu_model()
    x = torch.zeros(1)
    with pytest.raises(exc):
        m._sample(x, x, x, x, x, x, eval_opt)


def test_transformer_refuses_sample_n():
    m, opt = _cpu_model(att_model="transformer")
    x = torch.zeros(1)
    with pytest.raises(NotImplementedError):
        m._sample(x, x, x, x, x, x, {"sample_max": 0, "sample_n": 2})
    with pytest.raises(ValueError):                                 # beam_size > 1 is refused first, as for the top-down captioner
        m._sample(x, x, x, x, x, x, {"sample_max": 0, "sample_n": 2, "beam_size": 2})


# ------------------------------------------------------------------------------------------------------------ attn_group_kernel's grid
G_MAX = 8           # ATT_GMAX


def _cdiv(a, b):
    return -(-a // b)


def _emulate(B, div, R, T, RC, TC, dual=False, win=None):
    """attn_group_kernel's block decomposition and ticket protocol (csrc/gvd_decode.cu; keep in sync) for every CTA of the launch, in a
    shuffled completion order.  Returns the (row, chunk) records written, the out-of-window counts per row, the merging CTA of every row
    and the final tickets."""
    nch_r, nch_t = _cdiv(R, RC), 0 if dual else _cdiv(T, TC)
    nch = nch_r + nch_t
    ngroups = _cdiv(div, G_MAX)
    grid = (B // div) * ngroups * nch
    ticket = np.zeros(B, np.int64)
    records, n_out_rows, merged = {}, {}, {}
    for bid in np.random.RandomState(B * 31 + div).permutation(grid):
        c = bid % nch
        grp = (bid // nch) % ngroups
        fb = bid // nch // ngroups
        g0 = grp * G_MAX
        G = min(G_MAX, div - g0)
        b0 = fb * div + g0
        assert G >= 1 and 0 <= b0 and b0 + G <= B
        region = c < nch_r
        N = R if region else T
        chunk = RC if region else TC
        r0 = c * chunk if region else (c - nch_r) * chunk
        nrows = min(chunk, N - r0)
        n_out = 0
        if win is not None and not region:
            lo, hi = max(win[fb][0], 0), min(win[fb][1], N)
            wlo = min(lo, N)
            whi = max(hi, wlo)
            c0, c1 = max(r0, wlo), min(r0 + nrows, whi)
            if c == nch_r:
                n_out = N - (whi - wlo)
            r0, nrows = c0, max(c1 - c0, 0)
        for g in range(G):
            assert (b0 + g, c) not in records
            records[(b0 + g, c)] = (r0, nrows)
            if dual:
                assert (b0 + g, nch_r + c) not in records
                records[(b0 + g, nch_r + c)] = (r0, nrows)
            if n_out:
                n_out_rows[b0 + g] = n_out_rows.get(b0 + g, 0) + n_out
        last = ticket[b0] == nch - 1
        ticket[b0] += 1
        if last:
            for g in range(G):
                assert b0 + g not in merged
                merged[b0 + g] = bid
            ticket[b0] = 0
    return records, n_out_rows, merged, ticket, nch_r, nch_t


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("clips,div", [(4, 1), (5, 3), (2, 8), (3, 9), (2, 17), (1, 24)])
def test_every_row_chunk_once_and_one_merge_per_row(clips, div, dual):
    B, R, T, RC, TC = clips * div, 100, 37, 32, 16
    records, _, merged, ticket, nch_r, nch_t = _emulate(B, div, R, T, RC, TC, dual)
    nrec = 2 * nch_r if dual else nch_r + nch_t
    assert sorted(records) == [(b, c) for b in range(B) for c in range(nrec)]
    for (b, c), (r0, nrows) in records.items():
        cc = c % nch_r if dual else c
        region = cc < nch_r
        chunk = RC if region else TC
        assert r0 == (cc if region else cc - nch_r) * chunk and nrows == min(chunk, (R if region else T) - r0)
    assert sorted(merged) == list(range(B))
    assert not ticket.any()
    groups = {}                  # the merging CTA of a row is the last of its row group, which holds every one of the group's rows
    for b, bid in merged.items():
        groups.setdefault(bid, []).append(b)
    for rows in groups.values():
        assert len(rows) <= G_MAX and rows == list(range(rows[0], rows[0] + len(rows)))


@pytest.mark.parametrize("div", [2, 9])
def test_video_rows_windows(div):
    """Windowed temporal chunks: every row's chunks cover exactly its window ∩ [0, T), and the out-of-window count is recorded once per row
    (empty, past-T and negative windows included)."""
    T, TC, R, RC = 40, 16, 20, 16
    win = [(0, T), (5, 5), (T + 1, T + 4), (-3, 2), (14, 19), (T - 2, T + 6), (39, 40)]
    B = len(win) * div
    records, n_out, merged, ticket, nch_r, nch_t = _emulate(B, div, R, T, RC, TC, win=win)
    assert sorted(merged) == list(range(B)) and not ticket.any()
    for b in range(B):
        lo, hi = max(win[b // div][0], 0), min(win[b // div][1], T)
        inside = set(range(lo, hi)) if hi > lo else set()
        got = set()
        for c in range(nch_r, nch_r + nch_t):
            r0, nrows = records[(b, c)]
            assert not (got & set(range(r0, r0 + nrows)))
            got |= set(range(r0, r0 + nrows))
        assert got == inside
        assert n_out.get(b, 0) == T - len(inside)
