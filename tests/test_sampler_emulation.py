"""Thread-level emulation (numpy, on the CPU) of the three greedy samplers' top-2 / log-sum-exp merges, in the manner of
test_kernel_index_emulation.py: literal transliterations of

  reduce_pick_kernel<NPT>   csrc/gvd_skinny.cu   1024 threads, NPT strided logits each, warp butterfly, `wtop` second butterfly
  greedy_pick_kernel        csrc/gvd_decode.cu   256 threads, strided loop, warp butterfly, serial merge of the 8 warp results
  MODE_PICK                 csrc/gvd_wgmma.cu    one thread per (row, 64-column tile), partial (max, sum-exp, top-2) per CTA, merged in
                                                 CTA order by the last CTA

run on the tie / UNK rows of sampler_ref.special_rows and compared with sampler_ref.pick_reference.  This pins the tie rule (lower
index wins at every level of every merge tree) without a GPU; tests/test_gpu_decode_ops.py runs the kernels on the same rows.  Keep the
transliterations in sync with the .cu files when those change."""
import numpy as np
import pytest

from sampler_ref import KINDS, pick_reference, special_rows

NEG = -np.inf
BIG = 0x7FFFFFFF
F = np.float32


def top2_insert(t, v, i):
    v1, v2, i1, i2 = t
    if v > v1 or (v == v1 and i < i1):
        return (v, v1, i, i1)
    if v > v2 or (v == v2 and i < i2):
        return (v1, v, i1, i)
    return t


def butterfly(lanes):
    """#pragma unroll for (o = 16; o > 0; o >>= 1): every lane inserts both entries of lane ^ o (values read before anyone updates)"""
    o = 16
    while o:
        old = list(lanes)
        for lane in range(32):
            ov1, ov2, oi1, oi2 = old[lane ^ o]
            lanes[lane] = top2_insert(top2_insert(old[lane], ov1, oi1), ov2, oi2)
        o >>= 1
    return lanes


def finish(t, lse, unk, V):
    v1, v2, i1, i2 = t
    keep = i1 != unk
    it = i1 if keep else i2
    if not 0 <= it < V:
        it = 0
    return it, F(v1 if keep else v2) - lse


def emulate_reduce_pick(x, unk):
    V = len(x)
    NT = 1024
    NPT = 2 if V <= 2 * NT else (5 if V <= 5 * NT else 6)
    assert V <= NT * NPT
    per_thread = []
    for tid in range(NT):
        t = (NEG, NEG, BIG, BIG)
        for k in range(NPT):
            i = tid + k * NT
            if i < V:
                t = top2_insert(t, x[i], i)
        per_thread.append(t)
    wtop = [butterfly(per_thread[w * 32:(w + 1) * 32])[0] for w in range(32)]
    t = butterfly(list(wtop))[0]                                    # thread 0: lane 0 of the second butterfly
    m = F(t[0])
    s = F(np.exp((x.astype(F) - m)).sum(dtype=F))
    return finish(t, m + np.log(s, dtype=F), unk, V)


def emulate_greedy_pick(x, unk):
    V = len(x)
    per_thread = []
    for tid in range(256):
        t = (NEG, NEG, BIG, BIG)
        for i in range(tid, V, 256):
            t = top2_insert(t, x[i], i)
        per_thread.append(t)
    wtop = [butterfly(per_thread[w * 32:(w + 1) * 32])[0] for w in range(8)]
    t = wtop[0]
    for wv in range(1, 8):
        t = top2_insert(t, wtop[wv][0], wtop[wv][2])
        t = top2_insert(t, wtop[wv][1], wtop[wv][3])
    m = F(t[0])
    s = F(np.exp((x.astype(F) - m)).sum(dtype=F))
    return finish(t, m + np.log(s, dtype=F), unk, V)


def emulate_mode_pick(x, unk):
    V = len(x)
    part = []
    for cta in range((V + 63) // 64):                               # per-CTA partial of this row's thread
        n0 = cta * 64
        mloc, v1, v2, i1, i2 = F(NEG), NEG, NEG, BIG, BIG
        xs = []
        for j in range(64):
            n = n0 + j
            v = F(x[n]) if n < V else F(NEG)
            xs.append(v)
            mloc = max(mloc, v)
            if v > v1 or (v == v1 and n < i1):
                v2, i2, v1, i1 = v1, i1, v, n
            elif v > v2 or (v == v2 and n < i2):
                v2, i2 = v, n
        with np.errstate(invalid="ignore"):
            sloc = F(sum((np.exp(F(v - mloc)) for j, v in enumerate(xs) if n0 + j < V), F(0)))
        part.append((mloc, sloc, v1, i1, v2, i2))
    M, S, t = F(NEG), F(0), (NEG, NEG, BIG, BIG)
    for mloc, sloc, v1, i1, v2, i2 in part:                         # fixed CTA order
        if mloc > M:
            S = F(S * np.exp(F(M - mloc)) + sloc)
            M = mloc
        elif mloc > NEG:
            S = F(sloc * np.exp(F(mloc - M)) + S)
        for cv, ci in ((v1, i1), (v2, i2)):
            t = top2_insert(t, cv, ci)
    return finish(t, M + np.log(S, dtype=F), unk, V)


EMULATIONS = {"reduce_pick": emulate_reduce_pick, "greedy_pick": emulate_greedy_pick, "mode_pick": emulate_mode_pick}


@pytest.mark.parametrize("V,unk", [(2, 1), (2, 0), (64, 63), (65, 64), (301, 300), (301, 0), (2049, 1024), (2049, 2048), (4905, 4904)])
@pytest.mark.parametrize("name", sorted(EMULATIONS))
def test_sampler_merge_trees_follow_the_tie_rule(name, V, unk):
    x, kinds = special_rows(len(KINDS), V, unk, seed=V + unk)
    want_tok, want_lp = pick_reference(x, unk)
    for b in range(x.shape[0]):
        tok, lp = EMULATIONS[name](x[b], unk)
        assert tok == want_tok[b], (kinds[b], tok, want_tok[b])
        assert abs(float(lp) - want_lp[b]) <= 1e-5, (kinds[b], float(lp), want_lp[b])


@pytest.mark.parametrize("name", sorted(EMULATIONS))
def test_sampler_emulations_on_random_and_masked_rows(name):
    """Continuous random logits (no ties), then the same rows with masked (-inf) words, one whole 64-column tile among them."""
    rs = np.random.RandomState(3)
    for V, unk in [(301, 300), (1500, 7)]:
        x = (rs.randn(6, V) * 3).astype(np.float32).astype(np.float64)
        x[3:, 64:128] = NEG
        x[3:, rs.choice(V, 40, replace=False)] = NEG
        want_tok, want_lp = pick_reference(x, unk)
        for b in range(x.shape[0]):
            tok, lp = EMULATIONS[name](x[b], unk)
            assert tok == want_tok[b] and abs(float(lp) - want_lp[b]) <= 1e-5, (b, tok, want_tok[b], float(lp), want_lp[b])


def test_reference_rule_by_hand():
    x = np.array([[1.0, 3.0, 3.0, 2.0],       # tie: the lower index
                  [1.0, 3.0, 2.0, 3.0],       # unk (3) ties with a lower index: the lower index, unk never on top
                  [0.0, 1.0, 2.0, 5.0],       # unk on top: the runner-up
                  [4.0, 4.0, 4.0, 4.0]])      # all equal: index 0
    tok, lp = pick_reference(x, 3)
    assert tok.tolist() == [1, 1, 2, 0]
    lse = np.log(np.exp(x).sum(1))
    assert np.allclose(lp, x[np.arange(4), tok] - lse, atol=1e-12)
    tok0, _ = pick_reference(x, 0)
    assert tok0.tolist() == [1, 1, 3, 1]      # unk = 0 wins the all-equal row, so its runner-up (index 1) is taken
