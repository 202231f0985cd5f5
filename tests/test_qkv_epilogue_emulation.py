"""CPU emulation of the store plan of ss_gemm_kernel's Q|K|V epilogue (ss_store_qkv in csrc/gvd_wgmma.cu) over every tile of a launch:
every word of Q's rows, of the per-head K image (padding words [HS, KH) included) and of the V^T image (pad rows [R, Rp) included) is
written exactly once, by an aligned store that carries the right column / row pair, and every shared-memory read stays inside the tile.

The kernel's loops are products of a row part and a column part (Q and K: warp <-> row, lane <-> columns of that row; V: lane <-> row of a
32-row line, unit <-> 4 columns), so each part is emulated over every tile on its own and the coverage of the product follows.  The loop
bodies below transliterate the kernel; keep them in sync with it."""
import numpy as np
import pytest

BM = BN = 128
NW = 8                      # consumer warps


def _word(k_even):
    return (k_even >> 5) * 32 + ((k_even & 31) >> 1)


def _layout(H, R, clips):
    nh = len(range(0, H, -(-H // 6)))
    HS = -(-(-(-H // 6)) // 4) * 4
    return dict(nh=nh, HS=HS, HP=nh * HS, KH=-(-HS // 32) * 32, R=R, Rp=-(-R // 32) * 32, M=clips * R)


CASES = [(1024, 1000, 7), (1024, 1000, 100), (1024, 64, 9), (1024, 998, 5), (512, 1000, 7), (512, 998, 3)]


def _rows_of_tile(m0, M):
    """row loop of the Q and K passes: warp w takes tile rows w, w + 8, ... below mend"""
    mend = min(m0 + BM, M)
    rows = []
    for warp in range(NW):
        r = warp
        while m0 + r < mend:
            rows.append(m0 + r)
            r += NW
    return rows


@pytest.mark.parametrize("H,R,clips", CASES)
def test_qkv_epilogue_rows_are_visited_once(H, R, clips):
    M = _layout(H, R, clips)["M"]
    seen = np.zeros(M, np.int32)
    for m0 in range(0, M, BM):
        np.add.at(seen, _rows_of_tile(m0, M), 1)
    assert (seen == 1).all()


@pytest.mark.parametrize("H,R,clips", CASES)
def test_qkv_epilogue_q_and_k_words_of_a_row_are_written_once(H, R, clips):
    L = _layout(H, R, clips)
    nh, HS, HP, KH = L["nh"], L["HS"], L["HP"], L["KH"]
    N, KQ = 3 * HP, KH // 4
    q_cnt = np.zeros(HP, np.int32)
    k_cnt = np.zeros(nh * KH, np.int32)
    k_src = {}                                                   # image word -> (head, column pair, hi | lo)
    for n0 in range(0, N, BN):
        if n0 < HP:                                              # Q pass
            for lane in range(32):
                c = 4 * lane
                if n0 + c < HP:
                    q_cnt[n0 + c:n0 + c + 4] += 1
        ka, kb = max(n0, HP) - HP, min(n0 + BN, 2 * HP) - HP
        if ka < kb:                                              # K pass
            hlo, hhi = ka // HS, (kb - 1) // HS
            q0 = hlo * KQ + ((ka - hlo * HS) >> 5) * 8
            q1 = (hhi + 1) * KQ if hhi * HS + HS - 4 < kb else hhi * KQ + (((kb - 1 - hhi * HS) >> 5) + 1) * 8
            for lane in range(32):
                for q in range(q0 + lane, q1, 32):
                    h = q // KQ
                    u = q - h * KQ
                    c, last = (u >> 3) * 32 + (u & 3) * 8, h * HS + HS - 4
                    d = h * KH + 4 * u
                    own = []
                    for e in range(2):
                        g = c + 4 * e
                        kc = h * HS + g
                        own.append(ka <= kc < kb if g < HS else ka <= last < kb)
                        if g < HS and own[e]:
                            assert 0 <= HP + kc - n0 <= BN - 4 and (HP + kc - n0) % 4 == 0    # float4 read inside the tile
                    if own[0] and own[1]:
                        assert d % 4 == 0
                        words = [(d, c), (d + 1, c + 2), (d + 2, c + 4), (d + 3, c + 6)]
                    elif own[0]:
                        assert d % 2 == 0
                        words = [(d, c), (d + 1, c + 2)]
                    elif own[1]:
                        assert (d + 2) % 2 == 0
                        words = [(d + 2, c + 4), (d + 3, c + 6)]
                    else:
                        words = []
                    for w, col in words:
                        k_cnt[w] += 1
                        k_src[w] = (h, col, u & 4)
    assert (q_cnt == 1).all()
    assert (k_cnt == 1).all()
    for w, (h, col, lo) in k_src.items():                        # the word holds the pair (col, col + 1) of head h, hi or lo
        assert w == h * KH + _word(col) + (16 if lo else 0)
    pads = {w for w, (h, col, _) in k_src.items() if col >= HS}
    assert len(pads) == nh * (KH - HS)


@pytest.mark.parametrize("H,R,clips", CASES)
def test_qkv_epilogue_vt_image_is_written_once(H, R, clips):
    L = _layout(H, R, clips)
    HP, R, Rp, M = L["HP"], L["R"], L["Rp"], L["M"]
    N = 3 * HP
    # column part: the V columns [va, vb) of every column tile, in 4-column groups
    v_cols = np.zeros(HP, np.int32)
    ngs = set()
    for n0 in range(0, N, BN):
        va, vb = max(n0, 2 * HP), min(n0 + BN, N)
        if va < vb:
            assert (vb - va) % 4 == 0
            ng = (vb - va) // 4
            ngs.add(ng)
            for g in range(ng):
                v_cols[va + 4 * g - 2 * HP:va + 4 * g - 2 * HP + 4] += 1
    assert (v_cols == 1).all()
    # row part: per row tile, the words (clip, word of the pair, hi | lo) its lanes own in one column
    cnt = np.zeros((M // R, Rp), np.int32)
    for m0 in range(0, M, BM):
        mend = min(m0 + BM, M)
        b = m0 // R
        while b * R < mend:
            base = b * R
            ra, rb = max(m0, base) - base, min(mend, base + R) - base
            k0 = ra >> 5
            nl = ((rb - 1) >> 5) - k0 + 1
            for ng in ngs:                                       # units t -> (line, column group): each once over the warps
                units = sorted(t for warp in range(NW) for t in range(warp, nl * ng, NW))
                assert units == list(range(nl * ng))
            for k in range(k0, k0 + nl):
                own = []
                for lane in range(32):
                    r = 32 * k + lane
                    assert r < Rp
                    o = (ra <= r < rb) if r < R else rb == R
                    if r < R and o:
                        assert 0 <= base + r - m0 < BM                        # the row is in the tile
                    own.append(o)
                    if o:
                        w = 32 * k + (lane & 1) * 16 + (lane >> 1)
                        assert w == _word(r & ~1) + (16 if lane & 1 else 0)
                        cnt[b, w] += 1
                assert all(own[l] == own[l ^ 1] for l in range(32))            # a row pair never straddles a tile
            b += 1
    assert (cnt == 1).all()
