"""Thread-level emulation (numpy, on the CPU) of the INDEX ARITHMETIC of kernels whose indexing is easy to get wrong
(csrc/gvd_train.cu, the two grounding kernels of csrc/gvd_losses.cu, the epilogues of csrc/gvd_wgmma.cu).  Each emulation below is a literal
transliteration of the kernel body — same flattened-index expressions, same block / thread decomposition, same shared-memory tile
phases — run for every (block, thread) of a small launch and compared with the primitive's mathematical definition.  It cannot find
device-only problems (synchronisation, alignment), but a wrong stride, a swapped axis or an off-by-one tile is caught here instead of
on the GPU.  Keep the transliterations in sync with the .cu files when those change."""
import numpy as np
import torch

from ops_ref import TorchRefOps

R_ = TorchRefOps()
rs = np.random.RandomState(0)


def f32(*shape):
    return rs.randn(*shape).astype(np.float32)


def test_grounding_gather_kernel():
    B, L, NF, P, C = 3, 4, 5, 7, 7
    ppls, idx = f32(B, NF * P, C).ravel(), rs.randint(0, P, size=B * L * NF)
    n = B * L * NF * C
    boxes = np.zeros(n, np.float32)
    for t in range(n):                                   # one thread per (b, j, f, c)
        c = t % C
        e = t // C
        f = e % NF
        b = e // (NF * L)
        r = f * P + idx[e]
        boxes[t] = ppls[(b * NF * P + r) * C + c]
    want = np.zeros((B, L, NF, C), np.float32)
    p3, i4 = ppls.reshape(B, NF * P, C), idx.reshape(B, L, NF)
    for b in range(B):
        for j in range(L):
            for f in range(NF):
                want[b, j, f] = p3[b, f * P + i4[b, j, f]]
    assert np.array_equal(boxes.reshape(want.shape), want)


def test_class_target_and_cls_nll_kernels():
    B, R, NB, C = 2, 6, 3, 5
    ov, gt = rs.rand(B, R, NB).astype(np.float32), f32(B, NB, 6)
    gt[:, :, 5] = rs.randint(1, C, size=(B, NB))
    total = B * NB * R
    target = np.zeros(total, np.int32)
    for idx in range(total):                             # class_target_kernel: idx = (b, k, r)
        r, k = idx % R, (idx // R) % NB
        b = idx // (R * NB)
        target[idx] = int(gt.ravel()[(b * NB + k) * 6 + 5]) if ov.ravel()[(b * R + r) * NB + k] > 0.5 else 0
    want_t = ((torch.from_numpy(ov) > 0.5).long() * torch.from_numpy(gt[:, :, 5]).view(B, 1, -1).long()).permute(0, 2, 1)
    assert np.array_equal(target.reshape(B, NB, R), want_t.numpy())
    simT = torch.softmax(torch.from_numpy(f32(B, R, C)), -1)
    n = int((target > 0).sum())
    part, dsim = np.zeros(total, np.float32), np.zeros(B * R * C, np.float32)
    for idx in range(total):                             # cls_nll_kernel
        r = idx % R
        b = idx // (R * NB)
        t = target[idx]
        if t > 0:
            e = (b * R + r) * C + t
            p = simT.numpy().ravel()[e]
            part[idx] = -max(np.log(p), -100.0)
            dsim[e] += -(1.0 / n) / p
    loss, d = R_.cls_nll(simT, torch.from_numpy(target.reshape(B, NB, R)).long())
    assert abs(part.sum() / n - float(loss)) < 1e-5 and np.allclose(dsim.reshape(B, R, C), d.numpy(), atol=1e-6)


def test_elementwise_row_and_cell_kernels_index_math():
    B, N, H = 3, 5, 4
    a, v = f32(B, N), f32(B, H)
    out = np.zeros(B * N * H, np.float32)
    for i in range(B * N * H):                           # outer_rows_kernel
        h = i % H
        bn = i // H
        out[i] = a.ravel()[bn] * v.ravel()[(bn // N) * H + h]
    assert np.allclose(out.reshape(B, N, H), R_.outer_rows(torch.from_numpy(a), torch.from_numpy(v)).numpy())
    # lstm_cell_fwd / bwd: g0 = b*4H + j
    Bc, Hc = 3, 4
    gates, c = f32(Bc, 4 * Hc), f32(Bc, Hc)
    sig = lambda x: 1.0 / (1.0 + np.exp(-x))
    h2, c2, act = np.zeros(Bc * Hc, np.float32), np.zeros(Bc * Hc, np.float32), np.zeros(Bc * 4 * Hc, np.float32)
    gf, cf = gates.ravel(), c.ravel()
    for idx in range(Bc * Hc):
        j = idx % Hc
        b = idx // Hc
        g0 = b * 4 * Hc + j
        i_, f_, g_, o_ = sig(gf[g0]), sig(gf[g0 + Hc]), np.tanh(gf[g0 + 2 * Hc]), sig(gf[g0 + 3 * Hc])
        cc = f_ * cf[idx] + i_ * g_
        c2[idx], h2[idx] = cc, o_ * np.tanh(cc)
        act[g0], act[g0 + Hc], act[g0 + 2 * Hc], act[g0 + 3 * Hc] = i_, f_, g_, o_
    rh, rc, ra = R_.lstm_cell(torch.from_numpy(gates), torch.from_numpy(c))
    assert np.allclose(h2.reshape(Bc, Hc), rh.numpy(), atol=1e-6) and np.allclose(c2.reshape(Bc, Hc), rc.numpy(), atol=1e-6)
    assert np.allclose(act.reshape(Bc, 4 * Hc), ra.numpy(), atol=1e-6)
    dh, dc = f32(Bc, Hc), f32(Bc, Hc)
    dg, dcp = np.zeros(Bc * 4 * Hc, np.float32), np.zeros(Bc * Hc, np.float32)
    for idx in range(Bc * Hc):
        j = idx % Hc
        b = idx // Hc
        g0 = b * 4 * Hc + j
        i_, f_, g_, o_ = act[g0], act[g0 + Hc], act[g0 + 2 * Hc], act[g0 + 3 * Hc]
        tc = np.tanh(c2[idx])
        d2 = dc.ravel()[idx] + dh.ravel()[idx] * o_ * (1 - tc * tc)
        dg[g0], dg[g0 + Hc], dg[g0 + 2 * Hc], dg[g0 + 3 * Hc] = d2 * g_ * i_ * (1 - i_), d2 * cf[idx] * f_ * (1 - f_), d2 * i_ * (1 - g_ * g_), dh.ravel()[idx] * tc * o_ * (1 - o_)
        dcp[idx] = d2 * f_
    rg, rdc = R_.lstm_cell_bwd(torch.from_numpy(dh), torch.from_numpy(dc), ra, torch.from_numpy(c), rc)
    assert np.allclose(dg.reshape(Bc, 4 * Hc), rg.numpy(), atol=1e-5) and np.allclose(dcp.reshape(Bc, Hc), rdc.numpy(), atol=1e-5)
    # gru_cell_fwd / bwd: g0 = b*3G + j
    G = 5
    gi, gh, hh = f32(Bc, 3 * G), f32(Bc, 3 * G), f32(Bc, G)
    o_h, o_r, o_z, o_n = (np.zeros(Bc * G, np.float32) for _ in range(4))
    for idx in range(Bc * G):
        j = idx % G
        b = idx // G
        g0 = b * 3 * G + j
        r = sig(gi.ravel()[g0] + gh.ravel()[g0]); z = sig(gi.ravel()[g0 + G] + gh.ravel()[g0 + G])
        n = np.tanh(gi.ravel()[g0 + 2 * G] + r * gh.ravel()[g0 + 2 * G])
        o_h[idx], o_r[idx], o_z[idx], o_n[idx] = (1 - z) * n + z * hh.ravel()[idx], r, z, n
    for got, want in zip((o_h, o_r, o_z, o_n), R_.gru_cell(torch.from_numpy(gi), torch.from_numpy(gh), torch.from_numpy(hh))):
        assert np.allclose(got.reshape(Bc, G), want.numpy(), atol=1e-6)
    # att_scores_fwd (one warp per (b, n) row) and _bwd (flat over [B, N, A])
    Ba, Na, A = 2, 3, 40
    p, q, w, bias = f32(Ba, Na, A), f32(Ba, A), f32(A), f32(1)
    s = np.zeros(Ba * Na, np.float32)
    for row in range(Ba * Na):
        b = row // Na
        acc = 0.0
        for lane in range(32):
            for a_ in range(lane, A, 32):
                acc += w[a_] * np.tanh(p.ravel()[row * A + a_] + q.ravel()[b * A + a_])
        s[row] = acc + bias[0]
    assert np.allclose(s.reshape(Ba, Na), R_.att_scores(*(torch.from_numpy(x) for x in (p, q, w, bias))).numpy(), atol=1e-5)
    ds = f32(Ba, Na)
    dpre, dst = np.zeros(Ba * Na * A, np.float32), np.zeros(Ba * Na * A, np.float32)
    for i in range(Ba * Na * A):
        a_ = i % A
        row = i // A
        b = row // Na
        t = np.tanh(p.ravel()[i] + q.ravel()[b * A + a_])
        dpre[i], dst[i] = ds.ravel()[row] * w[a_] * (1 - t * t), ds.ravel()[row] * t
    rp, rq, rw, rb = R_.att_scores_bwd(*(torch.from_numpy(x) for x in (ds, p, q, w)))
    assert np.allclose(dpre.reshape(Ba, Na, A), rp.numpy(), atol=1e-5)
    # dq = batched colsum (batch = B, M = N rows, N = A columns), dw = colsum over all rows of dst
    dq = np.zeros(Ba * A, np.float32)
    for z in range(Ba):                                  # colsum_kernel: out[z*N + n] = sum_m x[z*M*N + m*N + n]
        for n_ in range(A):
            dq[z * A + n_] = sum(dpre[z * Na * A + m * A + n_] for m in range(Na))
    assert np.allclose(dq.reshape(Ba, A), rq.numpy(), atol=1e-5) and np.allclose(dst.reshape(-1, A).sum(0), rw.numpy(), atol=1e-5)


def test_gather_index_add_mean_kernels():
    table, idx = f32(9, 4), rs.randint(0, 9, size=6)
    D = 4
    out = np.zeros(6 * D, np.float32)
    for i in range(6 * D):                               # gather_rows_kernel
        out[i] = table.ravel()[idx[i // D] * D + (i % D)]
    assert np.array_equal(out.reshape(6, D), table[idx])
    rows = f32(6, D)
    acc = np.zeros((9, D), np.float32)
    for r in range(9):                                   # index_add_rows_kernel: one block per output row
        for d in range(D):
            acc[r, d] = sum(rows[m, d] for m in range(6) if idx[m] == r)
    assert np.allclose(acc, R_.index_add_rows(9, torch.from_numpy(idx), torch.from_numpy(rows)).numpy(), atol=1e-6)
    B, T, F = 2, 3, 5
    x = f32(B, T, F)
    m = np.zeros(B * F, np.float32)
    for i in range(B * F):                               # mean_dim1_kernel
        f = i % F
        b = i // F
        m[i] = sum(x.ravel()[(b * T + t) * F + f] for t in range(T)) / T
    assert np.allclose(m.reshape(B, F), x.mean(1), atol=1e-6)


def _emulate_reduce_tiles(part, S, H, ldp, B, ngate):
    """reduce_lstm_kernel / reduce_bias_T_kernel phase 1 + phase 2 tile logic: returns v[g][b][j] = sum_s part[s][(g*H + j)][b]."""
    plane = ngate * H * ldp
    out = np.zeros((ngate, B, H), np.float32)
    for bx in range(-(-H // 32)):
        for by in range(-(-B // 32)):
            tile = np.zeros((ngate, 32, 33), np.float32)
            j0, b0 = bx * 32, by * 32
            for ty in range(8):
                for tx in range(32):
                    for i in range(4):                   # phase 1: tx -> b, ty -> unit
                        jl = ty + 8 * i
                        j, b = j0 + jl, b0 + tx
                        for g in range(ngate):
                            v = 0.0
                            if j < H and b < B:
                                base = (g * H + j) * ldp + b
                                for s in range(S):
                                    v += part[base + s * plane]
                            tile[g, jl, tx] = v
            for ty in range(8):
                for tx in range(32):
                    for i in range(4):                   # phase 2: tx -> unit, ty -> b
                        bl = ty + 8 * i
                        b, j = b0 + bl, j0 + tx
                        if b < B and j < H:
                            for g in range(ngate):
                                out[g, b, j] = tile[g, tx, bl]
    return out


def test_split_k_as_batch_axis_is_the_full_contraction():
    """gvd_skinny_splitk: batch entry s of the batched NT GEMM reads columns [s.Ks, (s+1).Ks) of BOTH operands (batch stride = Ks
    elements along K, same row pitch); the partials summed over s are the full product, in the transposed [Nw, B] layout."""
    Nw, B, Ktot, S = 10, 6, 96, 3
    W, X = f32(Nw, Ktot), f32(B, Ktot)
    Ks = Ktot // S
    part = np.zeros((S, Nw, B), np.float32)
    for s in range(S):
        A_s = W.ravel()[s * Ks:].reshape(-1)             # base pointer advanced by the batch stride
        X_s = X.ravel()[s * Ks:].reshape(-1)
        for m in range(Nw):
            for n in range(B):
                part[s, m, n] = sum(A_s[m * Ktot + k] * X_s[n * Ktot + k] for k in range(Ks))      # lda = ldw = Ktot, K = Ks
    assert np.allclose(part.sum(0), W @ X.T, atol=1e-4)


# ----------------------------------------------------------------------------- epilogues of wg_gemm_kernel (csrc/gvd_wgmma.cu)
def _f16x3_word(k_even):
    """gvd_common.cuh::f16x3_word: word of the hi half of the fp16 pair (k, k + 1) inside a row image (32-wide K slices: 16 hi words | 16 lo words)."""
    return (k_even >> 5) * 32 + ((k_even & 31) >> 1)


def test_fragment_to_row_exchange_is_a_bijection():
    """wg_gemm_kernel's exchange of the wgmma accumulator fragments through shared memory: thread (warpgroup, warp, lane) writes, for each of the
    8 column blocks j, float2 pairs at rows r0 and r0 + 8; together the 256 consumer threads write every element of the 128 x 64 tile exactly once
    (pitch 68 words, 8-byte aligned), and the row-per-thread readers (row = (warp & 3) * 32 + lane, column half = warp >> 2) read all of it."""
    LDS, tile = 68, {}
    for warp in range(8):
        wg = warp >> 2
        for lane in range(32):
            r0, c0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), 2 * (lane & 3)
            for j in range(8):
                for rr, e0 in ((r0, 4 * j), (r0 + 8, 4 * j + 2)):
                    addr = rr * LDS + 8 * j + c0
                    assert addr % 2 == 0
                    for e in range(2):
                        assert addr + e not in tile
                        tile[addr + e] = (rr, 8 * j + c0 + e, e0 + e)
    assert len(tile) == 128 * 64 and all(a == r * LDS + c for a, (r, c, _) in tile.items())
    read = set()
    for warp in range(8):
        for lane in range(32):
            row, cbeg = (warp & 3) * 32 + lane, (warp >> 2) * 32
            for j in range(0, 32, 4):
                assert (row * LDS + cbeg + j) % 4 == 0        # float4 reads
                read.update(row * LDS + cbeg + j + e for e in range(4))
    assert read == set(tile)


def test_pv_epilogue_image_covers_every_word_of_the_row_once():
    """The P.V image epilogue of wg_gemm_kernel (reference-size heads: 6 heads of 171 / 169 columns in slots of 172, padded width 176 = three
    64-column tiles of two 32-column halves): over all (head, tile, column half, 4-column chunk) the stores of one row write every word of the Wo
    operand image row [0, rup32(6 * 172) = 1056) exactly once — head columns through the chunk loop, the K padding through the zeroing loop of
    the last head's first tile — with 8-byte aligned word pairs that never straddle a 32-wide K slice; pad columns (n >= N) carry zeros."""
    nh, sCh, bn, img_ld = 6, 172, 176, 1056
    N = [171] * 5 + [169]
    slot, written, zero_cols = min(bn, sCh), {}, set()
    for zh in range(nh):
        for bx in range(-(-bn // 64)):
            for cbeg in (0, 32):
                if zh == nh - 1 and bx == 0 and cbeg == 0:        # K padding of the Wo operand: zeros
                    for gc in range(nh * sCh, img_ld, 4):
                        w = _f16x3_word(gc)
                        for d in (w, w + 1, w + 16, w + 17):
                            assert d not in written
                            written[d] = "pad"
                for j in range(0, 32, 4):
                    n = bx * 64 + cbeg + j
                    if n >= slot:
                        continue                                  # columns past the slot belong to the next head's CTA
                    gc = zh * sCh + n
                    assert gc % 4 == 0 and (gc & 31) + 4 <= 32    # the chunk sits inside one K slice
                    w = _f16x3_word(gc)
                    assert w % 2 == 0                             # uint2 stores: 8-byte aligned
                    for d in (w, w + 1, w + 16, w + 17):
                        assert d not in written and 0 <= d < img_ld
                        written[d] = (zh, n)
                    zero_cols.update(zh * sCh + n + e for e in range(4) if n + e >= N[zh])
    assert sorted(written) == list(range(img_ld))
    assert zero_cols == {zh * sCh + n for zh in range(nh) for n in range(N[zh], sCh)}
