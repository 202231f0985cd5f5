// gvd-b200: on-device beam search bookkeeping (reference: misc/CaptionModelBU.py:24-185 beam_step /
// beam_search, misc/model.py:700-742), batched over clips.  The reference moves every step's
// log-probs to the CPU, sorts there and loops over clips in Python; here each clip's beams are rows
// of one device batch and the per-step bookkeeping is two tiny kernels.
//
// Semantics reproduced (see oracle/gvd_oracle.py::sample_beam, pinned to the shimmed reference):
// candidates enumerated word-rank-major / beam-minor, STABLE sort by descending joint log-prob,
// no UNK suppression, finished beams (token 0 or last step) get their running sum set to -1000,
// and — because the reference records a finished beam's score / attention column as un-cloned
// views — the FIRST finished beam is the result, with its attention column read at the end.
#include "gvd_kernels.cuh"

namespace {

constexpr int BEAM_MAXK = 8;
constexpr int BEAM_MAXL = 64;

// per row: log_softmax and the K best (value desc, index asc on ties) — ys/ix of CaptionModelBU.py:45.  NaN words are skipped (no
// comparison with a NaN succeeds); a pick that finds only NaN left takes the lowest untaken index, so an all-NaN row gives 0 .. K-1 like a
// stable torch.sort(descending=True), and the token never leaves the vocabulary.  (torch ranks NaN first: rows only partly NaN differ.)
__global__ void __launch_bounds__(256) beam_topk_kernel(const float* __restrict__ logits, long long ld, int V, int K,
                                                        float* __restrict__ topv, int* __restrict__ topi) {
    __shared__ float red[32];
    __shared__ float wv[8];
    __shared__ int wi[8];
    __shared__ int chosen[BEAM_MAXK];
    __shared__ float chosen_v[BEAM_MAXK];
    const int row = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* x = logits + (long long)row * ld;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < V; i += blockDim.x) m = fmaxf(m, x[i]);
    m = block_max(m, red);
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(x[i] - m);
    s = block_sum(s, red);
    const float lse = m + logf(s);
    for (int k = 0; k < K; ++k) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = threadIdx.x; i < V; i += blockDim.x) {
            bool taken = false;
            for (int j = 0; j < k; ++j) taken |= (chosen[j] == i);
            const float v = x[i];
            if (!taken && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; ++w)
                if (wv[w] > bv || (wv[w] == bv && wi[w] < bi)) { bv = wv[w]; bi = wi[w]; }
            if (bi == 0x7fffffff) {                   // every untaken word is NaN
                bool taken = true;                    // the lowest untaken index: at most k < K <= V
                for (bi = 0; taken; bi += taken) {
                    taken = false;
                    for (int j = 0; j < k; ++j) taken |= (chosen[j] == bi);
                }
                bv = x[bi];
            }
            chosen[k] = bi;
            chosen_v[k] = bv;
        }
        __syncthreads();
    }
    if (threadIdx.x < K) {
        topv[(long long)row * K + threadIdx.x] = chosen_v[threadIdx.x] - lse;
        topi[(long long)row * K + threadIdx.x] = chosen[threadIdx.x];
    }
}

// per clip: merge K x K candidates, fork beams, record the first finished beam (beam_step + the
// "done" loop of beam_search).  One thread per clip: K <= 8, L <= 64.
__global__ void beam_update_kernel(BeamBufs bb, int B, int K, int L, int t) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    int* seq = bb.seq + (long long)b * L * K;
    float* lp = bb.lp + (long long)b * L * K;
    int* att = bb.att + (long long)b * L * K;
    float* sums = bb.sums + (long long)b * K;
    const float* ys = bb.topv + (long long)b * K * K;
    const int* ix = bb.topi + (long long)b * K * K;
    const int* att_ind = bb.att_ind + (long long)b * K;
    const int rows = t == 0 ? 1 : K;
    // candidate list in the reference's order (c-major, q-minor) + stable sort by -p
    float cp[BEAM_MAXK * BEAM_MAXK];
    unsigned char ord[BEAM_MAXK * BEAM_MAXK];
    int n = 0;
    for (int c = 0; c < K; ++c)
        for (int q = 0; q < rows; ++q) {
            const float p = sums[q] + ys[q * K + c];
            int pos = n;
            while (pos > 0 && cp[ord[pos - 1]] < p) { ord[pos] = ord[pos - 1]; --pos; }   // strict <: equal keys keep insertion order
            ord[pos] = (unsigned char)(c * BEAM_MAXK + q);
            cp[c * BEAM_MAXK + q] = p;
            ++n;
        }
    // fork: new beam v continues old beam q with word ix[q][c]
    int pq[BEAM_MAXK], ptok[BEAM_MAXK], pw[BEAM_MAXK];
    float pp[BEAM_MAXK], pr[BEAM_MAXK];
    for (int v = 0; v < K; ++v) {
        const int c = ord[v] / BEAM_MAXK, q = ord[v] % BEAM_MAXK;
        pq[v] = q; ptok[v] = ix[q * K + c]; pr[v] = ys[q * K + c]; pp[v] = cp[ord[v]]; pw[v] = att_ind[q];
    }
    if (t >= 1) {
        int old_seq[BEAM_MAXK], old_att[BEAM_MAXK];
        float old_lp[BEAM_MAXK];
        for (int tt = 0; tt < t; ++tt) {
            for (int v = 0; v < K; ++v) { old_seq[v] = seq[tt * K + v]; old_lp[v] = lp[tt * K + v]; old_att[v] = att[tt * K + v]; }
            for (int v = 0; v < K; ++v) { seq[tt * K + v] = old_seq[pq[v]]; lp[tt * K + v] = old_lp[pq[v]]; att[tt * K + v] = old_att[pq[v]]; }
        }
    }
    for (int v = 0; v < K; ++v) {
        seq[t * K + v] = ptok[v];
        lp[t * K + v] = pr[v];
        if (t >= 1) att[t * K + v] = pw[v];
        sums[v] = pp[v];
        bb.parent[(long long)b * K + v] = pq[v];
        if (bb.parent_hist) bb.parent_hist[((long long)t * B + b) * K + v] = pq[v];
        bb.tokens[(long long)b * K + v] = ptok[v];
    }
    for (int v = 0; v < K; ++v) {
        if (ptok[v] == 0 || t == L - 1) {
            if (!bb.done_flag[b]) {                       // first pushed beam wins (see file header)
                bb.done_flag[b] = 1;
                bb.done_slot[b] = v;
                if (bb.done_step) bb.done_step[b] = t;
                for (int tt = 0; tt < L; ++tt) {
                    bb.done_seq[(long long)b * L + tt] = tt <= t ? seq[tt * K + v] : 0;
                    bb.done_lp[(long long)b * L + tt] = tt <= t ? lp[tt * K + v] : 0.f;
                }
            }
            sums[v] = -1000.f;
        }
    }
}

// dst[b*K + v, :] = src[b*K + parent[b*K + v], :]
__global__ void beam_gather_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ parent, int K,
                                        int H) {
    const int row = blockIdx.x, b = row / K;
    const int srow = b * K + parent[row];
    for (int h = threadIdx.x * 4; h < H; h += blockDim.x * 4)
        *reinterpret_cast<float4*>(dst + (long long)row * H + h) = *reinterpret_cast<const float4*>(src + (long long)srow * H + h);
}

// first index of the row maximum (torch.max(att2_weight, 1)[1], CaptionModelBU.py:182); NaN entries are skipped, an all-NaN row gives 0
// like torch.argmax
__global__ void __launch_bounds__(256) row_argmax_kernel(const float* __restrict__ z, long long ld, int R, int* __restrict__ out) {
    __shared__ float wv[8];
    __shared__ int wi[8];
    const int row = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* x = z + (long long)row * ld;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
        const float v = x[i];
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w)
            if (wv[w] > bv || (wv[w] == bv && wi[w] < bi)) { bv = wv[w]; bi = wi[w]; }
        out[row] = bi == 0x7fffffff ? 0 : bi;      // no comparison succeeded: every entry NaN
    }
}

// results: seq/logps cloned when the winning beam finished; its attention column read now (view semantics)
__global__ void beam_finish_kernel(BeamBufs bb, const int* __restrict__ bos_att, int B, int K, int L, long long* __restrict__ seq_out,
                                   float* __restrict__ lp_out, long long* __restrict__ att_out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * L) return;
    const int b = idx / L, t = idx % L;
    seq_out[idx] = bb.done_seq[idx];
    lp_out[idx] = bb.done_lp[idx];
    att_out[idx] = t == 0 ? bos_att[b * K] : bb.att[((long long)b * L + t) * K + bb.done_slot[b]];
}

// The region-attention logits the returned caption used (one CTA per clip).  Word t of the beam in slot s at step t was picked from the
// logits of old row parent_t[s] of step t, and that row is the beam's slot at step t - 1: walking the parents back from (done_step,
// done_slot) gives the row of every step.  hist holds step t's rows [B*K][R] at hist + t * step_stride.  out [B][L][R]: the rows up to
// the finishing step, zeros after it.  VEC: R, step_stride and both pointers allow float4 accesses.
template <bool VEC>
__global__ void __launch_bounds__(256) beam_backtrack_kernel(BeamBufs bb, const float* __restrict__ hist, long long step_stride, int B, int K,
                                                             int L, int R, float* __restrict__ out) {
    __shared__ int par[BEAM_MAXL * BEAM_MAXK];
    __shared__ int src[BEAM_MAXL];
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < L * K; i += blockDim.x) par[i] = bb.parent_hist[((long long)(i / K) * B + b) * K + i % K];
    __syncthreads();
    const int tf = bb.done_step[b];
    if (threadIdx.x == 0) {
        int slot = bb.done_slot[b];
        for (int t = tf; t >= 0; --t) {
            slot = par[t * K + slot];
            src[t] = b * K + slot;
        }
    }
    __syncthreads();
    float* o = out + (long long)b * L * R;
    if (VEC) {
        const int R4 = R / 4;
        for (int i = threadIdx.x; i < L * R4; i += blockDim.x) {
            const int t = i / R4, c = i - t * R4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t <= tf) v = __ldg(reinterpret_cast<const float4*>(hist + t * step_stride + (long long)src[t] * R) + c);
            reinterpret_cast<float4*>(o + (long long)t * R)[c] = v;
        }
    } else {
        for (int i = threadIdx.x; i < L * R; i += blockDim.x) {
            const int t = i / R, c = i - t * R;
            o[i] = t <= tf ? __ldg(hist + t * step_stride + (long long)src[t] * R + c) : 0.f;
        }
    }
}

}  // namespace

int gvd_beam_topk(const float* logits, long long ld, int rows, int V, int K, float* topv, int* topi, cudaStream_t st) {
    GVD_REQUIRE(K >= 1 && K <= BEAM_MAXK && K <= V, "beam: beam_size must be in [1,%d]", BEAM_MAXK);
    beam_topk_kernel<<<rows, 256, 0, st>>>(logits, ld, V, K, topv, topi);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_beam_update(const BeamBufs& bb, int B, int K, int L, int t, cudaStream_t st) {
    GVD_REQUIRE(K <= BEAM_MAXK && L <= BEAM_MAXL, "beam: beam_size <= %d and seq_length <= %d", BEAM_MAXK, BEAM_MAXL);
    beam_update_kernel<<<gvd_cdiv(B, 32), 32, 0, st>>>(bb, B, K, L, t);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_beam_gather_rows(const float* src, float* dst, const int* parent, int B, int K, int H, cudaStream_t st) {
    beam_gather_rows_kernel<<<B * K, 256, 0, st>>>(src, dst, parent, K, H);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_row_argmax(const float* z, long long ld, int rows, int R, int* out, cudaStream_t st) {
    row_argmax_kernel<<<rows, 256, 0, st>>>(z, ld, R, out);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_beam_finish(const BeamBufs& bb, const int* bos_att, int B, int K, int L, long long* seq_out, float* lp_out, long long* att_out,
                    cudaStream_t st) {
    beam_finish_kernel<<<gvd_cdiv((long long)B * L, 256), 256, 0, st>>>(bb, bos_att, B, K, L, seq_out, lp_out, att_out);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_beam_backtrack(const BeamBufs& bb, const float* hist, long long step_stride, int B, int K, int L, int R, float* out, cudaStream_t st) {
    GVD_REQUIRE(bb.parent_hist && bb.done_step && K <= BEAM_MAXK && L <= BEAM_MAXL, "beam: backtrack needs the parent history");
    const bool vec = R % 4 == 0 && step_stride % 4 == 0 && ((uintptr_t)hist & 15) == 0 && ((uintptr_t)out & 15) == 0;
    if (vec)
        beam_backtrack_kernel<true><<<B, 256, 0, st>>>(bb, hist, step_stride, B, K, L, R, out);
    else
        beam_backtrack_kernel<false><<<B, 256, 0, st>>>(bb, hist, step_stride, B, K, L, R, out);
    GVD_CHECK_LAUNCH();
    return 0;
}
