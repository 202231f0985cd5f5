// Multi-head attention of the transformer captioner's decoder for the training step (gvd_b200/train.py, att_model = 'transformer'):
// the causal self-attention and the attention over the encoder output of both DecoderLayers (misc/transformer.py:92-123), forward and
// backward, with the reference's attention-probability dropout (transformer.py:105).
//
// Shapes: Q [B, Lq, H], K and V [B, N, H] already projected (wq / wk / wv), O [B, Lq, H] with the heads concatenated (torch.cat order).
// Heads are the torch.chunk(6, -1) column ranges (171 x 5 + 169 at H = 1024), read in place.  Scores are q.k * scale (scale = 1 / sqrt(d_model),
// quirk Q1); `causal` gives query row t the keys r <= t, which is what the reference's `- 1e10` on the raw dot products does (those
// probabilities are exactly 0 in fp32).  There is no key mask.
//
// Regime: Lq <= 64 queries and N <= 1000 keys.  At these shapes the work is bound by reading K and V (B = 100 region cross-attention: 819 MB of
// K and V), so the kernels use fp32 CUDA cores: one CTA per (head, clip) holds every query row of the head in shared memory and streams
// that head's K and V once, KT keys at a time.
//   forward : online softmax over the key chunks; saves lse[b, head, t] = max + log(sum) for the backward.
//   backward: recomputes P = exp(s - lse); D = rowsum(dO * O) per head (also with dropout); dV and dK of a chunk are complete when the chunk
//             is done (every query row is in the CTA), so they are stored without atomics; dQ accumulates in registers.
// Dropout: element (b, t, r) of head h keeps with the mask gvd_tr_dropout draws for element (b * Lq + t) * N + r of the contiguous [B, Lq, N]
// probability tensor of that head at site `site_base + h`; the dropped probabilities are kept * 1 / (1 - p).  The backward regenerates the
// mask.  All sums run in a fixed order: a relaunch is bit-identical.
#include "../../include/gvd_b200.h"
#include "gvd_common.cuh"

namespace {

constexpr int MHA_THREADS = 256;                 // 16 x 16 thread grid
constexpr int MHA_MAX_LQ = 64;                   // query rows: ty + 16 i, i < 4
constexpr int MHA_MAX_N = 1000;
constexpr int MHA_MAX_HS = 192;                  // head width: tx + 16 j, j < 12
constexpr int MHA_KT = 32;                       // keys per chunk: tx + 16 j, j < 2 (one per lane in the row pass)
constexpr int MHA_HEADS = 6;                     // n_heads of the captioner (misc/model.py:140)
constexpr int RI = MHA_MAX_LQ / 16, CJ = MHA_MAX_HS / 16, KJ = MHA_KT / 16;
constexpr int PS = MHA_KT + 1;                   // row stride of the [Lq, KT] score tiles

struct MhaDrop {
    float p, inv_keep;
    uint32_t seed_lo, seed_hi, site_base, step_lo, step_hi;
};

// gvd_tr_dropout's keep decision for element i of the tensor at `site`
__device__ __forceinline__ bool mha_keep(long long i, const MhaDrop& d, uint32_t site) {
    const unsigned long long q = (unsigned long long)i >> 2;
    uint32_t r[4];
    philox4x32_10((uint32_t)q, site, d.step_lo ^ (uint32_t)(q >> 32), d.step_hi, d.seed_lo, d.seed_hi, r);
    return (float)(r[i & 3] >> 8) * (1.f / 16777216.f) >= d.p;
}

// rows [0, rows) x cols [0, hs) of a row-major global tile with row stride ld -> shared memory with row stride sp; rows [rows, cap) zeroed
__device__ __forceinline__ void mha_load(float* __restrict__ s, const float* __restrict__ g, long long ld, int rows, int cap, int hs, int sp) {
    for (int idx = threadIdx.x; idx < cap * hs; idx += MHA_THREADS) {
        const int r = idx / hs, c = idx - r * hs;
        s[r * sp + c] = r < rows ? g[(long long)r * ld + c] : 0.f;
    }
}

__global__ void __launch_bounds__(MHA_THREADS) mha_fwd_kernel(const float* __restrict__ Q, const float* __restrict__ K, const float* __restrict__ V,
                                                             float* __restrict__ O, float* __restrict__ lse, int Lq, int N, int H, int chunk,
                                                             int causal, float scale, MhaDrop drop) {
    extern __shared__ float sm[];
    const int h = blockIdx.x, b = blockIdx.y, nh = gridDim.x;
    const int off = h * chunk, hs = min(chunk, H - off), sp = hs | 1;
    float* Qs = sm;
    float* Ks = Qs + Lq * sp;
    float* Vs = Ks + MHA_KT * sp;
    float* Ps = Vs + MHA_KT * sp;
    float* mrow = Ps + MHA_MAX_LQ * PS;
    float* lrow = mrow + MHA_MAX_LQ;
    float* arow = lrow + MHA_MAX_LQ;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    mha_load(Qs, Q + (long long)b * Lq * H + off, H, Lq, Lq, hs, sp);
    if (threadIdx.x < MHA_MAX_LQ) { mrow[threadIdx.x] = -INFINITY; lrow[threadIdx.x] = 0.f; }
    float o[RI][CJ];
#pragma unroll
    for (int i = 0; i < RI; ++i)
#pragma unroll
        for (int j = 0; j < CJ; ++j) o[i][j] = 0.f;
    const int nk = causal ? min(N, Lq) : N;
    const uint32_t site = drop.site_base + (uint32_t)h;
    for (int k0 = 0; k0 < nk; k0 += MHA_KT) {
        const int kr = min(MHA_KT, nk - k0);
        __syncthreads();                                               // the previous chunk's K / V / P are consumed
        mha_load(Ks, K + ((long long)b * N + k0) * H + off, H, kr, MHA_KT, hs, sp);
        mha_load(Vs, V + ((long long)b * N + k0) * H + off, H, kr, MHA_KT, hs, sp);
        __syncthreads();
        float s[RI][KJ];
#pragma unroll
        for (int i = 0; i < RI; ++i)
#pragma unroll
            for (int j = 0; j < KJ; ++j) s[i][j] = 0.f;
        for (int c = 0; c < hs; ++c) {
            float qv[RI], kv[KJ];
#pragma unroll
            for (int i = 0; i < RI; ++i) qv[i] = Qs[min(ty + 16 * i, Lq - 1) * sp + c];
#pragma unroll
            for (int j = 0; j < KJ; ++j) kv[j] = Ks[(tx + 16 * j) * sp + c];
#pragma unroll
            for (int i = 0; i < RI; ++i)
#pragma unroll
                for (int j = 0; j < KJ; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
        }
#pragma unroll
        for (int i = 0; i < RI; ++i)
#pragma unroll
            for (int j = 0; j < KJ; ++j) {
                const int t = ty + 16 * i, rl = tx + 16 * j, r = k0 + rl;
                if (t < Lq) Ps[t * PS + rl] = (rl < kr && (!causal || r <= t)) ? s[i][j] * scale : -INFINITY;
            }
        __syncthreads();
        // row pass: online-softmax statistics, probabilities, dropout (one warp per row, one key per lane)
        for (int t = warp; t < Lq; t += MHA_THREADS / 32) {
            const float x = Ps[t * PS + lane];
            const float m_old = mrow[t], m_new = fmaxf(m_old, warp_max(x));
            float p = 0.f, alpha = 1.f;
            if (m_new != -INFINITY) {
                p = expf(x - m_new);
                alpha = expf(m_old - m_new);
            }
            const float sum = warp_sum(p);
            if (drop.p > 0.f && p != 0.f)
                p = mha_keep(((long long)b * Lq + t) * N + k0 + lane, drop, site) ? p * drop.inv_keep : 0.f;
            Ps[t * PS + lane] = p;
            if (lane == 0) { mrow[t] = m_new; lrow[t] = fmaf(lrow[t], alpha, sum); arow[t] = alpha; }
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < RI; ++i) {
            const int t = min(ty + 16 * i, Lq - 1);
            const float a = arow[t];
#pragma unroll
            for (int j = 0; j < CJ; ++j) o[i][j] *= a;
        }
        for (int rl = 0; rl < kr; ++rl) {
            float pv[RI], vv[CJ];
#pragma unroll
            for (int i = 0; i < RI; ++i) pv[i] = Ps[min(ty + 16 * i, Lq - 1) * PS + rl];
#pragma unroll
            for (int j = 0; j < CJ; ++j) vv[j] = Vs[rl * sp + min(tx + 16 * j, hs - 1)];
#pragma unroll
            for (int i = 0; i < RI; ++i)
#pragma unroll
                for (int j = 0; j < CJ; ++j) o[i][j] = fmaf(pv[i], vv[j], o[i][j]);
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < RI; ++i) {
        const int t = ty + 16 * i;
        if (t >= Lq) continue;
        const float inv_l = 1.f / lrow[t];
        float* orow = O + ((long long)b * Lq + t) * H + off;
#pragma unroll
        for (int j = 0; j < CJ; ++j) {
            const int c = tx + 16 * j;
            if (c < hs) orow[c] = o[i][j] * inv_l;
        }
    }
    if (threadIdx.x < Lq) lse[((long long)b * nh + h) * Lq + threadIdx.x] = mrow[threadIdx.x] + logf(lrow[threadIdx.x]);
}

__global__ void __launch_bounds__(MHA_THREADS) mha_bwd_kernel(const float* __restrict__ Q, const float* __restrict__ K, const float* __restrict__ V,
                                                             const float* __restrict__ O, const float* __restrict__ dO, const float* __restrict__ lse,
                                                             float* __restrict__ dQ, float* __restrict__ dK, float* __restrict__ dV, int Lq, int N,
                                                             int H, int chunk, int causal, float scale, MhaDrop drop) {
    extern __shared__ float sm[];
    const int h = blockIdx.x, b = blockIdx.y, nh = gridDim.x;
    const int off = h * chunk, hs = min(chunk, H - off), sp = hs | 1;
    float* Qs = sm;
    float* dOs = Qs + Lq * sp;
    float* Ks = dOs + Lq * sp;
    float* Vs = Ks + MHA_KT * sp;
    float* Pd = Vs + MHA_KT * sp;
    float* dS = Pd + MHA_MAX_LQ * PS;
    float* lse_s = dS + MHA_MAX_LQ * PS;
    float* D_s = lse_s + MHA_MAX_LQ;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long qbase = (long long)b * Lq * H + off;
    mha_load(Qs, Q + qbase, H, Lq, Lq, hs, sp);
    mha_load(dOs, dO + qbase, H, Lq, Lq, hs, sp);
    for (int t = warp; t < Lq; t += MHA_THREADS / 32) {               // D[t] = dO[t] . O[t] over the head's columns
        float a = 0.f;
        for (int c = lane; c < hs; c += 32) a = fmaf(dO[qbase + (long long)t * H + c], O[qbase + (long long)t * H + c], a);
        a = warp_sum(a);
        if (lane == 0) { D_s[t] = a; lse_s[t] = lse[((long long)b * nh + h) * Lq + t]; }
    }
    float dq[RI][CJ];
#pragma unroll
    for (int i = 0; i < RI; ++i)
#pragma unroll
        for (int j = 0; j < CJ; ++j) dq[i][j] = 0.f;
    const int nk = causal ? min(N, Lq) : N;
    const uint32_t site = drop.site_base + (uint32_t)h;
    for (int k0 = 0; k0 < nk; k0 += MHA_KT) {
        const int kr = min(MHA_KT, nk - k0);
        __syncthreads();
        mha_load(Ks, K + ((long long)b * N + k0) * H + off, H, kr, MHA_KT, hs, sp);
        mha_load(Vs, V + ((long long)b * N + k0) * H + off, H, kr, MHA_KT, hs, sp);
        __syncthreads();
        float s[RI][KJ], dp[RI][KJ];
#pragma unroll
        for (int i = 0; i < RI; ++i)
#pragma unroll
            for (int j = 0; j < KJ; ++j) s[i][j] = dp[i][j] = 0.f;
        for (int c = 0; c < hs; ++c) {
            float qv[RI], gv[RI], kv[KJ], vv[KJ];
#pragma unroll
            for (int i = 0; i < RI; ++i) {
                const int t = min(ty + 16 * i, Lq - 1);
                qv[i] = Qs[t * sp + c];
                gv[i] = dOs[t * sp + c];
            }
#pragma unroll
            for (int j = 0; j < KJ; ++j) {
                kv[j] = Ks[(tx + 16 * j) * sp + c];
                vv[j] = Vs[(tx + 16 * j) * sp + c];
            }
#pragma unroll
            for (int i = 0; i < RI; ++i)
#pragma unroll
                for (int j = 0; j < KJ; ++j) {
                    s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
                    dp[i][j] = fmaf(gv[i], vv[j], dp[i][j]);
                }
        }
#pragma unroll
        for (int i = 0; i < RI; ++i)
#pragma unroll
            for (int j = 0; j < KJ; ++j) {
                const int t = ty + 16 * i, rl = tx + 16 * j, r = k0 + rl;
                if (t >= Lq) continue;
                float pd = 0.f, ds = 0.f;
                if (rl < kr && (!causal || r <= t)) {
                    const float p = expf(s[i][j] * scale - lse_s[t]);
                    float dpv = dp[i][j];
                    pd = p;
                    if (drop.p > 0.f) {
                        const bool keep = mha_keep(((long long)b * Lq + t) * N + r, drop, site);
                        pd = keep ? p * drop.inv_keep : 0.f;
                        dpv = keep ? dpv * drop.inv_keep : 0.f;
                    }
                    ds = p * (dpv - D_s[t]);
                }
                Pd[t * PS + rl] = pd;
                dS[t * PS + rl] = ds;
            }
        __syncthreads();
        // dV = Pd^T dO and dK = scale * dS^T Q for the chunk's keys: complete here (every query row of the head is in this CTA)
#pragma unroll
        for (int i = 0; i < KJ; ++i) {
            const int rl = ty + 16 * i;
            float dv[CJ], dk[CJ];
#pragma unroll
            for (int j = 0; j < CJ; ++j) dv[j] = dk[j] = 0.f;
            for (int t = 0; t < Lq; ++t) {
                const float pd = Pd[t * PS + rl], ds = dS[t * PS + rl];
#pragma unroll
                for (int j = 0; j < CJ; ++j) {
                    const int c = min(tx + 16 * j, hs - 1);
                    dv[j] = fmaf(pd, dOs[t * sp + c], dv[j]);
                    dk[j] = fmaf(ds, Qs[t * sp + c], dk[j]);
                }
            }
            if (rl < kr) {
                const long long row = ((long long)b * N + k0 + rl) * H + off;
#pragma unroll
                for (int j = 0; j < CJ; ++j) {
                    const int c = tx + 16 * j;
                    if (c < hs) { dV[row + c] = dv[j]; dK[row + c] = dk[j] * scale; }
                }
            }
        }
        for (int rl = 0; rl < kr; ++rl) {
            float dsv[RI], kv[CJ];
#pragma unroll
            for (int i = 0; i < RI; ++i) dsv[i] = dS[min(ty + 16 * i, Lq - 1) * PS + rl];
#pragma unroll
            for (int j = 0; j < CJ; ++j) kv[j] = Ks[rl * sp + min(tx + 16 * j, hs - 1)];
#pragma unroll
            for (int i = 0; i < RI; ++i)
#pragma unroll
                for (int j = 0; j < CJ; ++j) dq[i][j] = fmaf(dsv[i], kv[j], dq[i][j]);
        }
    }
    // causal: keys past the last query row get no gradient
    if (causal && N > nk) {
        for (long long idx = threadIdx.x; idx < (long long)(N - nk) * hs; idx += MHA_THREADS) {
            const long long row = ((long long)b * N + nk + idx / hs) * H + off + idx % hs;
            dK[row] = 0.f;
            dV[row] = 0.f;
        }
    }
#pragma unroll
    for (int i = 0; i < RI; ++i) {
        const int t = ty + 16 * i;
        if (t >= Lq) continue;
        float* row = dQ + ((long long)b * Lq + t) * H + off;
#pragma unroll
        for (int j = 0; j < CJ; ++j) {
            const int c = tx + 16 * j;
            if (c < hs) row[c] = dq[i][j] * scale;
        }
    }
}

int mha_check(const void* q, const void* k, const void* v, int B, int Lq, int N, int H, float p, int* chunk, int* nh) {
    GVD_REQUIRE(q && k && v, "tr_mha: null tensor");
    GVD_REQUIRE(B >= 1 && H >= 1, "tr_mha: bad shape (B %d, H %d)", B, H);
    GVD_REQUIRE(Lq >= 1 && Lq <= MHA_MAX_LQ, "tr_mha: Lq = %d outside [1, %d]", Lq, MHA_MAX_LQ);
    GVD_REQUIRE(N >= 1 && N <= MHA_MAX_N, "tr_mha: N = %d outside [1, %d]", N, MHA_MAX_N);
    *chunk = (H + MHA_HEADS - 1) / MHA_HEADS;                          // torch.chunk(6, -1): ceil(H / 6) columns, the remainder last
    *nh = (H + *chunk - 1) / *chunk;
    GVD_REQUIRE(*chunk <= MHA_MAX_HS, "tr_mha: head width %d > %d (H = %d)", *chunk, MHA_MAX_HS, H);
    GVD_REQUIRE(p >= 0.f && p < 1.f, "tr_mha: dropout p = %f outside [0, 1)", (double)p);
    return 0;
}

MhaDrop mha_drop(float p, long long seed, int site_base, long long step) {
    MhaDrop d;
    d.p = p;
    d.inv_keep = 1.f / (1.f - p);
    d.seed_lo = (uint32_t)(seed & 0xffffffffll);
    d.seed_hi = (uint32_t)((unsigned long long)seed >> 32);
    d.site_base = (uint32_t)site_base;
    d.step_lo = (uint32_t)(step & 0xffffffffll);
    d.step_hi = (uint32_t)((unsigned long long)step >> 32);
    return d;
}

}  // namespace

extern "C" {
GVD_API int gvd_tr_mha_fwd(const float* q, const float* k, const float* v, float* o, float* lse, int B, int Lq, int N, int H, int causal, float scale,
                           float p, long long seed, int site_base, long long step, void* stream) {
    int chunk, nh;
    GVD_TRY(mha_check(q, k, v, B, Lq, N, H, p, &chunk, &nh));
    GVD_REQUIRE(o && lse, "tr_mha_fwd: null output");
    const int sp = chunk | 1;
    const size_t smem = ((size_t)(Lq + 2 * MHA_KT) * sp + MHA_MAX_LQ * PS + 3 * MHA_MAX_LQ) * sizeof(float);
    GVD_CHECK_CUDA(cudaFuncSetAttribute(mha_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mha_fwd_kernel<<<dim3(nh, B), MHA_THREADS, smem, (cudaStream_t)stream>>>(q, k, v, o, lse, Lq, N, H, chunk, causal ? 1 : 0, scale,
                                                                              mha_drop(p, seed, site_base, step));
    GVD_CHECK_LAUNCH();
    return 0;
}

GVD_API int gvd_tr_mha_bwd(const float* q, const float* k, const float* v, const float* o, const float* d_o, const float* lse, float* dq, float* dk,
                           float* dv, int B, int Lq, int N, int H, int causal, float scale, float p, long long seed, int site_base, long long step,
                           void* stream) {
    int chunk, nh;
    GVD_TRY(mha_check(q, k, v, B, Lq, N, H, p, &chunk, &nh));
    GVD_REQUIRE(o && d_o && lse && dq && dk && dv, "tr_mha_bwd: null tensor");
    const int sp = chunk | 1;
    const size_t smem = ((size_t)(2 * Lq + 2 * MHA_KT) * sp + 2 * MHA_MAX_LQ * PS + 2 * MHA_MAX_LQ) * sizeof(float);
    GVD_CHECK_CUDA(cudaFuncSetAttribute(mha_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mha_bwd_kernel<<<dim3(nh, B), MHA_THREADS, smem, (cudaStream_t)stream>>>(q, k, v, o, d_o, lse, dq, dk, dv, Lq, N, H, chunk, causal ? 1 : 0,
                                                                              scale, mha_drop(p, seed, site_base, step));
    GVD_CHECK_LAUNCH();
    return 0;
}
}  // extern "C"
