// gvd-b200: the transformer captioner (att_model = 'transformer'; SURVEY 8(f) row 4) — greedy incremental decode of
// misc/transformer.py:214-241 (Decoder.greedy) behind TransformerDecoder.forward(infer=True) (:271-274), called from
// misc/model.py:570-578 with the prologue's frame / region encodings.
//
// What the reference does per step and per layer: self-attention of the new position over the positions so far, attention of the
// result over the layer's encoder output, feed-forward, each in a ResidualBlock with the custom LayerNorm (:79-88,66-77); then the
// vocabulary head (tied with the embedding, :207,222) and an argmax.  It RE-PROJECTS the constant encoder output with wk / wv at every
// step (MultiHead.forward, :117-119) and re-projects every earlier position of the self-attention too; both are the same numbers each time,
// so this file projects the encoder output once per batch (wgmma GEMM) and caches the self-attention keys / values per position.
//
// The step is HBM-bound: the attention over the R = 1000 region rows streams K and V of every clip once (2 * R * H * 4 B per clip-step =
// 8.19 MB at H = 1024; 819 MB at B = 100) against ~30 MFLOP of products per clip.  tfm_cross_partial_kernel is that stream (flash-decoding
// split over row chunks: scores of all heads, chunk-local softmax numerators, weighted value sums in one pass over the chunk's K and V rows);
// everything else of the step is skinny M = B GEMMs (gvd_linear) and row kernels.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/gvd_b200.h"
#include "gvd_common.cuh"
#include "gvd_gemm.cuh"
#include "gvd_kernels.cuh"

namespace {

constexpr int TFM_MAX_HEADS = 8;
constexpr int TFM_MAX_L = 64;          // self-attention positions held in shared memory
constexpr int TFM_RC = 64;             // encoder rows per CTA of the attention stream (upper bound)
constexpr int TFM_HEAD_MAXV = 12000;   // tfm_head_kernel holds a logit row in shared memory; above this the sliced tail runs

// x0[b, :] = pe[t, :] + out_w[tok, :] * sqrt(d_model)       (transformer.py:222-231; two roundings as in the reference: fp32 product, then sum)
// tok[b] = tok_src[b * tok_stride + tok_off], or 0 (<bos>) when tok_src is null
// Producers of a product's activation rows also store the row's fp16x3 operand image (row_img != null; gvd_common.cuh layout, scale GVD_F16_SA) when the
// conversion-free products are on: column pairs (c, c + 1) sit in neighbouring lanes (every loop below walks columns with consecutive threads and a
// row length that is a multiple of 32, so whole warps are active), one shuffle fetches the partner.
__device__ __forceinline__ void tfm_img_store(uint32_t* __restrict__ row_img, int c, float v) {
    const float vn = __shfl_down_sync(0xffffffffu, v, 1);
    if (!(c & 1)) {
        uint32_t hi, lo;
        f16x3_split_pair(v, vn, GVD_F16_SA, hi, lo);
        uint32_t* d = row_img + f16x3_word(c);
        d[0] = hi; d[16] = lo;
    }
}

__global__ void tfm_embed_kernel(const float* __restrict__ pe, const float* __restrict__ out_w, const long long* __restrict__ tok_src, long long tok_stride,
                                 long long tok_off, int t, int H, int V, float sqrt_d, float* __restrict__ x, float* __restrict__ x_img) {
    const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= H) return;
    long long tok = tok_src ? tok_src[(long long)b * tok_stride + tok_off] : 0;
    tok = tok < 0 ? 0 : (tok >= V ? V - 1 : tok);                 // (ids are validated by the binding; never read outside the table)
    const float v = __fadd_rn(pe[(long long)t * H + c], __fmul_rn(out_w[tok * H + c], sqrt_d));
    x[(long long)b * H + c] = v;
    if (x_img) tfm_img_store(reinterpret_cast<uint32_t*>(x_img) + (long long)b * H, c, v);
}

// Partial sums: every skinny product of the step leaves split-K partials part[s][b][n] (s < S planes of B * ldp floats; S = 1 and one plane on the
// generic path); the consumers below sum them at load, add the bias and apply whatever follows (activation, residual + LayerNorm, argmax), so no
// product has a reduce pass of its own.
__device__ __forceinline__ float part_sum(const float* __restrict__ part, int S, long long plane, long long idx) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;                 // four independent chains: the loads of a group are in flight together
    int s = 0;
    for (; s + 3 < S; s += 4) {
        const float v0 = part[(long long)s * plane + idx], v1 = part[(long long)(s + 1) * plane + idx];
        const float v2 = part[(long long)(s + 2) * plane + idx], v3 = part[(long long)(s + 3) * plane + idx];
        a0 += v0; a1 += v1; a2 += v2; a3 += v3;
    }
    for (; s < S; ++s) a0 += part[(long long)s * plane + idx];
    return (a0 + a1) + (a2 + a3);
}

// self-attention of position t over the cached positions 0..t (MultiHead with a 2-D query: no causal mask needed, transformer.py:97-101,233-234)
// part: partials of (q | k_t | v_t) = x [Wq; Wk; Wv]^T, row pitch ldp >= 3H;  Kc / Vc [B, L, H] caches (row t written here).
// grid (heads, B): one CTA per (head, clip) — the head's columns of q / k_t / v_t are reduced, cached and used by the same CTA.
template <int NT>
__global__ void __launch_bounds__(NT)
tfm_self_attn_kernel(const float* __restrict__ part, int S, long long plane, int ldp, float* __restrict__ Kc, float* __restrict__ Vc,
                     float* __restrict__ out, int L, int t, int H, int cs, float inv_scale) {
    __shared__ float sc[TFM_MAX_L];
    extern __shared__ float q[];                                   // [cs]
    const int h = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = h * cs, c1 = min(H, c0 + cs), w = c1 - c0;
    float* kc = Kc + (long long)b * L * H + c0;
    float* vc = Vc + (long long)b * L * H + c0;
    for (int c = threadIdx.x; c < w; c += NT) {
        const long long o = (long long)b * ldp + c0 + c;
        q[c] = part_sum(part, S, plane, o);
        kc[(long long)t * H + c] = part_sum(part, S, plane, o + H);
        vc[(long long)t * H + c] = part_sum(part, S, plane, o + 2 * H);
    }
    __syncthreads();
    const int n = t + 1;
    for (int j = warp; j < n; j += NT / 32) {                      // one warp per position
        float s = 0.f;
        for (int c = lane; c < w; c += 32) s = fmaf(q[c], kc[(long long)j * H + c], s);
        s = warp_sum(s);
        if (lane == 0) sc[j] = s * inv_scale;
    }
    __syncthreads();
    if (warp == 0) {                                               // softmax over the positions (n <= 64)
        float m = -INFINITY;
        for (int j = lane; j < n; j += 32) m = fmaxf(m, sc[j]);
        m = warp_max(m);
        float s = 0.f;
        for (int j = lane; j < n; j += 32) { const float e = expf(sc[j] - m); sc[j] = e; s += e; }
        s = warp_sum(s);
        const float inv = 1.f / s;
        for (int j = lane; j < n; j += 32) sc[j] *= inv;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < w; c += NT) {
        float a0 = 0.f, a1 = 0.f;
        int j = 0;
        for (; j + 1 < n; j += 2) {
            a0 = fmaf(sc[j], vc[(long long)j * H + c], a0);
            a1 = fmaf(sc[j + 1], vc[(long long)(j + 1) * H + c], a1);
        }
        if (j < n) a0 = fmaf(sc[j], vc[(long long)j * H + c], a0);
        out[(long long)b * H + c0 + c] = a0 + a1;
    }
}

// y[b, :] = LN*(res[b, :] + sum_s part[s][b, :] + bias):  the ResidualBlock tail (transformer.py:87-88 with the LayerNorm of :66-77: unbiased std,
// eps added to the std) fused with the split-K reduce of the product that feeds it.  One CTA per row.
template <int NT>
__global__ void __launch_bounds__(NT)
tfm_reduce_ln_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias, const float* __restrict__ res,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y, int H, float* __restrict__ y_img) {
    __shared__ float red[32];
    extern __shared__ float vbuf[];
    const long long b = blockIdx.x;
    float s = 0.f;
    for (int c = threadIdx.x; c < H; c += NT) {
        float a = part_sum(part, S, plane, b * ldp + c);
        if (bias) a += bias[c];
        const float v = res[b * H + c] + a;
        vbuf[c] = v;
        s += v;
    }
    const float mu = block_sum(s, red) / (float)H;
    float q = 0.f;
    for (int c = threadIdx.x; c < H; c += NT) { const float d = vbuf[c] - mu; q += d * d; }
    const float sd = sqrtf(block_sum(q, red) / (float)(H - 1));
    const float inv = 1.f / (sd + 1e-6f);
    for (int c = threadIdx.x; c < H; c += NT) {
        const float v = gamma[c] * (vbuf[c] - mu) * inv + beta[c];
        y[b * H + c] = v;
        if (y_img) tfm_img_store(reinterpret_cast<uint32_t*>(y_img) + b * H, c, v);
    }
}

// out[b, n] = relu(sum_s part[s][b, n] + bias[n])     (FeedForward.linear1 + ReLU, transformer.py:132-133)
__global__ void tfm_reduce_relu_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias,
                                       float* __restrict__ out, int N, int B, float* __restrict__ out_img) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * N) return;
    const int b = (int)(i / N), n = (int)(i % N);
    const float v = fmaxf(part_sum(part, S, plane, (long long)b * ldp + n) + bias[n], 0.f);
    out[i] = v;
    if (out_img) tfm_img_store(reinterpret_cast<uint32_t*>(out_img) + (long long)b * N, n, v);
}

// The attention stream.  grid (chunks, B); CTA (chunk, b) owns encoder rows [r0, r1) of clip b:
//   s[r][h] = q_h . K[b, r, head h columns] / sqrt(d_model);  m[h] = max_r s;  e[r][h] = exp(s - m[h]);  l[h] = sum_r e
//   acc[c] = sum_r e[r][head(c)] * V[b, r, c]
// and writes (acc [H], m [nh], l [nh]) for tfm_cross_combine_kernel.  K and V rows are read exactly once, coalesced (one warp per K row in
// the score phase, the CTA's threads across the columns of a V row in the value phase).  H <= 1024, H % 4 == 0.
template <int NT>
__global__ void __launch_bounds__(NT, 4)
tfm_cross_partial_kernel(const float* __restrict__ qpart, int qS, long long qplane, int qld, const float* __restrict__ K, const float* __restrict__ V,
                         int n, int H, int cs, int nh, int rows_per_cta, float inv_scale, float* __restrict__ part_acc, float* __restrict__ part_ml) {
    __shared__ float e[TFM_RC][TFM_MAX_HEADS];
    __shared__ float mh[TFM_MAX_HEADS];
    const int b = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
    const int r0 = chunk * rows_per_cta, r1 = min(n, r0 + rows_per_cta), nr = r1 - r0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* qb = qpart + (long long)b * qld;               // split-K partials of the query projection, summed once per CTA
    __shared__ __align__(16) float qs[1024];
    for (int c = threadIdx.x; c < H; c += NT) qs[c] = part_sum(qb, qS, qplane, c);
    __syncthreads();
    const float* Kb = K + ((long long)b * n + r0) * H;
    const float* Vb = V + ((long long)b * n + r0) * H;
    // --- scores: warp per row; lane owns the float4 column groups lane * 4 + 128 * j
    float4 qr[8];
    int hq[8];                         // head of the group's first column; a group may straddle one head boundary
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = lane * 4 + 128 * j;
        qr[j] = c < H ? *reinterpret_cast<const float4*>(qs + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        hq[j] = c / cs;
    }
    for (int r = warp; r < nr; r += NT / 32) {
        const float* kr = Kb + (long long)r * H;
        float ph[TFM_MAX_HEADS];
#pragma unroll
        for (int h = 0; h < TFM_MAX_HEADS; ++h) ph[h] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = lane * 4 + 128 * j;
            if (c < H) {
                const float4 kv = __ldg(reinterpret_cast<const float4*>(kr + c));
                const float pr[4] = {qr[j].x * kv.x, qr[j].y * kv.y, qr[j].z * kv.z, qr[j].w * kv.w};
                const int h0 = hq[j];
                const int split = (h0 + 1) * cs - c;               // columns [c, c + split) belong to head h0, the rest to h0 + 1
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (i < split) a0 += pr[i]; else a1 += pr[i];
                }
#pragma unroll
                for (int h = 0; h < TFM_MAX_HEADS; ++h) {
                    ph[h] += (h == h0) ? a0 : 0.f;
                    ph[h] += (h == h0 + 1) ? a1 : 0.f;
                }
            }
        }
#pragma unroll
        for (int h = 0; h < TFM_MAX_HEADS; ++h) {
            if (h < nh) {
                const float s = warp_sum(ph[h]);
                if (lane == 0) e[r][h] = s * inv_scale;
            }
        }
    }
    __syncthreads();
    // --- chunk-local softmax numerators, one warp per head
    if (warp < nh) {
        float m = -INFINITY;
        for (int r = lane; r < nr; r += 32) m = fmaxf(m, e[r][warp]);
        m = warp_max(m);
        float l = 0.f;
        for (int r = lane; r < nr; r += 32) { const float x = expf(e[r][warp] - m); e[r][warp] = x; l += x; }
        l = warp_sum(l);
        if (lane == 0) {
            mh[warp] = m;
            float* ml = part_ml + ((long long)b * nchunks + chunk) * 2 * TFM_MAX_HEADS;
            ml[warp] = m;
            ml[TFM_MAX_HEADS + warp] = l;
        }
    }
    __syncthreads();
    // --- weighted value sum: thread owns 4 consecutive columns
    const int c = threadIdx.x * 4;
    if (c < H) {
        int hc[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) hc[i] = (c + i) / cs;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const float* vp = Vb + c;
#pragma unroll 8
        for (int r = 0; r < nr; ++r) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(vp + (long long)r * H));
            acc.x = fmaf(e[r][hc[0]], v.x, acc.x);
            acc.y = fmaf(e[r][hc[1]], v.y, acc.y);
            acc.z = fmaf(e[r][hc[2]], v.z, acc.z);
            acc.w = fmaf(e[r][hc[3]], v.w, acc.w);
        }
        *reinterpret_cast<float4*>(part_acc + ((long long)b * nchunks + chunk) * H + c) = acc;
    }
}

// out[b, c] = sum_k acc_k[c] * exp(m_k[h] - M[h]) / sum_k l_k[h] * exp(m_k[h] - M[h]),  h = head(c), M = max_k m_k
template <int NT>
__global__ void __launch_bounds__(NT)
tfm_cross_combine_kernel(const float* __restrict__ part_acc, const float* __restrict__ part_ml, int nchunks, int H, int cs, int nh,
                         float* __restrict__ out, float* __restrict__ out_img) {
    extern __shared__ float wgt[];                  // [nchunks][TFM_MAX_HEADS]: exp(m_k - M) / L
    __shared__ float Mh[TFM_MAX_HEADS], Lh[TFM_MAX_HEADS];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* ml = part_ml + (long long)b * nchunks * 2 * TFM_MAX_HEADS;
    if (warp < nh) {
        float m = -INFINITY;
        for (int k = lane; k < nchunks; k += 32) m = fmaxf(m, ml[(long long)k * 2 * TFM_MAX_HEADS + warp]);
        m = warp_max(m);
        float l = 0.f;
        for (int k = lane; k < nchunks; k += 32) {
            const float w = expf(ml[(long long)k * 2 * TFM_MAX_HEADS + warp] - m);
            wgt[k * TFM_MAX_HEADS + warp] = w;
            l += w * ml[(long long)k * 2 * TFM_MAX_HEADS + TFM_MAX_HEADS + warp];
        }
        l = warp_sum(l);
        if (lane == 0) { Mh[warp] = m; Lh[warp] = l; }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < H; c += NT) {
        const int h = c / cs;
        float a = 0.f;
        for (int k = 0; k < nchunks; ++k) a = fmaf(wgt[k * TFM_MAX_HEADS + h], part_acc[((long long)b * nchunks + k) * H + c], a);
        const float v = a / Lh[h];
        out[(long long)b * H + c] = v;
        if (out_img) tfm_img_store(reinterpret_cast<uint32_t*>(out_img) + (long long)b * H, c, v);
    }
}

// Vocabulary head tail: logits[b, v] = sum_s part[s][b, v] + bias[v]; prediction[b, t] = first index of the maximum (`.max(-1)`, transformer.py:240);
// optional copy of the logits; teacher forcing: nll[b, t] = logsumexp(logits) - logits[target], target = teacher[b, t + 1], 0 where the target is 0
// (mask(), transformer.py:51-54).  One CTA per clip.
template <int NT>
__global__ void __launch_bounds__(NT)
tfm_head_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias, int V, long long* __restrict__ seq,
                int L, int t, float* __restrict__ logits_out, const long long* __restrict__ teacher, float* __restrict__ nll) {
    __shared__ float red[32];
    __shared__ float bv[NT / 32];
    __shared__ int bi[NT / 32];
    extern __shared__ float lg[];                                  // [V]
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float best = -INFINITY;
    int idx = 0x7fffffff;
    for (int v = threadIdx.x; v < V; v += NT) {
        const float y = part_sum(part, S, plane, (long long)b * ldp + v) + bias[v];
        lg[v] = y;
        if (logits_out) logits_out[((long long)b * L + t) * V + v] = y;
        if (y > best || idx == 0x7fffffff) { best = y; idx = v; }                // v ascends per thread: the first maximum is kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ov > best || (ov == best && oi < idx)) { best = ov; idx = oi; }
    }
    if (lane == 0) { bv[warp] = best; bi[warp] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < NT / 32; ++w)
            if (bv[w] > best || (bv[w] == best && bi[w] < idx)) { best = bv[w]; idx = bi[w]; }
        bv[0] = best;
        if (seq) seq[(long long)b * L + t] = idx == 0x7fffffff ? 0 : idx;
    }
    if (!teacher) return;
    __syncthreads();
    const float m = bv[0];
    float s = 0.f;
    for (int v = threadIdx.x; v < V; v += NT) s += expf(lg[v] - m);
    s = block_sum(s, red);
    const long long tgt = teacher[(long long)b * (L + 1) + t + 1];
    if (threadIdx.x == 0) nll[(long long)b * L + t] = (tgt > 0 && tgt < V) ? (m + logf(s)) - lg[tgt] : 0.f;
}
// loss = sum(nll over kept targets) / #kept   (F.cross_entropy, mean reduction; 0 / 0 = NaN like the reference on an all-padding batch)
template <int NT>
__global__ void __launch_bounds__(NT)
tfm_loss_kernel(const float* __restrict__ nll, const long long* __restrict__ seq, int B, int S, float* __restrict__ loss) {
    __shared__ float red[32];
    float s = 0.f, n = 0.f;
    for (int i = threadIdx.x; i < B * S; i += NT) {
        const int b = i / S, t = i % S;
        if (seq[(long long)b * (S + 1) + t + 1] != 0) { s += nll[i]; n += 1.f; }
    }
    s = block_sum(s, red);
    n = block_sum(n, red);
    if (threadIdx.x == 0) loss[0] = s / n;
}

struct TfmWs {
    float *x, *y, *z, *sa, *ca, *f, *part;
    float *wqkv[2];                       // [Wq; Wk; Wv] of the self-attention, one product per layer and step
    float *Kc[2], *Vc[2], *Ke[2], *Ve[2];
    float *part_acc, *part_ml, *nll;
    float* vt_rec; int* vt_ticket;        // vocabularies above 12000 words: records and tickets of the sliced head tail (gvd_vocab_tail)
    long long* out_seq;                   // graph replay: the prediction lands here (fixed address), then is copied to the caller's tensor
    // conversion-free products (backend bit 4): fp16x3 operand images of the 13 weight matrices (packed once per batch by tfm_run) and of the
    // current product's activation rows; null when a contraction length is not a multiple of 32
    float *wi_qkv[2], *wi_swo[2], *wi_aq[2], *wi_awo[2], *wi_f1[2], *wi_f2[2], *wi_out, *ximg;
    float *ix, *iy, *iz, *ica, *iff;      // images of x / y / z / ca / f, stored by the kernels that produce those rows (the self-attention output is packed)
    int chunks[2], rows[2];
    size_t bytes;
};

int tfm_chunking(int B, int n, int* rows) {
    // enough CTAs to cover the machine a few times over, at most TFM_RC rows each
    int chunks = std::max(1, std::min(gvd_cdiv(n, 8), gvd_cdiv(132 * 6, std::max(B, 1))));
    int r = gvd_cdiv(n, chunks);
    r = std::min(r, TFM_RC);
    *rows = r;
    return gvd_cdiv(n, r);
}

inline int rup4i(int x) { return (x + 3) / 4 * 4; }

// split-K planes of one skinny product (0: generic path, one plane)
int tfm_splits(int Nw, int K, int B) {
    if (!gvd_backend_on(BK_TC | BK_SPLITK)) return 0;        // wgmma + split-K decode products
    return gvd_skinny_splits(Nw, K, B);
}
size_t tfm_part_floats(int Nw, int K, int B) { return (size_t)std::max(1, gvd_skinny_splits(Nw, K, B)) * B * rup4i(Nw); }

TfmWs tfm_layout(const gvd_tfm_weights_t* w, int B, int L, const int n[2], void* base) {
    TfmWs s{};
    const int H = w->d_model, V = w->vocab_size, DH = w->d_hidden;
    size_t off = 0;
    auto take = [&](size_t floats) {
        float* p = base ? reinterpret_cast<float*>(static_cast<char*>(base) + off) : nullptr;
        off += (floats * sizeof(float) + 255) / 256 * 256;
        return p;
    };
    const size_t BH = (size_t)B * H;
    s.x = take(BH); s.y = take(BH); s.z = take(BH); s.sa = take(BH); s.ca = take(BH);
    s.f = take((size_t)B * DH);
    s.part = take(std::max(std::max(tfm_part_floats(3 * H, H, B), tfm_part_floats(H, H, B)),
                           std::max(std::max(tfm_part_floats(DH, H, B), tfm_part_floats(H, DH, B)), tfm_part_floats(V, H, B))));
    size_t cmax = 0;
    for (int l = 0; l < 2; ++l) {
        s.wqkv[l] = take((size_t)3 * H * H);
        s.Kc[l] = take(BH * L); s.Vc[l] = take(BH * L);
        s.Ke[l] = take(BH * n[l]); s.Ve[l] = take(BH * n[l]);
        s.chunks[l] = tfm_chunking(B, n[l], &s.rows[l]);
        cmax = std::max(cmax, (size_t)s.chunks[l]);
    }
    s.part_acc = take(cmax * BH);
    s.part_ml = take((size_t)B * cmax * 2 * TFM_MAX_HEADS);
    s.nll = take((size_t)B * L);
    s.out_seq = reinterpret_cast<long long*>(take((size_t)B * L * 2));
    if (V > TFM_HEAD_MAXV) {
        s.vt_rec = take(gvd_vocab_rec_floats(B, V));
        s.vt_ticket = reinterpret_cast<int*>(take((size_t)B));
    }
    if (H % 32 == 0 && DH % 32 == 0 && B <= 128) {
        const size_t HH = (size_t)H * H;
        for (int l = 0; l < 2; ++l) {
            s.wi_qkv[l] = take(3 * HH); s.wi_swo[l] = take(HH); s.wi_aq[l] = take(HH); s.wi_awo[l] = take(HH);
            s.wi_f1[l] = take((size_t)DH * H); s.wi_f2[l] = take((size_t)H * DH);
        }
        s.wi_out = take((size_t)V * H);
        s.ximg = take((size_t)B * std::max(H, DH));
        s.ix = take(BH); s.iy = take(BH); s.iz = take(BH); s.ica = take(BH); s.iff = take((size_t)B * DH);
    }
    s.bytes = off;
    return s;
}

int tfm_check(const gvd_tfm_weights_t* w, int B, int L, int n0, int n1) {
    GVD_REQUIRE(w, "tfm: null weights");
    const int H = w->d_model;
    GVD_REQUIRE(H >= 8 && H <= 1024 && H % 4 == 0, "tfm: d_model must be a multiple of 4 in [8, 1024] (got %d)", H);
    GVD_REQUIRE(w->d_hidden >= 4 && w->d_hidden % 4 == 0, "tfm: d_hidden must be a multiple of 4 (got %d)", w->d_hidden);
    GVD_REQUIRE(w->n_heads >= 1 && w->n_heads <= TFM_MAX_HEADS, "tfm: 1..%d heads (got %d)", TFM_MAX_HEADS, w->n_heads);
    GVD_REQUIRE((H + w->n_heads - 1) / w->n_heads >= 4, "tfm: heads narrower than 4 columns are not supported (d_model %d, %d heads)", H, w->n_heads);
    GVD_REQUIRE(w->vocab_size >= 2 && w->vocab_size <= 65535 * VOCAB_SLICE, "tfm: vocab_size must be in [2, %d] (got %d)", 65535 * VOCAB_SLICE,
                w->vocab_size);
    GVD_REQUIRE(B >= 1 && L >= 1 && L <= TFM_MAX_L && n0 >= 1 && n1 >= 1, "tfm: bad sizes B=%d L=%d n0=%d n1=%d (L <= %d)", B, L, n0, n1, TFM_MAX_L);
    return 0;
}

// part[s][b][n] = partial sums of X[b, :] . W[n, :]: operand-swapped split-K wgmma product when the shape allows it (the weight rows fill the
// 128-row MMA tile, the batch is the N tile; S planes), else the generic GEMM into one plane.  Returns the plane count through *S.
// With backend bit 4 and the weight's fp16x3 image at hand (Wimg; Ximg = scratch for the image of X): one small pack pass over the B activation
// rows, then the conversion-free kernel of the greedy LSTM path (skinny_f16_kernel: TMA -> wgmma on both operand images, no conversion,
// ) — the products of this loop are 2-20 MB of weights each, so their time is the fixed latency of the kernel.
bool tfm_f16() { return gvd_backend_on(BK_F16X3); }
int tfm_product(const float* W, int Nw, int K, const float* X, long long ldx, int B, float* part, int ldp, int* S, cudaStream_t st,
                const float* Wimg = nullptr, float* Ximg = nullptr, const float* Xready = nullptr) {
    const int sp = tfm_splits(Nw, K, B);
    if (sp > 0 && Wimg && Ximg && K % 32 == 0 && B <= 128 && tfm_f16()) {
        *S = sp;
        if (!Xready) {              // (Xready: the producer of X stored the image itself)
            GVD_TRY(gvd_pack_f16x3(X, ldx, B, K, Ximg, K, st, GVD_F16_SA));
            Xready = Ximg;
        }
        return gvd_skinny_f16(Wimg, K, Nw, Xready, K, B, K, sp, part, ldp, st);
    }
    if (sp > 0) {
        *S = sp;
        return gvd_skinny_splitk(W, Nw, K, X, ldx, B, sp, part, ldp, st);
    }
    *S = 1;
    return gvd_linear(X, ldx, W, K, nullptr, part, ldp, B, Nw, K, GVD_ACT_NONE, st);
}

}  // namespace

extern "C" GVD_API size_t gvd_tfm_workspace_bytes(const gvd_tfm_weights_t* w, int B, int L, int n0, int n1) {
    if (tfm_check(w, B, L, n0, n1) != 0) return 0;
    const int n[2] = {n0, n1};
    return tfm_layout(w, B, L, n, nullptr).bytes;
}

static int tfm_loop(const gvd_tfm_weights_t* w, const TfmWs& s, int B, int L, int n0, int n1, const float* pe, int64_t* seq_out, float* logits_out,
                    const int64_t* teacher, float* loss_out, cudaStream_t st);

// The greedy loop as ONE CUDA graph (L x 29 launches replayed with a single cudaGraphLaunch), cached per (weights, sizes, workspace, backend).
// The prediction is written to a workspace-resident buffer inside the graph and copied to the caller's tensor after the replay.
namespace {
struct TfmGraph {
    std::mutex mu;
    cudaStream_t capture_stream = nullptr;
    cudaGraphExec_t exec = nullptr;
    gvd_tfm_weights_t w{};
    int B = 0, L = 0, n0 = 0, n1 = 0, backend = 0;
    const void *pe = nullptr, *ws = nullptr;
    long long nodes = 0;
} g_tfm_graph;
bool tfm_graph_ok() {
    static const bool no_graph = getenv("GVD_NO_GRAPH") != nullptr;
    return !no_graph;
}
}  // namespace

static int tfm_loop_graph(const gvd_tfm_weights_t* w, const TfmWs& s, int B, int L, int n0, int n1, const float* pe, void* workspace, int64_t* seq_out,
                          cudaStream_t st) {
    TfmGraph& g = g_tfm_graph;
    std::lock_guard<std::mutex> lk(g.mu);
    if (!g.exec || memcmp(&g.w, w, sizeof(*w)) != 0 || g.B != B || g.L != L || g.n0 != n0 || g.n1 != n1 || g.backend != gvd_backend() || g.pe != pe ||
        g.ws != workspace) {
        if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }
        if (!g.capture_stream) GVD_CHECK_CUDA(cudaStreamCreateWithFlags(&g.capture_stream, cudaStreamNonBlocking));
        // first use of every kernel of the loop outside a capture (function attributes are set lazily on first launch)
        GVD_TRY(tfm_loop(w, s, B, 1, n0, n1, pe, (int64_t*)s.out_seq, nullptr, nullptr, nullptr, st));
        GVD_CHECK_CUDA(cudaStreamSynchronize(st));
        cudaGraph_t graph = nullptr;
        GVD_CHECK_CUDA(cudaStreamBeginCapture(g.capture_stream, cudaStreamCaptureModeThreadLocal));
        const long long l0 = gvd_launch_count();
        const int rc = tfm_loop(w, s, B, L, n0, n1, pe, (int64_t*)s.out_seq, nullptr, nullptr, nullptr, g.capture_stream);
        const cudaError_t ce = cudaStreamEndCapture(g.capture_stream, &graph);
        g.nodes = gvd_launch_count() - l0;
        gvd_launch_count_add(-g.nodes);                    // capturing launches nothing
        if (rc != 0) { if (graph) cudaGraphDestroy(graph); return rc; }
        GVD_CHECK_CUDA(ce);
        const cudaError_t ie = cudaGraphInstantiate(&g.exec, graph, 0);
        cudaGraphDestroy(graph);
        GVD_CHECK_CUDA(ie);
        g.w = *w; g.B = B; g.L = L; g.n0 = n0; g.n1 = n1; g.backend = gvd_backend(); g.pe = pe; g.ws = workspace;
    }
    GVD_CHECK_CUDA(cudaGraphLaunch(g.exec, st));
    gvd_launch_count_add(g.nodes);
    GVD_CHECK_CUDA(cudaMemcpyAsync(seq_out, s.out_seq, (size_t)B * L * sizeof(long long), cudaMemcpyDeviceToDevice, st));
    return 0;
}

// greedy (teacher == null): token of step t = prediction of step t - 1, seq_out [B, L] filled;  teacher forcing (teacher [B, L + 1]): token of
// step t = teacher[:, t], loss_out = masked cross-entropy against teacher[:, t + 1]
static int tfm_run(const gvd_tfm_weights_t* w, int B, int L, const float* enc0, int n0, const float* enc1, int n1, const float* pe, void* workspace,
                   size_t workspace_bytes, int64_t* seq_out, float* logits_out, const int64_t* teacher, float* loss_out, void* stream) {
    GVD_TRY(tfm_check(w, B, L, n0, n1));
    GVD_REQUIRE(enc0 && enc1 && pe && (seq_out || teacher), "tfm: null argument");
    GVD_REQUIRE(workspace && ((uintptr_t)workspace & 255) == 0, "workspace must be a 256-byte aligned device pointer");
    const int n[2] = {n0, n1};
    const float* enc[2] = {enc0, enc1};
    TfmWs s = tfm_layout(w, B, L, n, workspace);
    GVD_REQUIRE(workspace_bytes >= s.bytes, "tfm workspace too small: %zu < %zu bytes", workspace_bytes, s.bytes);
    cudaStream_t st = (cudaStream_t)stream;
    const int H = w->d_model;
    GVD_REQUIRE(w->out_w && w->out_b, "tfm: null vocabulary head");
    for (int l = 0; l < 2; ++l) {
        const gvd_tfm_layer_t& y = w->layer[l];
        GVD_REQUIRE(y.self_wq && y.self_wk && y.self_wv && y.self_wo && y.self_gamma && y.self_beta && y.att_wq && y.att_wk && y.att_wv && y.att_wo &&
                    y.att_gamma && y.att_beta && y.ff_w1 && y.ff_b1 && y.ff_w2 && y.ff_b2 && y.ff_gamma && y.ff_beta, "tfm: layer %d has a null weight", l);
        // keys / values of the encoder output: once per batch instead of once per step
        GVD_TRY(gvd_linear(enc[l], H, y.att_wk, H, nullptr, s.Ke[l], H, B * n[l], H, H, GVD_ACT_NONE, st));
        GVD_TRY(gvd_linear(enc[l], H, y.att_wv, H, nullptr, s.Ve[l], H, B * n[l], H, H, GVD_ACT_NONE, st));
        // [Wq; Wk; Wv] of the self-attention as one weight matrix
        const size_t hh = (size_t)H * H * sizeof(float);
        GVD_CHECK_CUDA(cudaMemcpyAsync(s.wqkv[l], y.self_wq, hh, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(s.wqkv[l] + (size_t)H * H, y.self_wk, hh, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(s.wqkv[l] + (size_t)2 * H * H, y.self_wv, hh, cudaMemcpyDeviceToDevice, st));
        if (s.ximg && tfm_f16()) {     // operand images of the layer's weights (one element-wise pass per batch)
            const int DH = w->d_hidden;
            GVD_TRY(gvd_pack_f16x3(s.wqkv[l], H, 3 * H, H, s.wi_qkv[l], H, st, GVD_F16_SW));
            GVD_TRY(gvd_pack_f16x3(y.self_wo, H, H, H, s.wi_swo[l], H, st, GVD_F16_SW));
            GVD_TRY(gvd_pack_f16x3(y.att_wq, H, H, H, s.wi_aq[l], H, st, GVD_F16_SW));
            GVD_TRY(gvd_pack_f16x3(y.att_wo, H, H, H, s.wi_awo[l], H, st, GVD_F16_SW));
            GVD_TRY(gvd_pack_f16x3(y.ff_w1, H, DH, H, s.wi_f1[l], H, st, GVD_F16_SW));
            GVD_TRY(gvd_pack_f16x3(y.ff_w2, DH, H, DH, s.wi_f2[l], DH, st, GVD_F16_SW));
        }
    }
    if (s.ximg && tfm_f16()) GVD_TRY(gvd_pack_f16x3(w->out_w, H, w->vocab_size, H, s.wi_out, H, st, GVD_F16_SW));
    if (s.vt_ticket) GVD_CHECK_CUDA(cudaMemsetAsync(s.vt_ticket, 0, (size_t)B * sizeof(int), st));    // the tail resets them after each use
    if (!teacher && !logits_out && tfm_graph_ok()) return tfm_loop_graph(w, s, B, L, n0, n1, pe, workspace, seq_out, st);
    return tfm_loop(w, s, B, L, n0, n1, pe, seq_out, logits_out, teacher, loss_out, st);
}

// the L decode steps (29 launches each); every buffer they touch is in the workspace except pe / weights / seq_out / logits_out / teacher
static int tfm_loop(const gvd_tfm_weights_t* w, const TfmWs& s, int B, int L, int n0, int n1, const float* pe, int64_t* seq_out, float* logits_out,
                    const int64_t* teacher, float* loss_out, cudaStream_t st) {
    const int n[2] = {n0, n1};
    const int H = w->d_model, V = w->vocab_size, DH = w->d_hidden;
    // torch.chunk(n_heads, -1): ceil(H / n_heads) columns per head, the remainder in the last (transformer.py:120-121)
    const int cs = (H + w->n_heads - 1) / w->n_heads, nh = (H + cs - 1) / cs;
    const float inv_scale = 1.f / sqrtf((float)H);                         // Attention.scale = sqrt(d_key) with d_key = d_model (transformer.py:94,111)
    const float sqrt_d = sqrtf((float)H);
    const size_t smemH = (size_t)H * sizeof(float);
    int S = 1;
    // conversion-free products: the producers below store the operand images themselves (fi = fused images on; the conditions of tfm_product)
    const bool fi = s.ximg && tfm_f16() && gvd_backend_on(BK_TC | BK_SPLITK) && B <= 128;
    float *ix = fi ? s.ix : nullptr, *iy = fi ? s.iy : nullptr, *iz = fi ? s.iz : nullptr, *ica = fi ? s.ica : nullptr, *iff = fi ? s.iff : nullptr;
    for (int t = 0; t < L; ++t) {
        if (teacher) tfm_embed_kernel<<<dim3(gvd_cdiv(H, 256), B), 256, 0, st>>>(pe, w->out_w, (const long long*)teacher, L + 1, t, t, H, V, sqrt_d, s.x, ix);
        else tfm_embed_kernel<<<dim3(gvd_cdiv(H, 256), B), 256, 0, st>>>(pe, w->out_w, t == 0 ? nullptr : (const long long*)seq_out, L, t - 1, t, H, V, sqrt_d, s.x, ix);
        GVD_CHECK_LAUNCH();
        for (int l = 0; l < 2; ++l) {
            const gvd_tfm_layer_t& y = w->layer[l];
            // self-attention block: x -> y
            int ldp = rup4i(3 * H);
            GVD_TRY(tfm_product(s.wqkv[l], 3 * H, H, s.x, H, B, s.part, ldp, &S, st, s.wi_qkv[l], s.ximg, ix));
            tfm_self_attn_kernel<128><<<dim3(nh, B), 128, (size_t)cs * sizeof(float), st>>>(s.part, S, (long long)B * ldp, ldp, s.Kc[l], s.Vc[l], s.sa, L, t, H, cs,
                                                                                          inv_scale);
            GVD_CHECK_LAUNCH();
            GVD_TRY(tfm_product(y.self_wo, H, H, s.sa, H, B, s.part, H, &S, st, s.wi_swo[l], s.ximg));
            tfm_reduce_ln_kernel<256><<<B, 256, smemH, st>>>(s.part, S, (long long)B * H, H, nullptr, s.x, y.self_gamma, y.self_beta, s.y, H, iy);
            GVD_CHECK_LAUNCH();
            // attention over the encoder output: y -> z
            GVD_TRY(tfm_product(y.att_wq, H, H, s.y, H, B, s.part, H, &S, st, s.wi_aq[l], s.ximg, iy));
            tfm_cross_partial_kernel<256><<<dim3(s.chunks[l], B), 256, 0, st>>>(s.part, S, (long long)B * H, H, s.Ke[l], s.Ve[l], n[l], H, cs, nh, s.rows[l],
                                                                                inv_scale, s.part_acc, s.part_ml);
            GVD_CHECK_LAUNCH();
            tfm_cross_combine_kernel<256><<<B, 256, (size_t)s.chunks[l] * TFM_MAX_HEADS * sizeof(float), st>>>(s.part_acc, s.part_ml, s.chunks[l], H, cs, nh,
                                                                                                              s.ca, ica);
            GVD_CHECK_LAUNCH();
            GVD_TRY(tfm_product(y.att_wo, H, H, s.ca, H, B, s.part, H, &S, st, s.wi_awo[l], s.ximg, ica));
            tfm_reduce_ln_kernel<256><<<B, 256, smemH, st>>>(s.part, S, (long long)B * H, H, nullptr, s.y, y.att_gamma, y.att_beta, s.z, H, iz);
            GVD_CHECK_LAUNCH();
            // feed-forward: z -> x
            ldp = rup4i(DH);
            GVD_TRY(tfm_product(y.ff_w1, DH, H, s.z, H, B, s.part, ldp, &S, st, s.wi_f1[l], s.ximg, iz));
            tfm_reduce_relu_kernel<<<gvd_cdiv((long long)B * DH, 256), 256, 0, st>>>(s.part, S, (long long)B * ldp, ldp, y.ff_b1, s.f, DH, B, iff);
            GVD_CHECK_LAUNCH();
            GVD_TRY(tfm_product(y.ff_w2, H, DH, s.f, DH, B, s.part, H, &S, st, s.wi_f2[l], s.ximg, iff));
            tfm_reduce_ln_kernel<256><<<B, 256, smemH, st>>>(s.part, S, (long long)B * H, H, y.ff_b2, s.z, y.ff_gamma, y.ff_beta, s.x, H, ix);
            GVD_CHECK_LAUNCH();
        }
        const int ldv = rup4i(V);
        GVD_TRY(tfm_product(w->out_w, V, H, s.x, H, B, s.part, ldv, &S, st, s.wi_out, s.ximg, ix));
        if (V <= TFM_HEAD_MAXV) {
            tfm_head_kernel<256><<<B, 256, (size_t)V * sizeof(float), st>>>(s.part, S, (long long)B * ldv, ldv, w->out_b, V, (long long*)seq_out, L, t,
                                                                          logits_out, (const long long*)teacher, s.nll);
            GVD_CHECK_LAUNCH();
        } else {                  // one CTA per (clip, 1024 words), the last CTA of each clip merges
            VocabTailArgs a{};
            a.part = s.part; a.S = S; a.plane = (long long)B * ldv; a.ldp = ldv; a.bias = w->out_b; a.B = B; a.V = V; a.mode = VOCAB_ARGMAX;
            a.seq_out = seq_out ? (long long*)seq_out + t : nullptr; a.out_stride = L;
            a.logits_out = logits_out ? logits_out + (size_t)t * V : nullptr; a.ld_logits = (long long)L * V;
            a.target = teacher ? (const long long*)teacher + t + 1 : nullptr; a.target_stride = L + 1;
            a.nll = teacher ? s.nll + t : nullptr; a.nll_stride = L;
            a.rec = s.vt_rec; a.ticket = s.vt_ticket;
            GVD_TRY(gvd_vocab_tail(a, st));
        }
    }
    if (teacher) {
        tfm_loss_kernel<256><<<1, 256, 0, st>>>(s.nll, (const long long*)teacher, B, L, loss_out);
        GVD_CHECK_LAUNCH();
    }
    return 0;
}

extern "C" GVD_API int gvd_tfm_decode_greedy(const gvd_tfm_weights_t* w, int B, int L, const float* enc0, int n0, const float* enc1, int n1,
                                             const float* pe, void* workspace, size_t workspace_bytes, int64_t* seq_out, float* logits_out,
                                             void* stream) {
    GVD_REQUIRE(seq_out, "tfm_decode_greedy: null seq_out");
    return tfm_run(w, B, L, enc0, n0, enc1, n1, pe, workspace, workspace_bytes, seq_out, logits_out, nullptr, nullptr, stream);
}

// Decoder.forward + mask() + F.cross_entropy (transformer.py:207-212,276-280), eval mode, as S incremental steps with forced tokens: position t
// attends to positions <= t (the causal mask of the batched form), so the numbers are those of the reference's batched pass.
extern "C" GVD_API int gvd_tfm_teacher_fwd(const gvd_tfm_weights_t* w, int B, int S, const float* enc0, int n0, const float* enc1, int n1,
                                           const float* pe, void* workspace, size_t workspace_bytes, const int64_t* seq, float* loss_out, void* stream) {
    GVD_REQUIRE(seq && loss_out, "tfm_teacher_fwd: null argument");
    return tfm_run(w, B, S, enc0, n0, enc1, n1, pe, workspace, workspace_bytes, nullptr, nullptr, seq, loss_out, stream);
}
