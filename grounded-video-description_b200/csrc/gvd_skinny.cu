// Skinny (M = batch <= 128 rows) contractions of the decode step, operand-swapped and split along K (backend bit 3).
//
// Why: with the (padded) batch on the 128-row M side of a tile, every MMA of a decode-step GEMM (B = 100 rows of activations against
// 4096 x 3072 LSTM weights, the 4905 x 1024 vocabulary head, the 1024 x 1024 attention queries) would cover few weight rows.  Swapped, the
// WEIGHT rows are the M side and the batch the N side (two 64-column tiles).  The swap leaves only Nw/128 row blocks per launch (32 for an
// LSTM), so K is split across CTAs as well: split s owns the columns [s.Ks, (s+1).Ks) of both operands — a "batch" of the batched NT GEMM
// whose batch stride is Ks ELEMENTS ALONG K for both operands (the tensor-map trick of the attention heads).
//
// The partial sums leave the GEMM TRANSPOSED (GemmArgs::trans_c): part[s][b][n] with the weight-row index n contiguous, so the
// reductions below are plain coalesced element-wise passes:
//   reduce_lstm      gates partials -> + pre + biases -> LSTMCell pointwise -> h (up to three destinations: the state buffer and the
//                    slots of the concatenated inputs of the next products), c                                (AttModel.py:139,160)
//   reduce_bias      out[b][n] = sum_s part[s][b][n] + bias[n]                                                 (attention queries)
//   reduce_pick      vocabulary head: sum_s + bias -> log-softmax, top-2, UNK rule, next token + its embedding  (model.py:590-615)
//   reduce_sample    vocabulary head: sum_s + bias -> multinomial draw at a temperature (Gumbel-max), next token + its embedding
//                                                                                                              (model.py:595-605)
#include "gvd_common.cuh"
#include "gvd_kernels.cuh"

namespace {

// one thread = one hidden unit of one batch row: 4 gates x S partials + pre + biases; consecutive threads = consecutive units, so every
// access runs along the contiguous dimension (B * H threads: enough parallelism to hide the L2 latency of the partial reads)
__global__ void __launch_bounds__(256) reduce_lstm_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ pre,
                                                          int pre_div, const float* __restrict__ bias1, const float* __restrict__ bias2,
                                                          const float* __restrict__ c_prev, float* __restrict__ c_out, float* __restrict__ h0,
                                                          long long ldh0, float* __restrict__ h1, long long ldh1, float* __restrict__ h2,
                                                          long long ldh2, int B, int H, float* __restrict__ pk1, long long ldpk1,
                                                          float* __restrict__ pk2, long long ldpk2, float pk_scale) {
    const int idx0 = blockIdx.x * blockDim.x + threadIdx.x;
    pdl_trigger();
    pdl_wait();
    const bool valid = idx0 < B * H;
    const int idx = valid ? idx0 : B * H - 1;                            // inactive tail lanes recompute the last element (they take part in the shuffle)
    const int b = idx / H, j = idx % H;
    float g4[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        const float* p = part + (long long)b * ldp + (long long)g * H + j;
        float v = p[0];
        for (int s = 1; s < S; ++s) v += p[s * plane];                    // ascending split order: deterministic
        const long long col = (long long)g * H + j;
        if (pre) v += pre[(long long)(pre_div > 1 ? b / pre_div : b) * 4 * H + col];
        if (bias1) v += __ldg(bias1 + col);
        if (bias2) v += __ldg(bias2 + col);
        g4[g] = v;
    }
    const float ig = sigmoid_acc(g4[0]), fg = sigmoid_acc(g4[1]), gg = tanhf(g4[2]), og = sigmoid_acc(g4[3]);
    const float c = fg * c_prev[(long long)b * H + j] + ig * gg;
    const float h = og * tanhf(c);
    const float hn = __shfl_down_sync(0xffffffffu, h, 1);                 // unit j + 1 (H is even: pairs never straddle rows or warps)
    if (!valid) return;
    c_out[(long long)b * H + j] = c;
    h0[(long long)b * ldh0 + j] = h;
    if (h1) h1[(long long)b * ldh1 + j] = h;
    if (h2) h2[(long long)b * ldh2 + j] = h;
    if (pk1 && !(j & 1)) {                                                // the fp16x3 operand image of h for the next products
        uint32_t hi, lo;
        f16x3_split_pair(h, hn, pk_scale, hi, lo);
        const long long w = f16x3_word(j);
        uint32_t* d1 = reinterpret_cast<uint32_t*>(pk1) + (long long)b * ldpk1 + w;
        d1[0] = hi; d1[16] = lo;
        if (pk2) { uint32_t* d2 = reinterpret_cast<uint32_t*>(pk2) + (long long)b * ldpk2 + w; d2[0] = hi; d2[16] = lo; }
    }
}

__global__ void __launch_bounds__(256) reduce_bias_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias,
                                                          float* __restrict__ out, long long ld_out, int B, int Nw) {
    const int N4 = Nw >> 2;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    pdl_trigger();
    pdl_wait();
    if (idx >= B * N4) return;
    const int b = idx / N4, n = (idx % N4) * 4;
    const float* p = part + (long long)b * ldp + n;
    float4 v = *reinterpret_cast<const float4*>(p);
    for (int s = 1; s < S; ++s) {
        const float4 t = *reinterpret_cast<const float4*>(p + s * plane);
        v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    }
    if (bias) { const float4 t = __ldg(reinterpret_cast<const float4*>(bias + n)); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
    *reinterpret_cast<float4*>(out + (long long)b * ld_out + n) = v;
}

// Vocabulary head tail for one batch row per block: logits = sum_s part + bias held in registers (NPT per thread), ONE pass over memory:
// top-2 (ties -> lower index, torch.topk on the CPU oracle), log-sum-exp, UNK rule (model.py:590-594), next-step embedding (model.py:605).
struct Top2 { float v1, v2; int i1, i2; };
__device__ __forceinline__ void top2_insert(Top2& t, float v, int i) {
    if (v > t.v1 || (v == t.v1 && i < t.i1)) { t.v2 = t.v1; t.i2 = t.i1; t.v1 = v; t.i1 = i; }
    else if (v > t.v2 || (v == t.v2 && i < t.i2)) { t.v2 = v; t.i2 = i; }
}
constexpr int PICK_NT = 1024;
template <int NPT>
__global__ void __launch_bounds__(PICK_NT) reduce_pick_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias,
                                                          int V, int unk_idx, long long* __restrict__ it_out, long long* __restrict__ seq_out,
                                                          float* __restrict__ logp_out, long long out_stride, const float* __restrict__ embed,
                                                          float* __restrict__ xt, long long ld_xt, int E, float* __restrict__ logits_out,
                                                          long long ld_logits, float* __restrict__ xt_pk, long long ld_xt_pk, float pk_scale) {
    __shared__ float red[32];
    __shared__ Top2 wtop[32];
    __shared__ int tok_s;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    pdl_trigger();
    pdl_wait();
    const float* p = part + (long long)b * ldp;
    float x[NPT];
    Top2 t{-INFINITY, -INFINITY, 0x7fffffff, 0x7fffffff};
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
        const int i = threadIdx.x + k * PICK_NT;
        float v = -INFINITY;
        if (i < V) {
            v = p[i];
            for (int s = 1; s < S; ++s) v += p[i + s * plane];
            v += __ldg(bias + i);
            if (logits_out) logits_out[(long long)b * ld_logits + i] = v;
            top2_insert(t, v, i);
        }
        x[k] = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov1 = __shfl_xor_sync(0xffffffffu, t.v1, o), ov2 = __shfl_xor_sync(0xffffffffu, t.v2, o);
        const int oi1 = __shfl_xor_sync(0xffffffffu, t.i1, o), oi2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
        top2_insert(t, ov1, oi1);
        top2_insert(t, ov2, oi2);
    }
    if (lane == 0) wtop[warp] = t;
    __syncthreads();
    t = wtop[lane];                                              // every warp merges the 32 warp results the same way (fixed order)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov1 = __shfl_xor_sync(0xffffffffu, t.v1, o), ov2 = __shfl_xor_sync(0xffffffffu, t.v2, o);
        const int oi1 = __shfl_xor_sync(0xffffffffu, t.i1, o), oi2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
        top2_insert(t, ov1, oi1);
        top2_insert(t, ov2, oi2);
    }
    const float m = t.v1;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NPT; ++k) s += (threadIdx.x + k * PICK_NT < V) ? expf(x[k] - m) : 0.f;
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        const float lse = m + logf(s);
        const bool keep = t.i1 != unk_idx;                       // misc/model.py:590-594
        int it = keep ? t.i1 : t.i2;
        if ((unsigned)it >= (unsigned)V) it = 0;                 // every logit NaN: stay inside the embedding table
        it_out[b] = it;
        if (seq_out) seq_out[(long long)b * out_stride] = it;
        if (logp_out) logp_out[(long long)b * out_stride] = (keep ? t.v1 : t.v2) - lse;
        tok_s = it;
    }
    if (xt) {                                                    // next step's input xt = ReLU(embed[token]) (model.py:79-82,605)
        __syncthreads();
        const float* row = embed + (long long)tok_s * E;
        for (int e = threadIdx.x; e < E; e += blockDim.x) xt[(long long)b * ld_xt + e] = fmaxf(row[e], 0.f);
        if (xt_pk) {                                             // and its fp16x3 operand image (E is even)
            uint32_t* d = reinterpret_cast<uint32_t*>(xt_pk) + (long long)b * ld_xt_pk;
            for (int e2 = threadIdx.x; 2 * e2 < E; e2 += blockDim.x) {
                uint32_t hi, lo;
                f16x3_split_pair(fmaxf(row[2 * e2], 0.f), fmaxf(row[2 * e2 + 1], 0.f), pk_scale, hi, lo);
                const long long w = f16x3_word(2 * e2);
                d[w] = hi; d[w + 16] = lo;
            }
        }
    }
}

// Multinomial sampling (sample_max = 0, model.py:595-603): it ~ softmax(logit / temperature), drawn with the Gumbel-max trick
//   it = argmax_i (logit_i / temperature + g_i),  g_i = -log(-log(u_i)),  ties -> lower index,
//   logp = logit_it - logsumexp(logit)                    (untempered, model.py:602; no UNK rule in this branch)
// u_i for batch row b, decode step t: word (i & 3) of Philox4x32-10(counter = (i >> 2, b, t, 0), key = seed), u = ((word >> 9) + 0.5) 2^-23:
// 23-bit uniforms strictly inside (0, 1), exact in fp32, so g lies in [-2.82, 16.64] and a word whose key is more than ~19.5 below the
// best is never drawn (its probability is < 1e-8).  b is the row's index in THIS launch: splitting a batch changes the draws.
// A row whose keys are all -inf or all NaN yields token 0.
__device__ __forceinline__ float gumbel_from_word(uint32_t w) {
    const float u = ((float)(w >> 9) + 0.5f) * (1.f / 8388608.f);
    return -logf(-logf(u));
}
struct ArgKey { float key, logit; int i; };
__device__ __forceinline__ void argkey_merge(ArgKey& a, float key, float logit, int i) {
    if (key > a.key || (key == a.key && i < a.i)) { a.key = key; a.logit = logit; a.i = i; }
}
template <int NPT>
__global__ void __launch_bounds__(PICK_NT) reduce_sample_kernel(const float* __restrict__ part, int S, long long plane, int ldp, const float* __restrict__ bias,
                                                            int V, const GvdSampleParams* __restrict__ par, int step, long long* __restrict__ it_out,
                                                            long long* __restrict__ seq_out, float* __restrict__ logp_out, long long out_stride,
                                                            const float* __restrict__ embed, float* __restrict__ xt, long long ld_xt, int E,
                                                            float* __restrict__ xt_pk, long long ld_xt_pk, float pk_scale) {
    __shared__ __align__(16) float gum[PICK_NT * NPT];
    __shared__ float red[32];
    __shared__ ArgKey wbest[32];
    __shared__ float wmax[32];
    __shared__ int tok_s;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    pdl_trigger();
    // the noise depends on nothing the decode loop writes: drawn before waiting for the previous kernel
    const uint32_t seed_lo = par->seed_lo, seed_hi = par->seed_hi;
    const float temperature = par->temperature;
    for (int q = threadIdx.x; 4 * q < V; q += PICK_NT) {
        uint32_t r[4];
        philox4x32_10((uint32_t)q, (uint32_t)b, (uint32_t)step, 0u, seed_lo, seed_hi, r);
        reinterpret_cast<float4*>(gum)[q] = make_float4(gumbel_from_word(r[0]), gumbel_from_word(r[1]), gumbel_from_word(r[2]), gumbel_from_word(r[3]));
    }
    pdl_wait();
    __syncthreads();
    const float* p = part + (long long)b * ldp;
    float x[NPT];
    ArgKey a{-INFINITY, -INFINITY, 0x7fffffff};
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < NPT; ++k) {
        const int i = threadIdx.x + k * PICK_NT;
        float v = -INFINITY;
        if (i < V) {
            v = p[i];
            for (int s = 1; s < S; ++s) v += p[i + s * plane];
            if (bias) v += __ldg(bias + i);
            m = fmaxf(m, v);
            argkey_merge(a, v / temperature + gum[i], v, i);
        }
        x[k] = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ok = __shfl_xor_sync(0xffffffffu, a.key, o), ol = __shfl_xor_sync(0xffffffffu, a.logit, o);
        const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
        argkey_merge(a, ok, ol, oi);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    if (lane == 0) { wbest[warp] = a; wmax[warp] = m; }
    __syncthreads();
    a = wbest[lane];                                             // every warp merges the 32 warp results the same way (fixed order)
    m = wmax[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ok = __shfl_xor_sync(0xffffffffu, a.key, o), ol = __shfl_xor_sync(0xffffffffu, a.logit, o);
        const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
        argkey_merge(a, ok, ol, oi);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NPT; ++k) s += (threadIdx.x + k * PICK_NT < V) ? expf(x[k] - m) : 0.f;
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        int it = a.i;
        if ((unsigned)it >= (unsigned)V) it = 0;                 // every key NaN: stay inside the embedding table
        it_out[b] = it;
        if (seq_out) seq_out[(long long)b * out_stride] = it;
        if (logp_out) logp_out[(long long)b * out_stride] = a.logit - (m + logf(s));
        tok_s = it;
    }
    if (xt) {                                                    // next step's input xt = ReLU(embed[token]) (model.py:79-82,605)
        __syncthreads();
        const float* row = embed + (long long)tok_s * E;
        for (int e = threadIdx.x; e < E; e += blockDim.x) xt[(long long)b * ld_xt + e] = fmaxf(row[e], 0.f);
        if (xt_pk) {                                             // and its fp16x3 operand image (E is even)
            uint32_t* d = reinterpret_cast<uint32_t*>(xt_pk) + (long long)b * ld_xt_pk;
            for (int e2 = threadIdx.x; 2 * e2 < E; e2 += blockDim.x) {
                uint32_t hi, lo;
                f16x3_split_pair(fmaxf(row[2 * e2], 0.f), fmaxf(row[2 * e2 + 1], 0.f), pk_scale, hi, lo);
                const long long w = f16x3_word(2 * e2);
                d[w] = hi; d[w + 16] = lo;
            }
        }
    }
}

// Vocabulary head tail for any V (the two kernels above hold a whole row in one CTA's registers: at most 6 x 1024 words).
// Grid (row b, slice j): slice j covers the words [j * VOCAB_SLICE, (j + 1) * VOCAB_SLICE), thread x the four consecutive words from
// 4x on (one float4 per plane: ldp % 4 == 0 keeps the last group inside the row).  For sampling those four words are exactly the four
// outputs of Philox counter (i >> 2, b, step, 0), the noise of reduce_sample_kernel.  Each CTA writes one record of its slice:
//   m  = slice max (greedy / argmax: its top-1 value, as reduce_pick_kernel),  s = sum exp(x - m) over the slice (0 when m = -inf),
//   greedy / argmax: v1 i1 v2 i2 = the slice's top-2;  sampling: v1 i1 = its best key and that word, v2 = the word's raw logit.
// The last CTA of the row (ticket) merges the records in a fixed order — lane l of warp 0 takes slices l, l + 32, ... ascending, then a
// butterfly — so the result does not depend on which CTA finishes last, and writes the token, its log-prob and the next input.
constexpr int VT_NT = VOCAB_SLICE / 4;
struct VocabRec { float m, s, v1, v2; int i1, i2, pad0, pad1; };
__device__ __forceinline__ void top2_butterfly(Top2& t) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov1 = __shfl_xor_sync(0xffffffffu, t.v1, o), ov2 = __shfl_xor_sync(0xffffffffu, t.v2, o);
        const int oi1 = __shfl_xor_sync(0xffffffffu, t.i1, o), oi2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
        top2_insert(t, ov1, oi1);
        top2_insert(t, ov2, oi2);
    }
}
__device__ __forceinline__ void argkey_butterfly(ArgKey& a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ok = __shfl_xor_sync(0xffffffffu, a.key, o), ol = __shfl_xor_sync(0xffffffffu, a.logit, o);
        const int oi = __shfl_xor_sync(0xffffffffu, a.i, o);
        argkey_merge(a, ok, ol, oi);
    }
}
template <int MODE>
__global__ void __launch_bounds__(VT_NT) vocab_tail_kernel(const VocabTailArgs a) {
    __shared__ float red[32];
    __shared__ Top2 wtop[VT_NT / 32];
    __shared__ ArgKey wbest[VT_NT / 32];
    __shared__ int last_s, tok_s;
    const int b = blockIdx.x, slice = blockIdx.y, nsl = gridDim.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i0 = slice * VOCAB_SLICE + 4 * threadIdx.x;
    const int V = a.V;
    pdl_trigger();
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    float temperature = 1.f;
    if (MODE == VOCAB_SAMPLE) {     // the noise depends on nothing the decode loop writes: drawn before waiting for the previous kernel
        temperature = a.par->temperature;
        if (i0 < V) {
            uint32_t r[4];
            philox4x32_10((uint32_t)(i0 >> 2), (uint32_t)b, (uint32_t)a.step, 0u, a.par->seed_lo, a.par->seed_hi, r);
#pragma unroll
            for (int j = 0; j < 4; ++j) g[j] = gumbel_from_word(r[j]);
        }
    }
    pdl_wait();
    const float* p = a.part + (long long)b * a.ldp;
    float x[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    if (i0 < V) {
        float4 v = *reinterpret_cast<const float4*>(p + i0);
        for (int s = 1; s < a.S; ++s) {                                  // ascending split order, as the other tails
            const float4 t = *reinterpret_cast<const float4*>(p + i0 + s * a.plane);
            v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
        }
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (i0 + j < V) {
                x[j] = a.bias ? vv[j] + __ldg(a.bias + i0 + j) : vv[j];
                if (a.logits_out) a.logits_out[(long long)b * a.ld_logits + i0 + j] = x[j];
            }
        }
    }
    float m;
    Top2 t{-INFINITY, -INFINITY, 0x7fffffff, 0x7fffffff};
    ArgKey k{-INFINITY, -INFINITY, 0x7fffffff};
    if (MODE == VOCAB_SAMPLE) {
        m = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (i0 + j < V) { m = fmaxf(m, x[j]); argkey_merge(k, x[j] / temperature + g[j], x[j], i0 + j); }
        argkey_butterfly(k);
        if (lane == 0) wbest[warp] = k;
        m = block_max(m, red);                                           // (its barriers publish wbest)
        k = lane < VT_NT / 32 ? wbest[lane] : ArgKey{-INFINITY, -INFINITY, 0x7fffffff};
        argkey_butterfly(k);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (i0 + j < V) top2_insert(t, x[j], i0 + j);
        top2_butterfly(t);
        if (lane == 0) wtop[warp] = t;
        __syncthreads();
        t = lane < VT_NT / 32 ? wtop[lane] : Top2{-INFINITY, -INFINITY, 0x7fffffff, 0x7fffffff};
        top2_butterfly(t);
        m = t.v1;
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += (i0 + j < V) ? expf(x[j] - m) : 0.f;
    s = block_sum(s, red);
    VocabRec* rec = reinterpret_cast<VocabRec*>(a.rec) + (long long)b * nsl;
    if (threadIdx.x == 0) {
        if (m == -INFINITY) s = 0.f;
        rec[slice] = MODE == VOCAB_SAMPLE ? VocabRec{m, s, k.key, k.logit, k.i, 0, 0, 0} : VocabRec{m, s, t.v1, t.v2, t.i1, t.i2, 0, 0};
        __threadfence();                                                 // publish the record before taking a ticket
        last_s = atomicAdd(a.ticket + b, 1) == nsl - 1;
    }
    __syncthreads();
    if (!last_s) return;
    __threadfence();
    if (warp == 0) {
        float M = -INFINITY;
        t = Top2{-INFINITY, -INFINITY, 0x7fffffff, 0x7fffffff};
        k = ArgKey{-INFINITY, -INFINITY, 0x7fffffff};
        for (int j = lane; j < nsl; j += 32) {
            const float4 r = __ldcg(reinterpret_cast<const float4*>(rec + j));
            const int2 ri = __ldcg(reinterpret_cast<const int2*>(rec + j) + 2);
            M = fmaxf(M, r.x);
            if (MODE == VOCAB_SAMPLE) argkey_merge(k, r.z, r.w, ri.x);
            else { top2_insert(t, r.z, ri.x); top2_insert(t, r.w, ri.y); }
        }
        M = warp_max(M);
        if (MODE == VOCAB_SAMPLE) argkey_butterfly(k); else top2_butterfly(t);
        float sum = 0.f;
        for (int j = lane; j < nsl; j += 32) {
            const float2 r = __ldcg(reinterpret_cast<const float2*>(rec + j));
            if (r.x != -INFINITY) sum += r.y * expf(r.x - M);
        }
        sum = warp_sum(sum);
        if (lane == 0) {
            const float lse = M + logf(sum);
            int it;
            float lv;
            if (MODE == VOCAB_SAMPLE) { it = k.i; lv = k.logit; }                 // no UNK rule when sampling (model.py:595-603)
            else {
                const bool keep = MODE == VOCAB_ARGMAX || t.i1 != a.unk_idx;     // misc/model.py:590-594
                it = keep ? t.i1 : t.i2;
                lv = keep ? t.v1 : t.v2;
            }
            if ((unsigned)it >= (unsigned)V) it = 0;                             // no finite comparison: stay inside the embedding table
            if (a.it_out) a.it_out[b] = it;
            if (a.seq_out) a.seq_out[(long long)b * a.out_stride] = it;
            if (a.logp_out) a.logp_out[(long long)b * a.out_stride] = lv - lse;
            if (a.nll) {                                                         // teacher forcing (transformer.py:51-54)
                const long long tgt = a.target[(long long)b * a.target_stride];
                float y = 0.f;
                if (tgt > 0 && tgt < V) {                                        // the target's logit, summed in the order of the slice pass
                    y = p[tgt];
                    for (int s2 = 1; s2 < a.S; ++s2) y += p[tgt + s2 * a.plane];
                    if (a.bias) y += __ldg(a.bias + tgt);
                    y = lse - y;
                }
                a.nll[(long long)b * a.nll_stride] = y;
            }
            tok_s = it;
            a.ticket[b] = 0;                                                     // ready for the next launch
        }
    }
    if (a.xt) {                                                  // next step's input xt = ReLU(embed[token]) (model.py:79-82,605)
        __syncthreads();
        const float* row = a.embed + (long long)tok_s * a.E;
        for (int e = threadIdx.x; e < a.E; e += blockDim.x) a.xt[(long long)b * a.ld_xt + e] = fmaxf(row[e], 0.f);
        if (a.xt_pk) {                                           // and its fp16x3 operand image (E is even)
            uint32_t* d = reinterpret_cast<uint32_t*>(a.xt_pk) + (long long)b * a.ld_xt_pk;
            for (int e2 = threadIdx.x; 2 * e2 < a.E; e2 += blockDim.x) {
                uint32_t hi, lo;
                f16x3_split_pair(fmaxf(row[2 * e2], 0.f), fmaxf(row[2 * e2 + 1], 0.f), GVD_F16_SA, hi, lo);
                const long long w = f16x3_word(2 * e2);
                d[w] = hi; d[w + 16] = lo;
            }
        }
    }
}

}  // namespace

// Number of K splits for a skinny product with Nw weight rows and Ktot columns (0 = shape not supported by this path):
// as many CTAs as fit in one wave of the 132 SMs, every split a whole number of 32-wide K slices and at least two of them.
int gvd_skinny_splits(int Nw, int Ktot, int B) {
    if (B < 1 || B > 128 || Nw < 128 || Ktot % 32 != 0) return 0;
    const int mt = gvd_cdiv(Nw, 128);
    int S = 132 / mt;
    if (S < 1) return 0;
    if (S > Ktot / 64) S = Ktot / 64;
    while (S > 1 && Ktot % (S * 32) != 0) --S;
    return S < 1 ? 0 : S;
}

// part[s][b][n] = sum_{k in split s} W[n][k] X[b][k]   (W [Nw, Ktot] row-major; X [B, Ktot] with row pitch ldx; part row pitch ldp >= Nw,
// ldp % 4 == 0; plane stride = B * ldp)
int gvd_skinny_splitk(const float* W, int Nw, int Ktot, const float* X, long long ldx, int B, int S, float* part, int ldp, cudaStream_t st) {
    GVD_REQUIRE(W && X && part && S >= 1 && Ktot % (S * 32) == 0 && ldp >= Nw && ldp % 4 == 0 && ldx % 4 == 0, "skinny_splitk: bad split (Ktot=%d S=%d)", Ktot, S);
    const int Ks = Ktot / S;
    GemmArgs g{};
    g.A = W; g.lda = Ktot; g.sAb = Ks;             // batch entry s = the K range [s.Ks, (s+1).Ks) of the same rows
    g.W = X; g.ldw = ldx; g.sWb = Ks;
    g.C = part; g.ldc = ldp; g.sCb = (long long)B * ldp;
    g.M = Nw; g.N = B; g.K = Ks; g.nh = 1; g.act = GVD_ACT_NONE; g.alpha = 1.f;
    g.trans_c = 1;                                 // partials come out batch-major
    return gvd_gemm_nt_tc(g, S, st);
}

int gvd_reduce_lstm(const float* part, int S, int ldp, const float* pre, int pre_div, const float* bias1, const float* bias2, const float* c_prev,
                    float* c_out, float* h0, long long ldh0, float* h1, long long ldh1, float* h2, long long ldh2, int B, int H, cudaStream_t st,
                    float* pk1, long long ldpk1, float* pk2, long long ldpk2) {
    GVD_REQUIRE(H % 4 == 0 && ldp % 4 == 0 && ldh0 % 4 == 0 && ldh1 % 4 == 0 && ldh2 % 4 == 0 && h0, "reduce_lstm: 16-byte granularity");
    GVD_REQUIRE(!pk1 || (H % 32 == 0 && ldpk1 % 32 == 0 && ldpk2 % 32 == 0), "reduce_lstm: packed destinations need 32-column granularity");
    const int n = B * H;
    GVD_CHECK_CUDA(gvd_launch(reduce_lstm_kernel, dim3(gvd_cdiv(n, 256)), dim3(256), 0, st, part, S, (long long)B * ldp, ldp, pre, pre_div, bias1, bias2, c_prev,
                              c_out, h0, ldh0, h1, ldh1, h2, ldh2, B, H, pk1, ldpk1, pk2, ldpk2, GVD_F16_SA));
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_reduce_bias(const float* part, int S, int Nw, int ldp, const float* bias, float* out, long long ld_out, int B, cudaStream_t st) {
    GVD_REQUIRE(Nw % 4 == 0 && ldp % 4 == 0 && ld_out % 4 == 0, "reduce_bias: 16-byte granularity");
    const int n = B * (Nw / 4);
    GVD_CHECK_CUDA(gvd_launch(reduce_bias_kernel, dim3(gvd_cdiv(n, 256)), dim3(256), 0, st, part, S, (long long)B * ldp, ldp, bias, out, ld_out, B, Nw));
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_reduce_pick(const float* part, int S, int ldp, const float* bias, int B, int V, int unk_idx, long long* it_out, long long* seq_out,
                    float* logp_out, long long out_stride, const float* embed, float* xt, long long ld_xt, int E, float* logits_out,
                    long long ld_logits, cudaStream_t st, float* xt_pk, long long ld_xt_pk) {
    GVD_REQUIRE(V >= 2 && V <= PICK_NT * 6 && bias && it_out, "reduce_pick: vocabulary of 2..6144 entries");
    GVD_REQUIRE(!xt_pk || (xt && E % 2 == 0 && ld_xt_pk % 32 == 0 && ld_xt_pk >= (E + 31) / 32 * 32),
                "reduce_pick: the packed xt needs an even E and a 32-multiple pitch covering E");
    const long long plane = (long long)B * ldp;
    if (V <= PICK_NT * 2) GVD_CHECK_CUDA(gvd_launch(reduce_pick_kernel<2>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, unk_idx, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, logits_out, ld_logits, xt_pk, ld_xt_pk, GVD_F16_SA));
    else if (V <= PICK_NT * 5) GVD_CHECK_CUDA(gvd_launch(reduce_pick_kernel<5>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, unk_idx, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, logits_out, ld_logits, xt_pk, ld_xt_pk, GVD_F16_SA));
    else GVD_CHECK_CUDA(gvd_launch(reduce_pick_kernel<6>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, unk_idx, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, logits_out, ld_logits, xt_pk, ld_xt_pk, GVD_F16_SA));
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_reduce_sample(const float* part, int S, int ldp, const float* bias, int B, int V, const GvdSampleParams* params, int step,
                      long long* it_out, long long* seq_out, float* logp_out, long long out_stride, const float* embed, float* xt,
                      long long ld_xt, int E, cudaStream_t st, float* xt_pk, long long ld_xt_pk) {
    GVD_REQUIRE(V >= 2 && V <= PICK_NT * 6 && params && it_out && step >= 0, "reduce_sample: vocabulary of 2..6144 entries");
    GVD_REQUIRE(!xt_pk || (xt && E % 2 == 0 && ld_xt_pk % 32 == 0 && ld_xt_pk >= (E + 31) / 32 * 32),
                "reduce_sample: the packed xt needs an even E and a 32-multiple pitch covering E");
    const long long plane = (long long)B * ldp;
    if (V <= PICK_NT * 2) GVD_CHECK_CUDA(gvd_launch(reduce_sample_kernel<2>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, params, step, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, xt_pk, ld_xt_pk, GVD_F16_SA));
    else if (V <= PICK_NT * 5) GVD_CHECK_CUDA(gvd_launch(reduce_sample_kernel<5>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, params, step, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, xt_pk, ld_xt_pk, GVD_F16_SA));
    else GVD_CHECK_CUDA(gvd_launch(reduce_sample_kernel<6>, dim3(B), dim3(PICK_NT), 0, st, part, S, plane, ldp, bias, V, params, step, it_out, seq_out, logp_out, out_stride, embed, xt, ld_xt, E, xt_pk, ld_xt_pk, GVD_F16_SA));
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_vocab_tail(const VocabTailArgs& a, cudaStream_t st) {
    GVD_REQUIRE(a.part && a.S >= 1 && a.B >= 1 && a.V >= 2 && a.ldp >= a.V && a.ldp % 4 == 0 && a.plane % 4 == 0 && ((uintptr_t)a.part & 15) == 0,
                "vocab_tail: partial planes need V >= 2, a 4-multiple pitch >= V and 16-byte alignment (V=%d ldp=%d)", a.V, a.ldp);
    GVD_REQUIRE(gvd_vocab_slices(a.V) <= 65535, "vocab_tail: vocabulary of at most %d words (got %d)", 65535 * VOCAB_SLICE, a.V);
    GVD_REQUIRE(a.rec && ((uintptr_t)a.rec & 15) == 0 && a.ticket, "vocab_tail: records and tickets needed");
    GVD_REQUIRE(a.mode == VOCAB_GREEDY || a.mode == VOCAB_ARGMAX || (a.mode == VOCAB_SAMPLE && a.par && a.step >= 0), "vocab_tail: bad mode %d", a.mode);
    GVD_REQUIRE((!a.xt || a.embed) && (!a.nll || a.target), "vocab_tail: xt needs the embedding, nll the targets");
    GVD_REQUIRE(!a.xt_pk || (a.xt && a.E % 2 == 0 && a.ld_xt_pk % 32 == 0 && a.ld_xt_pk >= (a.E + 31) / 32 * 32),
                "vocab_tail: the packed xt needs an even E and a 32-multiple pitch covering E");
    const dim3 grid(a.B, gvd_vocab_slices(a.V));
    if (a.mode == VOCAB_GREEDY) GVD_CHECK_CUDA(gvd_launch(vocab_tail_kernel<VOCAB_GREEDY>, grid, dim3(VT_NT), 0, st, a));
    else if (a.mode == VOCAB_SAMPLE) GVD_CHECK_CUDA(gvd_launch(vocab_tail_kernel<VOCAB_SAMPLE>, grid, dim3(VT_NT), 0, st, a));
    else GVD_CHECK_CUDA(gvd_launch(vocab_tail_kernel<VOCAB_ARGMAX>, grid, dim3(VT_NT), 0, st, a));
    GVD_CHECK_LAUNCH();
    return 0;
}
