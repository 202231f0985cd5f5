// gvd: fp32-faithful NT GEMM family on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   C[M,N] = act(alpha * A[M,K] . W[N,K]^T + bias)      A, W, C fp32 in HBM, K contiguous
//
// Greedy token ids must be bit-exact against an fp32 oracle, so plain TF32 (10-bit mantissa) is not
// enough (SURVEY.md section 7).  Each operand is split into a "hi" and a "lo" part (x = hi + lo to ~21
// bits) and three tensor-core products accumulate  lo.hi + hi.lo + hi.hi :
//   3xTF32 : hi = tf32(x), lo = x - hi, wgmma m64n64k8 tf32 (gradient products: full fp32 exponent range)
//   fp16x3 : hi = fp16(round11(s x)), lo = fp16(s x - hi) with a power-of-two scale s, wgmma m64n64k16 f16
//            (forward products with O(1) operands; half the MMAs and operand bytes).  An operand may arrive
//            already split, as the fp16x3 operand image of gvd_common.cuh: per row and 32-wide K slice 64 B
//            of hi halves | 64 B of lo halves = one SWIZZLE_128B row of a K-major wgmma operand.
//
// wg_gemm_kernel serves the whole family but the prologue's operand-image GEMMs.  Per CTA (one 128 x 64 output tile, K streamed in
// 32-element = 128-byte slices through a ring of stages):
//   warp 8    : TMA producer  - cp.async.bulk.tensor (SWIZZLE_128B) of the A / W slices, one mbarrier per stage
//   warps 0-7 : two consumer warpgroups.  All 256 threads split the raw fp32 slices of the stage in shared
//               memory (skipped for pre-split operands), fence.proxy.async, then each warpgroup issues the
//               wgmma products of ITS 64 rows and folds the slice's result into fp32 register accumulators
//               (round-to-nearest adds; the tensor core's own accumulation is only trusted for one slice).
//   epilogue  : the accumulator fragments are exchanged through shared memory so that every thread owns one
//               output row (thread <-> row, lane <-> row within the warp); the epilogues are written for
//               that layout: bias / activation store, transposed split-K partial, fused LSTM cell, fused
//               greedy pick, fused GRU cell.
// Up to three K segments (different A / W tensors) feed one accumulator, so the LSTM gate GEMMs never
// materialise a concatenated input (AttModel.py:138,147-160).
//
// ss_gemm_kernel runs the prologue's dense GEMMs, whose operands both arrive as fp16x3 operand images (nothing to convert), on
// 128 x 128 tiles (a third less L2 -> SM operand traffic per MAC than 128 x 64) and warp-specialized, 384 threads:
//   warpgroup 2    : TMA producer (one thread, setmaxnreg 40), the same 4-stage ring of 32 KB stages
//   warpgroups 0-1 : consumers (setmaxnreg 232), 64 rows each.  The m64n128k16 products of slice i go into one of two result sets and
//                    are in flight while slice i - 1 is folded from the other one, so the tensor core does not idle during the fold.
// Per output element the products (lo.hi, hi.lo, hi.hi per k16 step, the first of a slice not accumulating) and the fold order are
// those of wg_gemm_kernel's fp16x3 products, so both kernels give the same bits.
#include <cuda.h>

#include <algorithm>
#include <cstdlib>

#include "gvd_wgmma.cuh"

namespace {

constexpr int TC_BM = 128;
constexpr int TC_BN = 64;
constexpr int WG_CONSUMERS = 256;         // two warpgroups
constexpr int WG_THREADS = WG_CONSUMERS + 32;
constexpr int WG_STAGES = 4;              // also at 128-wide tiles (32 KB stages): 6 stages measured no faster on the H100
constexpr int WG_UJ = 16;                 // hidden units per CTA of the gate-interleaved tiles (LSTM: 4 x 16, GRU: 3 x 16 columns)
constexpr int SS_BN = 128;                // tile width of ss_gemm_kernel
constexpr int SS_THREADS = 384;           // two consumer warpgroups + the producer warpgroup

enum { MODE_STORE = 0, MODE_LSTM = 1, MODE_PICK = 2, MODE_TRANS = 3, MODE_GRU = 5 };

struct TcSeg {
    int k_len;          // K extent of this segment
    int a_k0, w_k0;     // starting K coordinate inside the A / W tensor maps
};
struct SsParams {
    float* C; long long ldc;
    int M, N;
    int nk;                                             // 32-wide K slices
    float oscale;                                       // inverse product of the operand images' power-of-two scales
    const float* bias; const float* scale2; const float* shift2; int act;
    uint32_t* img; long long ld_img; float img_scale;   // also store the fp16x3 operand image of the (activated) output: the next GEMM streams
                                                        // it directly; C may then be null (output consumed by that GEMM only)
    // Q|K|V projection of the region encoder (qkv_hp > 0; N = 3 * qkv_hp head-padded columns): columns [0, HP) = Q -> fp32 C;
    // [HP, 2HP) = K -> per-head fp16x3 image k_img[(row * nh + h) * KH + word(c)] (the W operand of the score product); [2HP, 3HP) = V -> image
    // of V^T per clip vt_img[(b * HP + c) * Rp + word(r)] (the W operand of the P.V product).  Replaces pack_heads / transpose_pack passes.
    int qkv_hp, qkv_hs, qkv_kh, qkv_nh, qkv_R, qkv_Rp;
    uint32_t *k_img, *vt_img;
    float qkv_sk, qkv_sv;
};
struct GruStepParams {
    const float* gi;            // [B, T, 6G]  W_ih x + b_ih, direction d at column offset d * 3G
    const float* bhh;           // [2][3G]
    const float* h_prev;        // [2][B][G] fp32
    float* h_new;               // [2][B][G] fp32
    float* h_img_new;           // [2][B][G] words: fp16x3 image of h_new (A operand of the next step)
    float* out;                 // [B, T, 2G]
    const long long* sample_idx;
    int B, T, G, step;
    float sa;
};
struct TcParams {
    TcSeg seg[3];
    int nseg;
    int ksplit;                           // split-K: blockIdx.z also advances both operands by this many K elements (0: batched product)
    int M, N;
    int nh;                               // heads per batch entry: blockIdx.z = b * nh + h
    int a_mul_h, a_mul_b, w_mul_h, w_mul_b; // 0 when the operand is shared across that batch axis (stride 0), else 1
    float* C; long long ldc, sCb, sCh;
    const float* bias; long long sBb;
    const float* scale2; const float* shift2;
    int act;
    float alpha;
    int mode;
    int nbox, box_stride;                 // gate-interleaved W tile: nbox boxes of WG_UJ rows, box g at row g * box_stride + first unit
    int f16;                              // fp16x3 products (else 3xTF32)
    int apre, wpre;                       // fp16x3: the operand arrives as its operand image (no conversion)
    float sa, sw, oscale;                 // fp16x3: power-of-two operand scales applied before the split and their inverse product
    const float* Fc; int ngrp;            // per-(row, K slice) factor of the A operand, [batch][ngrp][M] (softmax factors of the P.V product) or null
    // LSTM mode: columns are gate-major [4][WG_UJ]; row block of W = gate * H + first unit
    int H;
    const float* pre;                     // [B / pre_div, 4H] additive term or nullptr
    int pre_div;
    const float* bias1; const float* bias2;
    const float* c_prev; float* h_out; float* c_out;
    // greedy-sampler mode: the vocabulary-head GEMM never stores its logits; every CTA reduces its columns to
    // (max, sum-exp, top-2) per clip and the last CTA to finish merges them, applies the UNK rule and embeds the next token
    float* pk_part; int* pk_ticket;                         // [gridDim.x][M][8] partials, one zero-initialised counter
    long long* pk_it; long long* pk_seq; float* pk_logp;    // next token [M]; seq / logprob outputs with stride pk_stride (may be null)
    long long pk_stride;
    int pk_unk;
    const float* pk_embed; float* pk_xt; int pk_E;          // xt[M, E] = ReLU(embed[token]) for the next step
    GruStepParams gru;
};

__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts128u(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// x (scaled) -> fp16 hi | fp16 lo of 4 consecutive K values: hi = round-to-11-bits(x) (exact in fp16), lo = fp16(x - hi)
__device__ __forceinline__ void split_h4(const float4& v, float s, uint32_t& h01, uint32_t& h23, uint32_t& l01, uint32_t& l23) {
    f16x3_split_pair(v.x, v.y, s, h01, l01);
    f16x3_split_pair(v.z, v.w, s, h23, l23);
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(WG_CONSUMERS) : "memory"); }

template <bool F16> struct WgCfg {
    static constexpr int A_BYTES = TC_BM * 128;            // one plane of the A slice (fp16x3: the whole slice, hi | lo halves per row)
    static constexpr int B_BYTES = TC_BN * 128;
    static constexpr int STAGE = F16 ? (A_BYTES + B_BYTES) : 2 * (A_BYTES + B_BYTES);
    static constexpr int B_OFF = F16 ? A_BYTES : 2 * A_BYTES;
    static constexpr int LDS = TC_BN + 4;                  // pitch of the fp32 exchange tile of the epilogue
    static constexpr size_t SMEM = (size_t)WG_STAGES * STAGE + 1024 /*align*/ + 8 * 2 * WG_STAGES + 64;
    static_assert((size_t)WG_STAGES * STAGE >= (size_t)TC_BM * LDS * 4, "the epilogue exchanges the C tile through the pipeline buffers");
    static_assert(SMEM <= 232448, "shared-memory budget (227 KB per CTA)");
};
struct SsCfg {                                             // ss_gemm_kernel: both slices are fp16x3 images, hi | lo halves per 128-byte row
    static constexpr int A_BYTES = TC_BM * 128;
    static constexpr int B_BYTES = SS_BN * 128;
    static constexpr int STAGE = A_BYTES + B_BYTES;
    static constexpr int LDS = SS_BN + 4;
    static constexpr size_t SMEM = (size_t)WG_STAGES * STAGE + 1024 /*align*/ + 8 * 2 * WG_STAGES + 64;
    static_assert((size_t)WG_STAGES * STAGE >= (size_t)TC_BM * LDS * 4, "the epilogue exchanges the C tile through the pipeline buffers");
    static_assert(SMEM <= 232448, "shared-memory budget (227 KB per CTA)");
};

// Q|K|V epilogue of ss_gemm_kernel (p.qkv_hp): stores the exchanged fp32 tile Cs (rows m0.., columns n0..) so that one store instruction
// of a warp writes whole 128-byte lines.  Every output word belongs to exactly one tile: a 4-column group (never straddles a tile, a head or
// Q / K / V: HS % 4 == HP % 4 == 0) to the tile holding its columns, the K padding words [HS, KH) of a head to the tile holding the head's
// last group, the V^T pad rows [R, Rp) of a clip to the tile holding the clip's last row.  tests/test_qkv_epilogue_emulation.py runs this
// plan over every tile of a launch on the CPU.
__device__ __forceinline__ void ss_store_qkv(const SsParams& p, const float* Cs, const int m0, const int n0, const int warp, const int lane) {
    constexpr int LDS_ = SsCfg::LDS, NW = WG_CONSUMERS / 32;
    const int HP = p.qkv_hp, HS = p.qkv_hs, KH = p.qkv_kh, R = p.qkv_R, mend = min(m0 + TC_BM, p.M);
    // Q (columns [0, HP) -> fp32 C): warp <-> row, lane l <-> columns [4 l, 4 l + 4), a 512-byte segment of C per instruction
    if (n0 < HP) {
        const int c = 4 * lane;
        for (int r = warp; m0 + r < mend; r += NW)
            if (n0 + c < HP)
                *reinterpret_cast<float4*>(p.C + (long long)(m0 + r) * p.ldc + n0 + c) = *reinterpret_cast<const float4*>(Cs + r * LDS_ + c);
    }
    // K (columns [HP, 2HP) -> k_img[(m * nh + h) * KH + word(c)]): warp <-> row, lane <-> 4-word quad u of a head's image row, which holds
    // the hi (u & 4 == 0) or lo words of the two groups at columns 32 (u >> 3) + 8 (u & 3) + {0, 4}; 32 consecutive quads are 4 whole lines
    const int ka = max(n0, HP) - HP, kb = min(n0 + SS_BN, 2 * HP) - HP;        // this tile's K columns [ka, kb)
    if (ka < kb) {
        const int KQ = KH / 4, hlo = ka / HS, hhi = (kb - 1) / HS;
        const int q0 = hlo * KQ + ((ka - hlo * HS) >> 5) * 8;                  // from the 32-column slice holding column ka ...
        const int q1 = hhi * HS + HS - 4 < kb ? (hhi + 1) * KQ                  // ... to the end of head hhi's padding if its last group is here
                                              : hhi * KQ + (((kb - 1 - hhi * HS) >> 5) + 1) * 8;
        for (int r = warp; m0 + r < mend; r += NW) {
            uint32_t* dk = p.k_img + (long long)(m0 + r) * p.qkv_nh * KH;
            for (int q = q0 + lane; q < q1; q += 32) {
                const int h = q / KQ, u = q - h * KQ, c = (u >> 3) * 32 + (u & 3) * 8, last = h * HS + HS - 4;
                bool own[2];
                uint32_t w[4];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int g = c + 4 * e, kc = h * HS + g;
                    own[e] = g < HS ? (kc >= ka && kc < kb) : (last >= ka && last < kb);
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);                 // padding words are the split of zeros
                    if (g < HS && own[e]) v = *reinterpret_cast<const float4*>(Cs + r * LDS_ + HP + kc - n0);
                    uint32_t h0, l0, h1, l1;
                    f16x3_split_pair(v.x, v.y, p.qkv_sk, h0, l0);
                    f16x3_split_pair(v.z, v.w, p.qkv_sk, h1, l1);
                    w[2 * e] = (u & 4) ? l0 : h0;
                    w[2 * e + 1] = (u & 4) ? l1 : h1;
                }
                uint32_t* d = dk + h * KH + 4 * u;
                if (own[0] && own[1]) *reinterpret_cast<uint4*>(d) = make_uint4(w[0], w[1], w[2], w[3]);
                else if (own[0]) *reinterpret_cast<uint2*>(d) = make_uint2(w[0], w[1]);
                else if (own[1]) *reinterpret_cast<uint2*>(d + 2) = make_uint2(w[2], w[3]);
            }
        }
    }
    // V (columns [2HP, 3HP) -> vt_img[(b * HP + c) * Rp + word(r)]): warp <-> (32-row line k of clip b, 4 columns), lane l <-> row 32 k + l.
    // Lane pairs exchange their rows; the even lane stores the hi, the odd lane the lo word of the pair, so each store instruction writes
    // one 128-byte line.  Pairs never straddle a tile (m0 % 128 == 0, R even).
    const int va = max(n0, 2 * HP), vb = min(n0 + SS_BN, p.N);                 // this tile's V columns [va, vb)
    if (va < vb) {
        const int ng = (vb - va) / 4;
        for (int b = m0 / R; b * R < mend; ++b) {
            const int base = b * R, ra = max(m0, base) - base, rb = min(mend, base + R) - base;   // this tile's rows [ra, rb) of clip b
            const int k0 = ra >> 5, nl = ((rb - 1) >> 5) - k0 + 1;
            for (int t = warp; t < nl * ng; t += NW) {
                const int k = k0 + t / ng, n = va + 4 * (t % ng), r = 32 * k + lane;
                const bool own = r < R ? (r >= ra && r < rb) : rb == R;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);                     // pad rows are the split of zeros
                if (r < R && own) v = *reinterpret_cast<const float4*>(Cs + (base + r - m0) * LDS_ + n - n0);
                const float vv[4] = {v.x, v.y, v.z, v.w};
                uint32_t* d = p.vt_img + ((long long)b * HP + n - 2 * HP) * p.qkv_Rp + 32 * k + (lane & 1) * 16 + (lane >> 1);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float o = __shfl_xor_sync(0xffffffffu, vv[e], 1);
                    uint32_t hi, lo;
                    if (lane & 1) f16x3_split_pair(o, vv[e], p.qkv_sv, hi, lo); else f16x3_split_pair(vv[e], o, p.qkv_sv, hi, lo);
                    if (own) d[(long long)e * p.qkv_Rp] = (lane & 1) ? lo : hi;
                }
            }
        }
    }
}

// C = A W^T on 128 x 128 tiles, both operands fp16x3 images.  Stage / phase schedule over nk slices: the producer fills slice i into
// stage i % 4 once slice i - 4 is retired (empty parity ((i / 4) & 1) ^ 1); consumers wait full with parity (i / 4) & 1, issue slice i
// into d[i & 1], then retire slice i - 1 (wgmma_wait<1>, arrive on empty, fold); the last slice is retired with wgmma_wait<0> and needs
// no arrival (nothing is loaded after it).  tests/test_ss_pipeline_emulation.py runs this schedule on the CPU.
__global__ void __launch_bounds__(SS_THREADS, 1)
ss_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW, const SsParams p) {
    constexpr int ST = WG_STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)ST * SsCfg::STAGE);
    uint64_t* empty = full + ST;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * SS_BN, nk = p.nk;

    if (tid == 0) {
        for (int s = 0; s < ST; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WG_CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();                                 // (no-op unless launched with programmatic stream serialization)

    if (warp >= WG_CONSUMERS / 32) {
        // ------------------------------------------------------------------ TMA producer (warpgroup 2)
        setmaxnreg_dec<40>();
        if (tid == WG_CONSUMERS) {
            prefetch_tmap(&mapA); prefetch_tmap(&mapW);
            for (int i = 0; i < nk; ++i) {
                const int s = i % ST;
                mbar_wait(&empty[s], ((uint32_t)(i / ST) & 1u) ^ 1u);
                unsigned char* st = smem + (size_t)s * SsCfg::STAGE;
                mbar_expect_tx(&full[s], SsCfg::STAGE);
                tma_load_4d(st, &mapA, &full[s], i * TC_BK, m0, 0, 0);
                tma_load_4d(st + SsCfg::A_BYTES, &mapW, &full[s], i * TC_BK, n0, 0, 0);
            }
        }
    } else {
        // ------------------------------------------------------------------ consumer warpgroups (warps 0..7)
        setmaxnreg_inc<232>();
        const int wg = warp >> 2;
        const float osc = p.oscale;
        float acc[SS_BN / 2], d0[SS_BN / 2], d1[SS_BN / 2];
#pragma unroll
        for (int e = 0; e < SS_BN / 2; ++e) acc[e] = 0.f;
        // products of this warpgroup's 64 rows for slice i, small terms first: lo.hi, hi.lo, hi.hi per K step (+32 bytes inside the
        // swizzled row); the first product of the slice does not accumulate
        auto issue = [&](int i, float (&d)[SS_BN / 2]) {
            const int s = i % ST;
            mbar_wait(&full[s], (uint32_t)(i / ST) & 1u);
            const uint32_t st_addr = smem_u32(smem + (size_t)s * SsCfg::STAGE);
            const uint64_t da = make_smem_desc_sw128(st_addr + (uint32_t)wg * 64u * 128u);
            const uint64_t db = make_smem_desc_sw128(st_addr + SsCfg::A_BYTES);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const uint64_t ah = da + 2 * ks, al = ah + 4, bh = db + 2 * ks, bl = bh + 4;
                wgmma_f16(d, al, bh, ks == 0 ? 0u : 1u);
                wgmma_f16(d, ah, bl, 1u);
                wgmma_f16(d, ah, bh, 1u);
            }
            wgmma_commit();
        };
        // slice i (the older of the two groups in flight) is done: free its stage, fold it (undo the power-of-two operand scales, exact)
        auto retire = [&](int i, float (&d)[SS_BN / 2]) {
            wgmma_wait<1>(d);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[i % ST]);
#pragma unroll
            for (int e = 0; e < SS_BN / 2; ++e) acc[e] = fmaf(d[e], osc, acc[e]);
        };
        for (int i = 0; i < nk; i += 2) {
            issue(i, d0);
            if (i > 0) retire(i - 1, d1);
            if (i + 1 < nk) {
                issue(i + 1, d1);
                retire(i, d0);
            }
        }
        if ((nk - 1) & 1) {
            wgmma_wait<0>(d1);
#pragma unroll
            for (int e = 0; e < SS_BN / 2; ++e) acc[e] = fmaf(d1[e], osc, acc[e]);
        } else {
            wgmma_wait<0>(d0);
#pragma unroll
            for (int e = 0; e < SS_BN / 2; ++e) acc[e] = fmaf(d0[e], osc, acc[e]);
        }

        // ------------------------------------------------------------------ fragment -> row exchange through the (idle) operand ring
        constexpr int LDS_ = SsCfg::LDS;
        float* Cs = reinterpret_cast<float*>(smem);
        consumer_sync();                        // every warpgroup's products have read their last stage
        {
            const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < SS_BN / 8; ++j) {
                *reinterpret_cast<float2*>(Cs + r0 * LDS_ + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2*>(Cs + (r0 + 8) * LDS_ + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
        }
        consumer_sync();
        if (p.qkv_hp) {
            ss_store_qkv(p, Cs, m0, n0, warp, lane);
        } else {
            // plain store: warp w takes rows w, w + 8, ...; lane l columns [4 l, 4 l + 4) of the tile, so one store instruction writes a
            // 512-byte segment of C (or four whole 128-byte lines of the output image) instead of 16 bytes in each of 32 rows
            const int c = 4 * lane, n = n0 + c;
            float bv[4], sc2[4], sh2[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const bool in = n + e < p.N;
                bv[e] = (in && p.bias) ? __ldg(p.bias + n + e) : 0.f;
                sc2[e] = (in && p.act == GVD_ACT_RELU_AFFINE_RELU) ? __ldg(p.scale2 + n + e) : 0.f;
                sh2[e] = (in && p.act == GVD_ACT_RELU_AFFINE_RELU) ? __ldg(p.shift2 + n + e) : 0.f;
            }
            const bool vec_ok = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
            for (int r = warp; r < TC_BM; r += WG_CONSUMERS / 32) {
                const int m = m0 + r;
                if (m >= p.M) break;
                const float4 t = *reinterpret_cast<const float4*>(Cs + r * LDS_ + c);
                float v[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float x = v[e];
                    if (n + e < p.N) {
                        if (p.bias) x += bv[e];
                        if (p.act >= GVD_ACT_RELU) x = fmaxf(x, 0.f);
                        if (p.act == GVD_ACT_RELU_AFFINE_RELU) x = fmaxf(fmaf(x, sc2[e], sh2[e]), 0.f);
                    } else {
                        x = 0.f;                                // padding columns of the image are zeros
                    }
                    v[e] = x;
                }
                if (p.C) {
                    float* dst = p.C + (long long)m * p.ldc + n;
                    if (vec_ok && n + 3 < p.N) {
                        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (n + e < p.N) dst[e] = v[e];
                    }
                }
                if (p.img && n < p.ld_img) {                    // 4 columns = 2 hi words + 2 lo words of one K slice of the next GEMM
                    uint32_t h0, l0, h1, l1;
                    f16x3_split_pair(v[0], v[1], p.img_scale, h0, l0);
                    f16x3_split_pair(v[2], v[3], p.img_scale, h1, l1);
                    uint32_t* w = p.img + (long long)m * p.ld_img + f16x3_word(n);
                    *reinterpret_cast<uint2*>(w) = make_uint2(h0, h1);
                    *reinterpret_cast<uint2*>(w + 16) = make_uint2(l0, l1);
                }
            }
        }
    }
}

template <bool F16>
__global__ void __launch_bounds__(WG_THREADS, 1)
wg_gemm_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
               const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapW0,
               const __grid_constant__ CUtensorMap mapW1, const __grid_constant__ CUtensorMap mapW2, const TcParams p) {
    using Cfg = WgCfg<F16>;
    constexpr int ST = WG_STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)ST * Cfg::STAGE);
    uint64_t* empty = full + ST;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int zb = p.ksplit ? 0 : blockIdx.z / p.nh, zh = p.ksplit ? 0 : blockIdx.z % p.nh;
    const int kz = p.ksplit * (int)blockIdx.z;
    const int m0 = blockIdx.y * TC_BM;
    const int n0 = blockIdx.x * (p.nbox > 1 ? WG_UJ : TC_BN);        // first output column / first hidden unit (gate-interleaved tiles)

    if (tid == 0) {
        for (int s = 0; s < ST; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WG_CONSUMERS / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();
    pdl_wait();                                 // (no-op unless launched with programmatic stream serialization)

    if (warp == WG_CONSUMERS / 32) {
        // ------------------------------------------------------------------ TMA producer
        if (lane == 0) {
            prefetch_tmap(&mapA0); prefetch_tmap(&mapW0);
            const uint32_t w_bytes = p.nbox > 1 ? (uint32_t)p.nbox * WG_UJ * 128u : (uint32_t)Cfg::B_BYTES;
            int i = 0;
            for (int sg = 0; sg < p.nseg; ++sg) {
                const CUtensorMap* ma = sg == 0 ? &mapA0 : (sg == 1 ? &mapA1 : &mapA2);
                const CUtensorMap* mw = sg == 0 ? &mapW0 : (sg == 1 ? &mapW1 : &mapW2);
                const int nb = (p.seg[sg].k_len + TC_BK - 1) / TC_BK;
                for (int kb = 0; kb < nb; ++kb, ++i) {
                    const int s = i % ST;
                    mbar_wait(&empty[s], ((uint32_t)(i / ST) & 1u) ^ 1u);
                    unsigned char* st = smem + (size_t)s * Cfg::STAGE;
                    mbar_expect_tx(&full[s], Cfg::A_BYTES + w_bytes);
                    tma_load_4d(st, ma, &full[s], p.seg[sg].a_k0 + kz + kb * TC_BK, m0, zh * p.a_mul_h, zb * p.a_mul_b);
                    if (p.nbox <= 1) {
                        tma_load_4d(st + Cfg::B_OFF, mw, &full[s], p.seg[sg].w_k0 + kz + kb * TC_BK, n0, zh * p.w_mul_h, zb * p.w_mul_b);
                    } else {
                        // gate-interleaved rows: nbox boxes of WG_UJ rows (WG_UJ * 128 B = whole swizzle atoms)
                        for (int g = 0; g < p.nbox; ++g)
                            tma_load_4d(st + Cfg::B_OFF + g * WG_UJ * 128, mw, &full[s], p.seg[sg].w_k0 + kb * TC_BK, g * p.box_stride + n0,
                                        zh * p.w_mul_h, zb * p.w_mul_b);
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumer warpgroups (warps 0..7)
    const int wg = warp >> 2;
    float acc[TC_BN / 2];
#pragma unroll
    for (int j = 0; j < TC_BN / 2; ++j) acc[j] = 0.f;
    const float* Fz = p.Fc ? p.Fc + (long long)blockIdx.z * p.ngrp * p.M : nullptr;
    {
        int i = 0;
        for (int sg = 0; sg < p.nseg; ++sg) {
            const int nb = (p.seg[sg].k_len + TC_BK - 1) / TC_BK;
            for (int kb = 0; kb < nb; ++kb, ++i) {
                const int s = i % ST;
                mbar_wait(&full[s], (uint32_t)(i / ST) & 1u);
                const uint32_t st_addr = smem_u32(smem + (size_t)s * Cfg::STAGE);
                if constexpr (F16) {
                    // ---- raw fp32 slice -> operand image, in place: a 128-byte row of 32 floats becomes 64 B of hi halves | 64 B of lo halves.
                    // Chunk pair c2 (2 x 16 B = 8 floats) of a row -> hi chunk c2, lo chunk 4 + c2; the threads that share a row are
                    // neighbouring lanes of one warp: read, __syncwarp, write.
                    if (!p.apre) {
                        const int row = tid >> 1, m = m0 + row;
                        float sc = p.sa;
                        if (Fz) sc *= (m < p.M && kb < p.ngrp) ? __ldg(Fz + (long long)kb * p.M + m) : 0.f;
                        const uint32_t rb = st_addr + (uint32_t)row * 128u;
                        float4 w0[2], w1[2];
#pragma unroll
                        for (int u0 = 0; u0 < 2; ++u0) {
                            const int c2 = (tid & 1) * 2 + u0;
                            w0[u0] = lds128(rb + (uint32_t)(((2 * c2) ^ (row & 7)) << 4));
                            w1[u0] = lds128(rb + (uint32_t)(((2 * c2 + 1) ^ (row & 7)) << 4));
                        }
                        __syncwarp();
#pragma unroll
                        for (int u0 = 0; u0 < 2; ++u0) {
                            const int c2 = (tid & 1) * 2 + u0;
                            uint32_t h[4], l[4];
                            split_h4(w0[u0], sc, h[0], h[1], l[0], l[1]);
                            split_h4(w1[u0], sc, h[2], h[3], l[2], l[3]);
                            sts128u(rb + (uint32_t)((c2 ^ (row & 7)) << 4), h[0], h[1], h[2], h[3]);
                            sts128u(rb + (uint32_t)(((4 + c2) ^ (row & 7)) << 4), l[0], l[1], l[2], l[3]);
                        }
                    }
                    if (!p.wpre) {
                        const int wr = tid >> 2, c2 = tid & 3;
                        const uint32_t rb = st_addr + Cfg::B_OFF + (uint32_t)wr * 128u;
                        const float4 w0 = lds128(rb + (uint32_t)(((2 * c2) ^ (wr & 7)) << 4));
                        const float4 w1 = lds128(rb + (uint32_t)(((2 * c2 + 1) ^ (wr & 7)) << 4));
                        __syncwarp();
                        uint32_t h[4], l[4];
                        split_h4(w0, p.sw, h[0], h[1], l[0], l[1]);
                        split_h4(w1, p.sw, h[2], h[3], l[2], l[3]);
                        sts128u(rb + (uint32_t)((c2 ^ (wr & 7)) << 4), h[0], h[1], h[2], h[3]);
                        sts128u(rb + (uint32_t)(((4 + c2) ^ (wr & 7)) << 4), l[0], l[1], l[2], l[3]);
                    }
                    if (!p.apre || !p.wpre) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
                        consumer_sync();
                    }
                } else {
                    // ---- tf32 hi in place, lo into the twin plane (same swizzled position)
#pragma unroll
                    for (int j = 0; j < Cfg::A_BYTES / 16 / WG_CONSUMERS; ++j) {
                        const int f = tid + j * WG_CONSUMERS, row = f >> 3, m = m0 + row;
                        const uint32_t a = st_addr + (uint32_t)f * 16u;
                        float4 v = lds128(a);
                        if (Fz) {
                            const float sc = (m < p.M && kb < p.ngrp) ? __ldg(Fz + (long long)kb * p.M + m) : 0.f;
                            v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
                        }
                        float4 h, l;
                        h.x = tf32_rna(v.x); h.y = tf32_rna(v.y); h.z = tf32_rna(v.z); h.w = tf32_rna(v.w);
                        l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
                        sts128(a, h);
                        sts128(a + Cfg::A_BYTES, l);
                    }
#pragma unroll
                    for (int j = 0; j < Cfg::B_BYTES / 16 / WG_CONSUMERS; ++j) {
                        const uint32_t a = st_addr + Cfg::B_OFF + (uint32_t)(tid + j * WG_CONSUMERS) * 16u;
                        const float4 v = lds128(a);
                        float4 h, l;
                        h.x = tf32_rna(v.x); h.y = tf32_rna(v.y); h.z = tf32_rna(v.z); h.w = tf32_rna(v.w);
                        l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
                        sts128(a, h);
                        sts128(a + Cfg::B_BYTES, l);
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    consumer_sync();
                }
                // ---- products of this warpgroup's 64 rows, small terms first: lo.hi, hi.lo, hi.hi per K step (+32 bytes inside the swizzled row)
                float d[TC_BN / 2];
                const uint64_t da = make_smem_desc_sw128(st_addr + (uint32_t)wg * 64u * 128u);
                const uint64_t db = make_smem_desc_sw128(st_addr + Cfg::B_OFF);
                wgmma_fence();
                if constexpr (F16) {
#pragma unroll
                    for (int ks = 0; ks < 2; ++ks) {
                        const uint64_t ah = da + 2 * ks, al = ah + 4, bh = db + 2 * ks, bl = bh + 4;
                        wgmma_f16(d, al, bh, ks == 0 ? 0u : 1u);
                        wgmma_f16(d, ah, bl, 1u);
                        wgmma_f16(d, ah, bh, 1u);
                    }
                } else {
                    constexpr uint64_t ALO = (uint64_t)Cfg::A_BYTES >> 4, BLO = (uint64_t)Cfg::B_BYTES >> 4;
#pragma unroll
                    for (int ks = 0; ks < TC_BK / 8; ++ks) {
                        const uint64_t ah = da + 2 * ks, al = ah + ALO, bh = db + 2 * ks, bl = bh + BLO;
                        wgmma_tf32(d, al, bh, ks == 0 ? 0u : 1u);
                        wgmma_tf32(d, ah, bl, 1u);
                        wgmma_tf32(d, ah, bh, 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait0(d);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);          // stage free once this warp's MMAs have read it
#pragma unroll
                for (int e = 0; e < TC_BN / 2; ++e) {
                    if constexpr (F16) acc[e] = fmaf(d[e], p.oscale, acc[e]);      // undo the power-of-two operand scales (exact)
                    else acc[e] += d[e];
                }
            }
        }
    }

    // ---------------------------------------------------------------------- fragment -> row exchange through the (idle) operand ring
    constexpr int LDS_ = Cfg::LDS;
    float* Cs = reinterpret_cast<float*>(smem);
    consumer_sync();                            // every warpgroup's MMAs have read their last stage
    {
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < TC_BN / 8; ++j) {
            *reinterpret_cast<float2*>(Cs + r0 * LDS_ + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(Cs + (r0 + 8) * LDS_ + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
    }
    consumer_sync();
    const int q = warp & 3, row = q * 32 + lane, m = m0 + row;
    const int cbeg = (warp >> 2) * (TC_BN / 2);    // thread = (row, column half) in the modes that use all eight warps

    if (p.mode == MODE_STORE) {
        // bias / activation, whole contiguous row segments per store instruction (128-bit, coalesced)
        const float* bias = p.bias ? p.bias + zb * p.sBb : nullptr;
        float* C = p.C + zb * p.sCb + zh * p.sCh;
        const bool vec_ok = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
        for (int idx = tid; idx < TC_BM * (TC_BN / 4); idx += WG_CONSUMERS) {
            const int rr = idx / (TC_BN / 4), c4 = (idx % (TC_BN / 4)) * 4, mm = m0 + rr, n = n0 + c4;
            if (mm >= p.M || n >= p.N) continue;
            const float4 t = *reinterpret_cast<const float4*>(Cs + rr * LDS_ + c4);
            float v[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float x = v[e] * p.alpha;
                const int nn = n + e;
                if (nn < p.N) {
                    if (bias) x += __ldg(bias + nn);
                    if (p.act >= GVD_ACT_RELU) x = fmaxf(x, 0.f);
                    if (p.act == GVD_ACT_RELU_AFFINE_RELU) x = fmaxf(fmaf(x, __ldg(p.scale2 + nn), __ldg(p.shift2 + nn)), 0.f);
                }
                v[e] = x;
            }
            float* dst = C + (long long)mm * p.ldc + n;
            if (vec_ok && n + 3 < p.N) {
                *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (n + e < p.N) dst[e] = v[e];
            }
        }
    } else if (p.mode == MODE_TRANS) {
        // transposed store: this thread's row m is a column of C^T; lanes = consecutive m, so every store of a warp is one 128-byte line
        float* C = p.C + (p.ksplit ? (long long)blockIdx.z * p.sCb : zb * p.sCb + zh * p.sCh);
        if (m < p.M) {
#pragma unroll 8
            for (int j = 0; j < 32; ++j) {
                const int n = n0 + cbeg + j;
                if (n < p.N) C[(long long)n * p.ldc + m] = Cs[row * LDS_ + cbeg + j] * p.alpha;
            }
        }
    } else if (warp < 4) {
        // ---- modes in which one thread finishes a whole row of the tile alone: all 64 columns of row m
        float a64[TC_BN];
#pragma unroll
        for (int j = 0; j < TC_BN; j += 4) {
            const float4 t = *reinterpret_cast<const float4*>(Cs + row * LDS_ + j);
            a64[j] = t.x; a64[j + 1] = t.y; a64[j + 2] = t.z; a64[j + 3] = t.w;
        }
        if (p.mode == MODE_LSTM) {
            // fused LSTMCell pointwise: this thread holds i,f,g,o of WG_UJ hidden units of clip row m (AttModel.py:139,160)
            if (m < p.M) {
                const int H = p.H;
#pragma unroll
                for (int jj = 0; jj < WG_UJ; ++jj) {
                    const int j = n0 + jj;
                    if (j < H) {
                        float g4[4];
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            float v = a64[g * WG_UJ + jj];
                            const long long col = (long long)g * H + j;
                            if (p.pre) v += p.pre[(long long)(p.pre_div > 1 ? m / p.pre_div : m) * 4 * H + col];
                            if (p.bias1) v += __ldg(p.bias1 + col);
                            if (p.bias2) v += __ldg(p.bias2 + col);
                            g4[g] = v;
                        }
                        const float ig = sigmoid_acc(g4[0]), fg = sigmoid_acc(g4[1]), gg = tanhf(g4[2]), og = sigmoid_acc(g4[3]);
                        const float c = fg * p.c_prev[(long long)m * H + j] + ig * gg;
                        p.c_out[(long long)m * H + j] = c;
                        p.h_out[(long long)m * H + j] = og * tanhf(c);
                    }
                }
            }
        } else if (p.mode == MODE_PICK) {
                    // ---- fused greedy sampler (misc/model.py:590-594,615): log_softmax + top-2 + UNK rule without materialising logits
                    const int ncta = gridDim.x;
                    float mloc = -INFINITY, v1 = -INFINITY, v2 = -INFINITY;
                    int i1 = 0x7fffffff, i2 = 0x7fffffff;
                    float xs[TC_BN];
#pragma unroll
                    for (int j = 0; j < TC_BN; ++j) {
                        const int n = n0 + j;
                        const float x = n < p.N ? a64[j] + __ldg(p.bias + n) : -INFINITY;
                        xs[j] = x;
                        mloc = fmaxf(mloc, x);
                        if (x > v1 || (x == v1 && n < i1)) { v2 = v1; i2 = i1; v1 = x; i1 = n; }
                        else if (x > v2 || (x == v2 && n < i2)) { v2 = x; i2 = n; }
                    }
                    float sloc = 0.f;
#pragma unroll
                    for (int j = 0; j < TC_BN; ++j) sloc += (n0 + j < p.N) ? expf(xs[j] - mloc) : 0.f;
                    if (m < p.M) {
                        float* pp = p.pk_part + ((long long)blockIdx.x * p.M + m) * 8;
                        *reinterpret_cast<float4*>(pp) = make_float4(mloc, sloc, v1, __int_as_float(i1));
                        *reinterpret_cast<float2*>(pp + 4) = make_float2(v2, __int_as_float(i2));
                    }
                    __threadfence();
                    asm volatile("bar.sync 2, %0;" ::"n"(128) : "memory");
                    int* flag = reinterpret_cast<int*>(smem);
                    if (tid == 0) *flag = (atomicAdd(p.pk_ticket, 1) == ncta - 1) ? 1 : 0;
                    asm volatile("bar.sync 2, %0;" ::"n"(128) : "memory");
                    if (*flag) {
                        __threadfence();
                        long long* tok_s = reinterpret_cast<long long*>(smem + 64);
                        if (m < p.M) {
                            float M = -INFINITY, S = 0.f, t1 = -INFINITY, t2 = -INFINITY;
                            int j1 = 0x7fffffff, j2 = 0x7fffffff;
                            for (int cta = 0; cta < ncta; ++cta) {          // fixed merge order: independent of which CTA is last
                                const float* pp = p.pk_part + ((long long)cta * p.M + m) * 8;
                                const float4 a4 = __ldcg(reinterpret_cast<const float4*>(pp));
                                const float2 b2 = __ldcg(reinterpret_cast<const float2*>(pp + 4));
                                if (a4.x > M) { S = S * expf(M - a4.x) + a4.y; M = a4.x; }
                                else if (a4.x > -INFINITY) { S = fmaf(a4.y, expf(a4.x - M), S); }   // a tile of -inf logits adds nothing (its own sum is NaN)
                                const float cv[2] = {a4.z, b2.x};
                                const int ci[2] = {__float_as_int(a4.w), __float_as_int(b2.y)};
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    if (cv[e] > t1 || (cv[e] == t1 && ci[e] < j1)) { t2 = t1; j2 = j1; t1 = cv[e]; j1 = ci[e]; }
                                    else if (cv[e] > t2 || (cv[e] == t2 && ci[e] < j2)) { t2 = cv[e]; j2 = ci[e]; }
                                }
                            }
                            const float lse = M + logf(S);
                            const bool keep = j1 != p.pk_unk;
                            long long it = keep ? j1 : j2;
                            if ((unsigned long long)it >= (unsigned long long)p.N) it = 0;   // every logit NaN: stay inside the embedding table
                            p.pk_it[m] = it;
                            if (p.pk_seq) p.pk_seq[(long long)m * p.pk_stride] = it;
                            if (p.pk_logp) p.pk_logp[(long long)m * p.pk_stride] = (keep ? t1 : t2) - lse;
                            tok_s[m] = it;
                        }
                        asm volatile("bar.sync 2, %0;" ::"n"(128) : "memory");
                        if (p.pk_xt) {                                       // xt = ReLU(embed[token]) (model.py:79-82,605), coalesced
                            const int E4 = p.pk_E / 4;
                            for (int idx = tid; idx < p.M * E4; idx += 128) {
                                const int r = idx / E4, e4 = idx % E4;
                                float4 v = __ldg(reinterpret_cast<const float4*>(p.pk_embed + tok_s[r] * p.pk_E) + e4);
                                v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
                                reinterpret_cast<float4*>(p.pk_xt + (long long)r * p.pk_E)[e4] = v;
                            }
                        }
                        if (tid == 0) *p.pk_ticket = 0;
                    }
        } else if (p.mode == MODE_GRU) {
            // ---- fused GRU cell: thread b owns clip b and WG_UJ hidden units; a64[0..16) = W_hr h, [16..32) = W_hz h, [32..48) = W_hn h
            const GruStepParams& gp = p.gru;
            const int b = row, u0 = n0, d = blockIdx.z, G = gp.G;
            if (b < gp.B) {
                // gate math: r, z, n order, b_hn inside the r product (torch.nn.GRU)
                const int t = d ? (gp.T - 1 - gp.step) : gp.step;
                const float* gir = gp.gi + ((size_t)b * gp.T + t) * (6 * G) + (size_t)d * 3 * G + u0;
                const float* bh = gp.bhh + (size_t)d * 3 * G + u0;
                const size_t so = ((size_t)d * gp.B + b) * G + u0;
                float hv[WG_UJ];
#pragma unroll
                for (int j = 0; j < WG_UJ; j += 4) {
                    const float4 gr = *reinterpret_cast<const float4*>(gir + j), gz = *reinterpret_cast<const float4*>(gir + G + j);
                    const float4 gn = *reinterpret_cast<const float4*>(gir + 2 * G + j), hp = *reinterpret_cast<const float4*>(gp.h_prev + so + j);
                    const float4 br = __ldg(reinterpret_cast<const float4*>(bh + j)), bz = __ldg(reinterpret_cast<const float4*>(bh + G + j));
                    const float4 bn = __ldg(reinterpret_cast<const float4*>(bh + 2 * G + j));
                    const float grr[4] = {gr.x, gr.y, gr.z, gr.w}, gzz[4] = {gz.x, gz.y, gz.z, gz.w}, gnn[4] = {gn.x, gn.y, gn.z, gn.w};
                    const float hpp[4] = {hp.x, hp.y, hp.z, hp.w}, brr[4] = {br.x, br.y, br.z, br.w}, bzz[4] = {bz.x, bz.y, bz.z, bz.w};
                    const float bnn[4] = {bn.x, bn.y, bn.z, bn.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float rg = sigmoid_acc(grr[e] + a64[j + e] + brr[e]);
                        const float zg = sigmoid_acc(gzz[e] + a64[WG_UJ + j + e] + bzz[e]);
                        const float ng = tanhf(gnn[e] + rg * (a64[2 * WG_UJ + j + e] + bnn[e]));
                        hv[j + e] = (1.f - zg) * ng + zg * hpp[e];
                    }
                }
                bool keep = true;
                if (gp.sample_idx) {
                    const long long lo = gp.sample_idx[2 * b], hi = gp.sample_idx[2 * b + 1];
                    keep = !(t < lo || t >= hi);
                }
                float* hn = gp.h_new + so;
                float* o = gp.out + ((size_t)b * gp.T + t) * (2 * G) + (size_t)d * G + u0;
                // u0 is a multiple of 16: this thread's units are one half of a K slice of the next step's A operand (8 hi words, 8 lo words)
                uint32_t* img = reinterpret_cast<uint32_t*>(gp.h_img_new) + ((size_t)d * gp.B + b) * G + f16x3_word(u0);
#pragma unroll
                for (int j = 0; j < WG_UJ; j += 4) {
                    *reinterpret_cast<float4*>(hn + j) = make_float4(hv[j], hv[j + 1], hv[j + 2], hv[j + 3]);
                    *reinterpret_cast<float4*>(o + j) = keep ? make_float4(hv[j], hv[j + 1], hv[j + 2], hv[j + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                uint32_t hi_w[WG_UJ / 2], lo_w[WG_UJ / 2];
#pragma unroll
                for (int pr = 0; pr < WG_UJ / 2; ++pr) f16x3_split_pair(hv[2 * pr], hv[2 * pr + 1], gp.sa, hi_w[pr], lo_w[pr]);
#pragma unroll
                for (int j = 0; j < WG_UJ / 2; j += 4) {
                    *reinterpret_cast<uint4*>(img + j) = make_uint4(hi_w[j], hi_w[j + 1], hi_w[j + 2], hi_w[j + 3]);
                    *reinterpret_cast<uint4*>(img + 16 + j) = make_uint4(lo_w[j], lo_w[j + 1], lo_w[j + 2], lo_w[j + 3]);
                }
            }
        }
    }
}


// fp32 [N, K] (row pitch ldw) -> the W-operand image of the fp16x3 kernel: per row and 32-wide K slice 16 words of hi pairs then 16 words
// of lo pairs (k = 2p, 2p + 1 in word p), values scaled by GVD_F16_SW; K padded with zeros to a multiple of 32 (row pitch Kp words)
__global__ void pack_f16x3_kernel(const float* __restrict__ W, long long ldw, int N, int K, float sw, uint32_t* __restrict__ out, long long Kp) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;         // (n, slice, pair)
    const long long per_row = Kp / 2;
    if (idx >= (long long)N * per_row) return;
    const long long n = idx / per_row;
    const int r = (int)(idx % per_row), kb = r / 16, pr = r % 16, k = kb * 32 + 2 * pr;
    const float x0 = k < K ? W[n * ldw + k] * sw : 0.f, x1 = k + 1 < K ? W[n * ldw + k + 1] * sw : 0.f;
    const float a0 = tf32_rna(x0), a1 = tf32_rna(x1);
    out[n * Kp + kb * 32 + pr] = f16x3_pack_pair(a0, a1);
    out[n * Kp + kb * 32 + 16 + pr] = f16x3_pack_pair(x0 - a0, x1 - a1);
}

// 128 x 64 tiles
int launch_wg(const CUtensorMap* mA, const CUtensorMap* mW, const TcParams& p, dim3 grid, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        GVD_CHECK_CUDA(cudaFuncSetAttribute(wg_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WgCfg<false>::SMEM));
        GVD_CHECK_CUDA(cudaFuncSetAttribute(wg_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WgCfg<true>::SMEM));
        attr_set = true;
    }
    GVD_REQUIRE(p.f16 || (!p.apre && !p.wpre), "tcgemm: operand images belong to the fp16x3 products");
    if (p.f16)
        GVD_CHECK_CUDA(gvd_launch(wg_gemm_kernel<true>, grid, dim3(WG_THREADS), WgCfg<true>::SMEM, st, mA[0], mA[1], mA[2], mW[0], mW[1], mW[2], p));
    else
        GVD_CHECK_CUDA(gvd_launch(wg_gemm_kernel<false>, grid, dim3(WG_THREADS), WgCfg<false>::SMEM, st, mA[0], mA[1], mA[2], mW[0], mW[1], mW[2], p));
    GVD_CHECK_LAUNCH();
    return 0;
}
// precision of the products launched by this thread: fp16x3 inside a gvd_f16_scope, else 3xTF32
void set_precision(TcParams& p) {
    if (gvd_gemm_f16()) { p.f16 = 1; p.sa = GVD_F16_SA; p.sw = GVD_F16_SW; p.oscale = 1.f / (GVD_F16_SA * GVD_F16_SW); }   // |activation| <= 16376, |weight| <= 255 after scaling
    else { p.f16 = 0; p.sa = p.sw = 1.f; p.oscale = 1.f; }
}

// softmax numerator of one score row in place: C = exp((s - max) * c), F[g][m] = 1 / sum for every 32-column group g of the row
__global__ void attn_softmax_rows_kernel(float* __restrict__ C, long long ldc, long long sCb, long long sCh, int nh, int M, int N, float c2,
                                         float* __restrict__ F, int ngrp) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = blockIdx.x * (blockDim.x >> 5) + warp, z = blockIdx.y;
    if (m >= M) return;
    float* r = C + (z / nh) * sCb + (z % nh) * sCh + (long long)m * ldc;
    float mx = -INFINITY;
    for (int n = lane; n < N; n += 32) mx = fmaxf(mx, r[n]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int n = lane; n < N; n += 32) {
        const float e = ex2_approx((r[n] - mx) * c2);
        r[n] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
    float* Fz = F + (long long)z * ngrp * M;
    for (int g = lane; g < ngrp; g += 32) Fz[(long long)g * M + m] = inv;
}

}  // namespace


// Batched product without bias / activation for the self-attention scores.
//   W_lo == nullptr : g.W is plain fp32 (split inside the kernel);  else g.W / W_lo are its tf32 hi / lo planes (same strides): two K segments
//   F    != nullptr : C = exp((s - max_row) * smx_scale) and F[batch][ceil(N/32)][M] = 1 / sum_row (the P.V product multiplies it in)
// f16: g.W is the fp16x3 image of the streamed operand (K rounded up to 32 words per (row, head)), scale GVD_ATT_SK; the A operand is scaled
// by GVD_ATT_SQ inside the kernel; both are undone when the slice results are folded
static int launch_scores(const GemmArgs& g, const float* W_lo, float* F, float smx_scale, int batch, cudaStream_t stream, int f16) {
    GVD_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0 && g.nh >= 1 && batch % g.nh == 0, "score gemm: bad problem");
    GVD_REQUIRE(!g.bias && g.act == GVD_ACT_NONE, "score gemm: no bias / activation epilogue");
    GVD_REQUIRE(g.K % 4 == 0 && g.lda % 4 == 0 && g.ldw % 4 == 0, "score gemm: K/lda/ldw must be multiples of 4");
    const int nb = batch / g.nh;
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    const int Kw = f16 ? (g.K + 31) / 32 * 32 : g.K;          // the image holds whole 32-wide slices
    GVD_TRY(make_map(&mA[0], g.A, g.K, g.M, g.lda, g.nh, g.sAh, nb, g.sAb, TC_BM, &p.a_mul_h, &p.a_mul_b));
    GVD_TRY(make_map(&mW[0], g.W, Kw, g.N, g.ldw, g.nh, g.sWh, nb, g.sWb, TC_BN, &p.w_mul_h, &p.w_mul_b));
    GVD_TRY(make_map(&mW[1], (W_lo && !f16) ? W_lo : g.W, Kw, g.N, g.ldw, g.nh, g.sWh, nb, g.sWb, TC_BN, &p.w_mul_h, &p.w_mul_b));
    mA[1] = mA[2] = mA[0];
    mW[2] = mW[0];
    p.nseg = (W_lo && !f16) ? 2 : 1;
    p.seg[0] = p.seg[1] = TcSeg{g.K, 0, 0};
    p.M = g.M; p.N = g.N; p.nh = g.nh;
    p.C = g.C; p.ldc = g.ldc; p.sCb = g.sCb; p.sCh = g.sCh; p.alpha = F ? 1.f : g.alpha;
    p.mode = MODE_STORE;
    p.sa = p.sw = p.oscale = 1.f;
    if (f16) { p.f16 = 1; p.wpre = 1; p.sa = GVD_ATT_SQ; p.oscale = 1.f / (GVD_ATT_SQ * GVD_ATT_SK); }
    GVD_TRY(launch_wg(mA, mW, p, dim3(gvd_cdiv(g.N, TC_BN), gvd_cdiv(g.M, TC_BM), batch), stream));
    if (F) {
        attn_softmax_rows_kernel<<<dim3(gvd_cdiv(g.M, 4), batch), 128, 0, stream>>>(g.C, g.ldc, g.sCb, g.sCh, g.nh, g.M, g.N, smx_scale * 1.4426950408889634f,
                                                                                   F, gvd_cdiv(g.N, 32));
        GVD_CHECK_LAUNCH();
    }
    return 0;
}
int gvd_gemm_nt_astat(const GemmArgs& g, int batch, cudaStream_t stream) { return launch_scores(g, nullptr, nullptr, 0.f, batch, stream, 0); }
int gvd_attn_scores_tc(const GemmArgs& g, const float* W_lo, float* F, float smx_scale, int batch, cudaStream_t stream, int f16) {
    GVD_REQUIRE(!F || W_lo || f16, "attn scores: the softmax epilogue is built for pre-split operands");
    return launch_scores(g, W_lo, F, smx_scale, batch, stream, f16);
}
// O[z] = (F (.) A[z]) W[z]^T with W given as tf32 hi / lo planes or (f16) as its fp16x3 image, N <= 192, any K;  F [batch][ceil(K/32)][M] or null
int gvd_attn_pv_tc(const GemmArgs& g, const float* W_lo, const float* F, int batch, cudaStream_t stream, int f16) {
    GVD_REQUIRE(g.M > 0 && g.N > 0 && g.N <= 192 && g.K > 0 && g.nh >= 1 && batch % g.nh == 0 && (W_lo || f16), "attn pv: needs N <= 192 and pre-split W");
    GVD_REQUIRE(!g.bias && g.act == GVD_ACT_NONE, "attn pv: no bias / activation epilogue");
    GVD_REQUIRE(g.K % 4 == 0 && g.lda % 4 == 0 && g.ldw % 4 == 0, "attn pv: K/lda/ldw must be multiples of 4");
    const int nb = batch / g.nh;
    const int bn = ((g.N + 15) / 16) * 16;
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    GVD_TRY(make_map(&mA[0], g.A, g.K, g.M, g.lda, g.nh, g.sAh, nb, g.sAb, TC_BM, &p.a_mul_h, &p.a_mul_b));
    const int Kw = f16 ? (g.K + 31) / 32 * 32 : g.K;          // the image holds whole 32-wide slices
    GVD_TRY(make_map(&mW[0], g.W, Kw, g.N, g.ldw, g.nh, g.sWh, nb, g.sWb, TC_BN, &p.w_mul_h, &p.w_mul_b));
    GVD_TRY(make_map(&mW[1], f16 ? g.W : W_lo, Kw, g.N, g.ldw, g.nh, g.sWh, nb, g.sWb, TC_BN, &p.w_mul_h, &p.w_mul_b));
    mA[1] = mA[2] = mA[0];
    mW[2] = mW[0];
    p.nseg = f16 ? 1 : 2;
    p.seg[0] = p.seg[1] = TcSeg{g.K, 0, 0};
    p.M = g.M; p.N = g.N; p.nh = g.nh;
    p.C = g.C; p.ldc = g.ldc; p.sCb = g.sCb; p.sCh = g.sCh; p.alpha = g.alpha;
    p.Fc = F; p.ngrp = gvd_cdiv(g.K, 32);
    p.mode = MODE_STORE;
    p.sa = p.sw = p.oscale = 1.f;
    if (f16) { p.f16 = 1; p.wpre = 1; p.sa = GVD_ATT_SP; p.oscale = 1.f / (GVD_ATT_SP * GVD_ATT_SV); }
    return launch_wg(mA, mW, p, dim3(gvd_cdiv(bn, TC_BN), gvd_cdiv(g.M, TC_BM), batch), stream);
}

int gvd_pack_f16x3(const float* W, long long ldw, int N, int K, float* out, long long Kp, cudaStream_t st, float scale) {
    GVD_REQUIRE(W && out && Kp % 32 == 0 && Kp >= K, "pack_f16x3: bad arguments");
    const long long n = (long long)N * (Kp / 2);
    pack_f16x3_kernel<<<(unsigned)gvd_cdiv(n, 256), 256, 0, st>>>(W, ldw, N, K, scale, reinterpret_cast<uint32_t*>(out), Kp);
    GVD_CHECK_LAUNCH();
    return 0;
}

// part[s][b][n] = sum_{k in split s} Wp[n][k] Xp[b][k] with both operands in the fp16x3 image (gvd_pack_f16x3 / the packed activation
// buffers): Wp [Nw, Kp] words, Xp [B, ldx] words; Kp, ldx multiples of 32.  The weight rows are the M side, the batch the N side, the
// partial of split s is stored transposed (batch-major) so that the reductions of gvd_skinny.cu read along the contiguous dimension.
int gvd_skinny_f16(const float* Wp, long long ldw, int Nw, const float* Xp, long long ldx, int B, int Ktot, int S, float* part, int ldp,
                   cudaStream_t st) {
    GVD_REQUIRE(Wp && Xp && part && B >= 1 && B <= 128 && S >= 1 && Ktot % (32 * S) == 0 && ldw % 32 == 0 && ldx % 32 == 0 && ldp >= Nw,
                "skinny_f16: bad arguments (Ktot=%d S=%d)", Ktot, S);
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    GVD_TRY(make_map(&mA[0], Wp, Ktot, Nw, ldw, 1, 0, 1, 0, TC_BM, &p.a_mul_h, &p.a_mul_b));
    GVD_TRY(make_map(&mW[0], Xp, Ktot, B, ldx, 1, 0, 1, 0, TC_BN, &p.w_mul_h, &p.w_mul_b));
    mA[1] = mA[2] = mA[0];
    mW[1] = mW[2] = mW[0];
    p.nseg = 1;
    p.seg[0] = TcSeg{Ktot / S, 0, 0};
    p.ksplit = Ktot / S;
    p.M = Nw; p.N = B; p.nh = 1;
    p.C = part; p.ldc = ldp; p.sCb = (long long)B * ldp; p.alpha = 1.f;
    p.mode = MODE_TRANS;
    p.f16 = 1; p.apre = p.wpre = 1; p.sa = p.sw = 1.f; p.oscale = 1.f / (GVD_F16_SA * GVD_F16_SW);
    return launch_wg(mA, mW, p, dim3(gvd_cdiv(B, TC_BN), gvd_cdiv(Nw, TC_BM), S), st);
}

// One bidirectional GRU layer on the tensor cores: T launches of the GRU-cell mode (model.py:150-154): gh = W_hh h(t-1) with the gate math
// fused.  The batch (<= 128 clips) is the M side: thread b of the epilogue owns clip b; the N side is a gate-interleaved tile of W_hh: rows
// [r | z | n] of 16 hidden units (three TMA boxes of 16 rows), so every thread ends up with the r, z and n pre-activations of 16 units of
// ITS clip and finishes the cell alone.  Both operands arrive pre-split (h image written by the previous step, W_hh image packed once).
// hstate / h_img: [2 parity][2 dir][B][G] fp32 / fp16x3 words, zero-initialised here.  Whh_img: [2][3G][G] words.  B <= 128, G % 32 == 0.
int gvd_gru_layer_f16(const float* gi, const float* Whh_img, const float* bhh, float* hstate, float* h_img, float* out, const long long* sample_idx, int B,
                      int T, int G, cudaStream_t st) {
    GVD_REQUIRE(gi && Whh_img && bhh && hstate && h_img && out && B >= 1 && B <= 128 && G % 32 == 0, "gru_layer_f16: bad arguments");
    const size_t half = (size_t)2 * B * G;
    GVD_CHECK_CUDA(cudaMemsetAsync(hstate, 0, 2 * half * sizeof(float), st));
    GVD_CHECK_CUDA(cudaMemsetAsync(h_img, 0, 2 * half * sizeof(float), st));
    CUtensorMap mH[2][3], mW[3];
    TcParams p{};
    for (int par = 0; par < 2; ++par) {
        GVD_TRY(make_map(&mH[par][0], h_img + par * half, G, B, G, 1, 0, 2, (long long)B * G, TC_BM, &p.a_mul_h, &p.a_mul_b));
        mH[par][1] = mH[par][2] = mH[par][0];
    }
    GVD_TRY(make_map(&mW[0], Whh_img, G, 3ll * G, G, 1, 0, 2, 3ll * G * G, WG_UJ, &p.w_mul_h, &p.w_mul_b));
    mW[1] = mW[2] = mW[0];
    p.nseg = 1;
    p.seg[0] = TcSeg{G, 0, 0};
    p.M = B; p.N = 3 * WG_UJ; p.nh = 1;
    p.mode = MODE_GRU; p.nbox = 3; p.box_stride = G;
    p.f16 = 1; p.apre = p.wpre = 1; p.sa = p.sw = 1.f; p.oscale = 1.f / (GVD_F16_SA * GVD_F16_SW);
    for (int s = 0; s < T; ++s) {
        const size_t cur = (size_t)(s & 1) * half, nxt = (size_t)((s + 1) & 1) * half;
        p.gru = GruStepParams{gi, bhh, hstate + cur, hstate + nxt, h_img + nxt, out, sample_idx, B, T, G, s, GVD_F16_SA};
        GVD_TRY(launch_wg(mH[s & 1], mW, p, dim3(G / WG_UJ, 1, 2), st));
    }
    return 0;
}

// C[M, N] = act(A W^T + bias) with both operands in the fp16x3 image: Ap [M, lda] words (scale GVD_F16_SA), Wp [N, ldw] words (scale
// GVD_F16_SW), lda / ldw multiples of 32 covering K rounded up to 32 (zero padded)
int gvd_gemm_f16ss(const float* Ap, long long lda, const float* Wp, long long ldw, const float* bias, const float* scale2, const float* shift2, int act,
                   float* C, long long ldc, int M, int N, int K, cudaStream_t st, float* img, long long ld_img, const GvdQkvImages* qkv) {
    GVD_REQUIRE(Ap && Wp && (C || img) && M > 0 && N > 0 && K > 0 && lda % 32 == 0 && ldw % 32 == 0, "gemm_f16ss: bad arguments");
    if (qkv) {
        GVD_REQUIRE(C && !img && !bias && act == GVD_ACT_NONE && qkv->k_img && qkv->vt_img, "gemm_f16ss(qkv): plain projection, Q to C, K / V to their images");
        GVD_REQUIRE(N == 3 * qkv->HP && qkv->HP == qkv->nh * qkv->HS && qkv->HS % 4 == 0 && qkv->KH % 32 == 0 && qkv->KH >= qkv->HS && qkv->KH - qkv->HS < 32,
                    "gemm_f16ss(qkv): head layout");
        GVD_REQUIRE(qkv->R % 2 == 0 && M % qkv->R == 0 && qkv->Rp % 32 == 0 && qkv->Rp >= qkv->R && qkv->Rp - qkv->R < 32 && ldc % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(C) & 15) == 0, "gemm_f16ss(qkv): row layout");
    }
    GVD_REQUIRE(!img || (ld_img % 32 == 0 && ld_img >= N), "gemm_f16ss: the output image needs a 32-multiple pitch >= N");
    const int Kp = (K + 31) / 32 * 32;
    GVD_REQUIRE(lda >= Kp && ldw >= Kp, "gemm_f16ss: operand images must cover K rounded up to 32");
    CUtensorMap mA, mW;
    int unused;
    GVD_TRY(make_map(&mA, Ap, Kp, M, lda, 1, 0, 1, 0, TC_BM, &unused, &unused));
    GVD_TRY(make_map(&mW, Wp, Kp, N, ldw, 1, 0, 1, 0, SS_BN, &unused, &unused));
    SsParams s{};
    s.C = C; s.ldc = ldc; s.M = M; s.N = N;
    s.nk = Kp / TC_BK; s.oscale = 1.f / (GVD_F16_SA * GVD_F16_SW);
    s.bias = bias; s.scale2 = scale2; s.shift2 = shift2; s.act = act;
    s.img = reinterpret_cast<uint32_t*>(img); s.ld_img = ld_img; s.img_scale = GVD_F16_SA;
    if (qkv) {
        s.qkv_hp = qkv->HP; s.qkv_hs = qkv->HS; s.qkv_kh = qkv->KH; s.qkv_nh = qkv->nh; s.qkv_R = qkv->R; s.qkv_Rp = qkv->Rp;
        s.k_img = reinterpret_cast<uint32_t*>(qkv->k_img); s.vt_img = reinterpret_cast<uint32_t*>(qkv->vt_img);
        s.qkv_sk = qkv->sk; s.qkv_sv = qkv->sv;
    }
    static bool attr_set = false;
    if (!attr_set) {
        GVD_CHECK_CUDA(cudaFuncSetAttribute(ss_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SsCfg::SMEM));
        attr_set = true;
    }
    const dim3 grid(gvd_cdiv(N, SS_BN), gvd_cdiv(M, TC_BM), 1);
    GVD_CHECK_CUDA(gvd_launch(ss_gemm_kernel, grid, dim3(SS_THREADS), SsCfg::SMEM, st, mA, mW, s));
    GVD_CHECK_LAUNCH();
    return 0;
}

// C = act(alpha * A W^T + bias) with the GemmArgs contract of gvd_gemm.cuh (batched over (b,h))
int gvd_gemm_nt_tc(const GemmArgs& g, int batch, cudaStream_t stream) {
    GVD_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0 && g.nh >= 1 && batch % g.nh == 0, "tcgemm: bad problem");
    GVD_REQUIRE(g.K % 4 == 0 && g.lda % 4 == 0 && g.ldw % 4 == 0, "tcgemm: K/lda/ldw must be multiples of 4");
    GVD_REQUIRE(!g.trans_c || (!g.bias && g.act == GVD_ACT_NONE), "tcgemm: the transposed store takes no bias / activation");
    const int nb = batch / g.nh;
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    set_precision(p);
    if (g.trans_c) std::swap(p.sa, p.sw);   // operand-swapped product: the M side holds the weights, so it takes the weight scale
    GVD_TRY(make_map(&mA[0], g.A, g.K, g.M, g.lda, g.nh, g.sAh, nb, g.sAb, TC_BM, &p.a_mul_h, &p.a_mul_b));
    {
        // fp16x3: a registered constant weight has a pre-split copy (hi | lo halves per 32-wide K slice, gvd_pack_f16x3): stream that one and
        // skip the in-kernel W conversion
        const float* Wp = nullptr;
        long long ldp = 0;
        if (p.f16 && batch == 1 && g.nh == 1 && gvd_packed_lookup(g.W, g.ldw, g.N, g.K, &Wp, &ldp)) {
            GVD_TRY(make_map(&mW[0], Wp, (g.K + 31) / 32 * 32, g.N, ldp, 1, 0, 1, 0, TC_BN, &p.w_mul_h, &p.w_mul_b));
            p.wpre = 1;
        } else {
            GVD_TRY(make_map(&mW[0], g.W, g.K, g.N, g.ldw, g.nh, g.sWh, nb, g.sWb, TC_BN, &p.w_mul_h, &p.w_mul_b));
        }
    }
    mA[1] = mA[2] = mA[0];
    mW[1] = mW[2] = mW[0];
    p.nseg = 1;
    p.seg[0] = TcSeg{g.K, 0, 0};
    p.M = g.M; p.N = g.N; p.nh = g.nh;
    p.C = g.C; p.ldc = g.ldc; p.sCb = g.sCb; p.sCh = g.sCh;
    p.bias = g.bias; p.sBb = g.sBb; p.scale2 = g.scale2; p.shift2 = g.shift2; p.act = g.act; p.alpha = g.alpha;
    p.mode = g.trans_c ? MODE_TRANS : MODE_STORE;
    return launch_wg(mA, mW, p, dim3(gvd_cdiv(g.N, TC_BN), gvd_cdiv(g.M, TC_BM), batch), stream);
}

// Vocabulary head + greedy pick fused: logits = h W^T + b are reduced on the fly, nothing [B,V]-sized is stored.
int gvd_logit_pick_tc(const float* h, long long ldh, const float* W, long long ldw, const float* bias, int B, int V, int K, int unk_idx,
                      float* part, int* ticket, long long* it_out, long long* seq_out, float* logp_out, long long out_stride,
                      const float* embed, float* xt, int E, cudaStream_t stream) {
    GVD_REQUIRE(B >= 1 && B <= TC_BM, "logit_pick: at most %d rows per launch (got %d)", TC_BM, B);
    GVD_REQUIRE(bias && part && ticket && it_out, "logit_pick: null argument");
    GVD_REQUIRE(!xt || (embed && E % 4 == 0), "logit_pick: the embedding row is copied in 16-byte pieces (E=%d)", E);
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    set_precision(p);
    GVD_TRY(make_map(&mA[0], h, K, B, ldh, 1, 0, 1, 0, TC_BM, &p.a_mul_h, &p.a_mul_b));
    GVD_TRY(make_map(&mW[0], W, K, V, ldw, 1, 0, 1, 0, TC_BN, &p.w_mul_h, &p.w_mul_b));
    mA[1] = mA[2] = mA[0];
    mW[1] = mW[2] = mW[0];
    p.nseg = 1;
    p.seg[0] = TcSeg{K, 0, 0};
    p.M = B; p.N = V; p.nh = 1; p.mode = MODE_PICK; p.bias = bias; p.alpha = 1.f;
    p.pk_part = part; p.pk_ticket = ticket; p.pk_it = it_out; p.pk_seq = seq_out; p.pk_logp = logp_out; p.pk_stride = out_stride;
    p.pk_unk = unk_idx; p.pk_embed = embed; p.pk_xt = xt; p.pk_E = E;
    return launch_wg(mA, mW, p, dim3(gvd_cdiv(V, TC_BN), 1, 1), stream);
}

// LSTMCell step on the tensor cores: same contract as gvd_lstm_step, but segment inputs must be dense
// activation matrices (the caller materialises xt = ReLU(embed[token]) once per step).
int gvd_lstm_step_tc(const LstmArgs& a, cudaStream_t stream) {
    GVD_REQUIRE(a.nseg >= 1 && a.nseg <= 3 && a.H % 8 == 0, "lstm_tc: needs 1..3 segments and H %% 8 == 0");
    CUtensorMap mA[3], mW[3];
    TcParams p{};
    set_precision(p);
    p.nseg = a.nseg;
    for (int s = 0; s < 3; ++s) {
        const LstmSeg& sg = a.seg[s < a.nseg ? s : 0];
        GVD_REQUIRE(!sg.gather && !sg.relu, "lstm_tc: gather/ReLU segments must be materialised by the caller");
        GVD_TRY(make_map(&mA[s], sg.x, sg.K, a.B, sg.ldx, 1, 0, 1, 0, TC_BM, &p.a_mul_h, &p.a_mul_b));
        GVD_TRY(make_map(&mW[s], sg.w, sg.K, 4ll * a.H, sg.ldw, 1, 0, 1, 0, WG_UJ, &p.w_mul_h, &p.w_mul_b));
        if (s < a.nseg) p.seg[s] = TcSeg{sg.K, 0, 0};
    }
    p.M = a.B; p.N = 4 * a.H; p.nh = 1; p.mode = MODE_LSTM; p.H = a.H; p.nbox = 4; p.box_stride = a.H;
    p.pre = a.pre; p.pre_div = a.pre_div; p.bias1 = a.bias1; p.bias2 = a.bias2; p.c_prev = a.c_prev; p.h_out = a.h_out; p.c_out = a.c_out;
    p.alpha = 1.f;
    return launch_wg(mA, mW, p, dim3(gvd_cdiv(a.H, WG_UJ), gvd_cdiv(a.B, TC_BM), 1), stream);
}
