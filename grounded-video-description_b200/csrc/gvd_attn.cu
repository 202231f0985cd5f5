// gvd: fused self-attention of the region encoder on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
//   O[b, r, h] = softmax(Q_h K_h^T * scale) V_h      per (clip b, head h), flash-style: the scores never leave the SM
//
// One CTA per (128 query rows, head, clip); the grid runs in that order, so the query tiles of one (clip, head) run together and share its
// key / value images through L2.  384 threads:
//   warpgroup 2    : TMA producer (one thread, setmaxnreg 40).  Per 32-key block: the key image slices (32 rows x 128 B each, one per 32-wide
//                    slice of the head dimension) and the V^T image block (NV rows x 128 B) into a ring of 2 stages.
//   warpgroups 0-1 : consumers (setmaxnreg 232), 64 query rows each.  The Q tile is loaded once and split into its fp16x3 image in shared
//                    memory.  Per key block: S = Q K^T as m64n32k16 products (lo.hi + hi.lo + hi.hi per k16 step, one fold into fp32
//                    registers per head-dimension slice), an online softmax in fp32 registers, P -> fp16 hi / lo register fragments (the
//                    accumulator fragment of S is the A fragment of the next product), then P.V as two m64n(NV/2)k16 register-A products
//                    per k16 step and one fold per block: O = O * alpha + d * oscale.  At the end O / row sum is stored.
// Numerics follow the score / P.V pair of gvd_wgmma.cu (operand scales, hi / lo split, product order, one fold per 32-wide slice), except that
// P is normalised once at the end instead of before its split.
#include <cuda.h>

#include "gvd_wgmma.cuh"

namespace {

constexpr int ATT_BM = 128;               // query rows per CTA
constexpr int ATT_BK = 32;                // keys per block
constexpr int ATT_QS = 6;                 // head-dimension slices of 32 (head size <= 192)
constexpr int ATT_THREADS = 384;
constexpr int ATT_Q_BYTES = ATT_QS * ATT_BM * 128;
constexpr int ATT_K_BYTES = ATT_QS * ATT_BK * 128;

template <int NV> struct AttCfg {
    static constexpr int V_BYTES = NV * 128;
    static constexpr int STAGE = ATT_K_BYTES + V_BYTES;
    static constexpr size_t SMEM = (size_t)ATT_Q_BYTES + 2 * STAGE + 1024 /*align*/ + 64;
    static_assert(V_BYTES % 1024 == 0 && SMEM <= 232448, "shared-memory budget (227 KB per CTA)");
};

struct AttnParams {
    const float* q; long long ldq;        // Q of (b, r, h): q + (b * R + r) * ldq + h * hs
    float* out; long long ldo;            // fp32 O (columns [h * hs, h * hs + hs) of row b * R + r), or null
    uint32_t* img; long long img_ld;      // else the fp16x3 operand image of O (scale GVD_F16_SA); columns [nh * hs, img_ld) zeroed
    int R, nh, hs, ns;                    // ns: 32-wide slices of the key image per head
    int k_mul_h, k_mul_b, v_mul_b;        // tensor-map coordinates of axes of extent 1 are 0
    float c2;                             // softmax scale * log2 e
};

__device__ __forceinline__ void sts64u(uint32_t addr, uint32_t a, uint32_t b) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}

template <int NV>
__global__ void __launch_bounds__(ATT_THREADS, 1)
self_attn_fused_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapV, const AttnParams p) {
    using Cfg = AttCfg<NV>;
    constexpr int NH = NV / 2;                                  // columns of one P.V half
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* ring = smem + ATT_Q_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + 2 * Cfg::STAGE);
    uint64_t* empty = full + 2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int nkb = (p.R + ATT_BK - 1) / ATT_BK;
    if (tid == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);                            // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp >= 8) {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (tid == 256) {
            prefetch_tmap(&mapK); prefetch_tmap(&mapV);
            for (int kb = 0; kb < nkb; ++kb) {
                const int s = kb & 1;
                mbar_wait(&empty[s], ((uint32_t)(kb >> 1) & 1u) ^ 1u);
                unsigned char* st = ring + s * Cfg::STAGE;
                mbar_expect_tx(&full[s], (uint32_t)(p.ns * ATT_BK * 128 + Cfg::V_BYTES));
                for (int sl = 0; sl < p.ns; ++sl)
                    tma_load_4d(st + sl * ATT_BK * 128, &mapK, &full[s], sl * 32, kb * ATT_BK, h * p.k_mul_h, b * p.k_mul_b);
                tma_load_4d(st + ATT_K_BYTES, &mapV, &full[s], kb * ATT_BK, h * p.hs, 0, b * p.v_mul_b);
            }
        }
        return;
    }

    // ---------------------------------------------------------------------- consumer warpgroups (warps 0..7)
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, c = lane & 3;
    {
        // Q tile -> fp16x3 image (scale GVD_ATT_SQ): slice sl of row i at smem + sl * 16 KB + i * 128 B, 16-byte chunks swizzled by i % 8;
        // columns past hs and rows past R are zeros
        const int m0 = qt * ATT_BM;
        for (int t = tid; t < ATT_BM * ATT_QS * 8; t += 256) {
            const int row = t / (ATT_QS * 8), g = t % (ATT_QS * 8), sl = g >> 3, c4 = (g & 7) * 4, col = sl * 32 + c4, r = m0 + row;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < p.R && col < p.hs) v = *reinterpret_cast<const float4*>(p.q + ((long long)b * p.R + r) * p.ldq + (long long)h * p.hs + col);
            uint32_t h01, l01, h23, l23;
            f16x3_split_pair(v.x, v.y, GVD_ATT_SQ, h01, l01);
            f16x3_split_pair(v.z, v.w, GVD_ATT_SQ, h23, l23);
            const uint32_t rb = smem_u32(smem + sl * ATT_BM * 128 + row * 128), off = (uint32_t)(c4 & 4) * 2;
            sts64u(rb + (uint32_t)(((c4 >> 3) ^ (row & 7)) << 4) + off, h01, h23);
            sts64u(rb + (uint32_t)(((4 + (c4 >> 3)) ^ (row & 7)) << 4) + off, l01, l23);
        }
        // the products always run over 6 slices: key slices past the image's ns (never loaded) are zeros in both stages
        for (int t = tid; t < 2 * (ATT_QS - p.ns) * ATT_BK * 8; t += 256) {
            const int per = (ATT_QS - p.ns) * ATT_BK * 8, s = t / per, i = t % per;
            const uint32_t a = smem_u32(ring + s * Cfg::STAGE + p.ns * ATT_BK * 128) + (uint32_t)i * 16u;
            asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u) : "memory");
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }

    float o[NV / 2];
#pragma unroll
    for (int e = 0; e < NV / 2; ++e) o[e] = 0.f;
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};   // running max, this thread's share of the running sum (rows r, r + 8)
    const uint64_t dq = make_smem_desc_sw128(smem_u32(smem) + (uint32_t)wg * 64u * 128u);
    const float osq = 1.f / (GVD_ATT_SQ * GVD_ATT_SK), osv = 1.f / (GVD_ATT_SP * GVD_ATT_SV);
    constexpr bool SKIP_LAST = NV <= ATT_QS * 32 - 16;             // hs <= 176: the last k16 step of the key image holds only zero pads

    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb & 1;
        mbar_wait(&full[s], (uint32_t)(kb >> 1) & 1u);
        const uint32_t kbase = smem_u32(ring + s * Cfg::STAGE);

        // ---- S = Q K^T: one fold per head-dimension slice; slice sl + 1 is in flight while slice sl is folded
        float sc[16], d[2][16];
#pragma unroll
        for (int e = 0; e < 16; ++e) sc[e] = 0.f;
#pragma unroll
        for (int sl = 0; sl <= ATT_QS; ++sl) {
            if (sl < ATT_QS) {
                const uint64_t da = dq + (uint64_t)((sl * ATT_BM * 128) >> 4), db = make_smem_desc_sw128(kbase + (uint32_t)sl * ATT_BK * 128u);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < ((SKIP_LAST && sl == ATT_QS - 1) ? 1 : 2); ++ks) {
                    const uint64_t ah = da + 2 * ks, al = ah + 4, bh = db + 2 * ks, bl = bh + 4;
                    wgmma_f16(d[sl & 1], al, bh, ks == 0 ? 0u : 1u);
                    wgmma_f16(d[sl & 1], ah, bl, 1u);
                    wgmma_f16(d[sl & 1], ah, bh, 1u);
                }
                wgmma_commit();
            }
            if (sl >= 1) {
                if (sl < ATT_QS) wgmma_wait<1>(d[(sl - 1) & 1]);
                else wgmma_wait<0>(d[(sl - 1) & 1]);
#pragma unroll
                for (int e = 0; e < 16; ++e) sc[e] = fmaf(d[(sl - 1) & 1][e], osq, sc[e]);   // undo the power-of-two operand scales (exact)
            }
        }

        // ---- online softmax; thread holds rows r (sc[4j], sc[4j + 1]) and r + 8 (sc[4j + 2], sc[4j + 3]) at keys 8j + 2c (+1)
        const int key0 = kb * ATT_BK;
        if (key0 + ATT_BK > p.R) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (key0 + 8 * j + 2 * c + e >= p.R) sc[4 * j + e] = sc[4 * j + 2 + e] = -INFINITY;
        }
        float mx0 = mrow[0], mx1 = mrow[1];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            mx0 = fmaxf(mx0, fmaxf(sc[4 * j], sc[4 * j + 1]));
            mx1 = fmaxf(mx1, fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float al0 = ex2_approx((mrow[0] - mx0) * p.c2), al1 = ex2_approx((mrow[1] - mx1) * p.c2);
        mrow[0] = mx0; mrow[1] = mx1;
        // A fragment of k16 step ks: [4 ks + 0] row r keys 16 ks + 2c, [+1] row r + 8, [+2] row r keys 16 ks + 8 + 2c, [+3] row r + 8
        uint32_t ph[8], pl[8];
        float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float e0 = ex2_approx((sc[4 * j] - mx0) * p.c2), e1 = ex2_approx((sc[4 * j + 1] - mx0) * p.c2);
            const float e2 = ex2_approx((sc[4 * j + 2] - mx1) * p.c2), e3 = ex2_approx((sc[4 * j + 3] - mx1) * p.c2);
            ps0 += e0 + e1;
            ps1 += e2 + e3;
            const int f = 4 * (j >> 1) + 2 * (j & 1);
            f16x3_split_pair(e0, e1, GVD_ATT_SP, ph[f], pl[f]);
            f16x3_split_pair(e2, e3, GVD_ATT_SP, ph[f + 1], pl[f + 1]);
        }
        lrow[0] = fmaf(lrow[0], al0, ps0);
        lrow[1] = fmaf(lrow[1], al1, ps1);

        // ---- O = O * alpha + (P V) * oscale: two column halves, the second in flight while the first is folded
        float pv[2][NH / 2];
        const uint64_t dv = make_smem_desc_sw128(kbase + ATT_K_BYTES);
        wgmma_fence();
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const uint64_t bh = dv + (uint64_t)((hf * NH * 128) >> 4) + 2 * ks, bl = bh + 4;
                const uint32_t ahi[4] = {ph[4 * ks], ph[4 * ks + 1], ph[4 * ks + 2], ph[4 * ks + 3]};
                const uint32_t alo[4] = {pl[4 * ks], pl[4 * ks + 1], pl[4 * ks + 2], pl[4 * ks + 3]};
                wgmma_f16_rs(pv[hf], alo, bh, ks == 0 ? 0u : 1u);
                wgmma_f16_rs(pv[hf], ahi, bl, 1u);
                wgmma_f16_rs(pv[hf], ahi, bh, 1u);
            }
            wgmma_commit();
        }
        wgmma_wait<1>(pv[0]);
#pragma unroll
        for (int e = 0; e < NH / 2; ++e) o[e] = fmaf(pv[0][e], osv, o[e] * ((e & 2) ? al1 : al0));
        wgmma_wait<0>(pv[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);                  // stage free once this warp's products have read it
#pragma unroll
        for (int e = 0; e < NH / 2; ++e) o[NH / 2 + e] = fmaf(pv[1][e], osv, o[NH / 2 + e] * ((e & 2) ? al1 : al0));
    }

    // ---------------------------------------------------------------------- O / row sum -> fp32 O or its operand image
    lrow[0] += __shfl_xor_sync(0xffffffffu, lrow[0], 1); lrow[0] += __shfl_xor_sync(0xffffffffu, lrow[0], 2);
    lrow[1] += __shfl_xor_sync(0xffffffffu, lrow[1], 1); lrow[1] += __shfl_xor_sync(0xffffffffu, lrow[1], 2);
    const float inv0 = 1.f / lrow[0], inv1 = 1.f / lrow[1];
    // lane pairs (c, c ^ 1) trade halves: even c stores 4 columns of row r, odd c the same 4 columns of row r + 8
    const bool odd = c & 1;
    const int r = qt * ATT_BM + wg * 64 + (warp & 3) * 16 + (lane >> 2) + (odd ? 8 : 0);
    const bool row_ok = r < p.R;
    const long long grow = (long long)b * p.R + r;
#pragma unroll
    for (int j = 0; j < NV / 8; ++j) {
        const float x0 = o[4 * j] * inv0, x1 = o[4 * j + 1] * inv0, y0 = o[4 * j + 2] * inv1, y1 = o[4 * j + 3] * inv1;
        const float t0 = __shfl_xor_sync(0xffffffffu, odd ? x0 : y0, 1), t1 = __shfl_xor_sync(0xffffffffu, odd ? x1 : y1, 1);
        const float v0 = odd ? t0 : x0, v1 = odd ? t1 : x1, v2 = odd ? y0 : t0, v3 = odd ? y1 : t1;
        const int n = 8 * j + 4 * (c >> 1);
        if (!row_ok || n >= p.hs) continue;                     // columns [hs, NV) of the product belong to the next head
        if (p.img) {
            uint32_t h0, l0, h1, l1;
            f16x3_split_pair(v0, v1, GVD_F16_SA, h0, l0);
            f16x3_split_pair(v2, v3, GVD_F16_SA, h1, l1);
            uint32_t* w = p.img + grow * p.img_ld + f16x3_word(h * p.hs + n);
            *reinterpret_cast<uint2*>(w) = make_uint2(h0, h1);
            *reinterpret_cast<uint2*>(w + 16) = make_uint2(l0, l1);
        } else {
            *reinterpret_cast<float4*>(p.out + grow * p.ldo + (long long)h * p.hs + n) = make_float4(v0, v1, v2, v3);
        }
    }
    if (p.img && row_ok && h == p.nh - 1 && c < 2) {
        // the K padding of the next GEMM's operand (columns [nh * hs, img_ld) of the row) belongs to no head: zeros
        uint32_t* irow = p.img + grow * p.img_ld;
        for (int gc = p.nh * p.hs; gc < (int)p.img_ld; gc += 4) {
            uint32_t* w = irow + f16x3_word(gc);
            *reinterpret_cast<uint2*>(w) = make_uint2(0u, 0u);
            *reinterpret_cast<uint2*>(w + 16) = make_uint2(0u, 0u);
        }
    }
}

template <int NV>
int launch_attn(const CUtensorMap& mK, const CUtensorMap& mV, const AttnParams& p, dim3 grid, cudaStream_t st) {
    static bool attr_set = false;
    if (!attr_set) {
        GVD_CHECK_CUDA(cudaFuncSetAttribute(self_attn_fused_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AttCfg<NV>::SMEM));
        attr_set = true;
    }
    GVD_CHECK_CUDA(gvd_launch(self_attn_fused_kernel<NV>, grid, dim3(ATT_THREADS), AttCfg<NV>::SMEM, st, mK, mV, p));
    GVD_CHECK_LAUNCH();
    return 0;
}

}  // namespace

int gvd_self_attn_fused(const float* q, long long ldq, const float* k_img, const float* vt_img, int B, int R, int nh, int hs, int HP, float scale,
                        float* out, long long ldo, float* img, long long img_ld, cudaStream_t st) {
    GVD_REQUIRE(q && k_img && vt_img && (out || img) && B > 0 && R > 0 && nh > 0 && hs > 0 && hs <= ATT_QS * 32 && hs % 4 == 0 && nh * hs <= HP,
                "self_attn_fused: bad problem (head size %d must be a multiple of 4, <= 192)", hs);
    GVD_REQUIRE(ldq % 4 == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0, "self_attn_fused: Q rows must be 16-byte aligned");
    GVD_REQUIRE(img || (ldo % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0), "self_attn_fused: O rows must be 16-byte aligned");
    GVD_REQUIRE(!img || (img_ld % 32 == 0 && img_ld >= (long long)nh * hs && (reinterpret_cast<uintptr_t>(img) & 15) == 0),
                "self_attn_fused: output image pitch");
    const int KH = (hs + 31) / 32 * 32, Rp = (R + 31) / 32 * 32;
    const int NV = hs <= 176 ? 176 : 192;
    AttnParams p{};
    p.q = q; p.ldq = ldq; p.out = img ? nullptr : out; p.ldo = ldo;
    p.img = reinterpret_cast<uint32_t*>(img); p.img_ld = img_ld;
    p.R = R; p.nh = nh; p.hs = hs; p.ns = KH / 32;
    p.c2 = scale * 1.4426950408889634f;
    CUtensorMap mK, mV;
    int unused;
    // key image [b][r][h][KH words]: box = one 32-word slice of 32 keys; V^T image [b][HP columns][Rp words]: box = one 32-key block of NV columns
    GVD_TRY(make_map(&mK, k_img, KH, R, (long long)nh * KH, nh, KH, B, (long long)R * nh * KH, ATT_BK, &p.k_mul_h, &p.k_mul_b));
    GVD_TRY(make_map(&mV, vt_img, Rp, HP, Rp, 1, 0, B, (long long)HP * Rp, NV, &unused, &p.v_mul_b));
    const dim3 grid(gvd_cdiv(R, ATT_BM), nh, B);
    return NV == 176 ? launch_attn<176>(mK, mV, p, grid, st) : launch_attn<192>(mK, mV, p, grid, st);
}
