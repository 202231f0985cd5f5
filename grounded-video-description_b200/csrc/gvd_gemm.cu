// gvd-b200: register-tiled fp32 NT GEMM (see gvd_gemm.cuh).  sm_90a, no tensor cores:
// BMxBN CTA tile, BK=16 slices staged k-major in double-buffered shared memory, TMxTN
// accumulators per thread, 128-bit global loads along K, 128-bit shared loads, 128-bit stores.
#include "gvd_gemm.cuh"

namespace {

constexpr int BK = 16;
constexpr int PAD = 4;

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_nt_kernel(GemmArgs g) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int NTX = BN / TN;                      // threads along N
    constexpr int A_F4 = BM * BK / 4, W_F4 = BN * BK / 4;
    constexpr int A_IT = A_F4 / NT, W_IT = W_F4 / NT;
    static_assert(A_F4 % NT == 0 && W_F4 % NT == 0, "tile/threads mismatch");
    static_assert(TM == 4 || TM == 8, "TM");
    static_assert(TN == 4 || TN == 8, "TN");

    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Ws[2][BK][BN + PAD];

    const int tid = threadIdx.x;
    const int tx = tid % NTX, ty = tid / NTX;
    const int zb = blockIdx.z / g.nh, zh = blockIdx.z % g.nh;
    const float* __restrict__ A = g.A + zb * g.sAb + zh * g.sAh;
    const float* __restrict__ W = g.W + zb * g.sWb + zh * g.sWh;
    float* __restrict__ C = g.C + zb * g.sCb + zh * g.sCh;
    const float* __restrict__ bias = g.bias ? g.bias + zb * g.sBb : nullptr;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float4 ra[A_IT], rw[W_IT];
    auto gload = [&](int k0) {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int f = tid + i * NT, row = f / (BK / 4), kq = f % (BK / 4);
            const int m = m0 + row, k = k0 + kq * 4;
            ra[i] = (m < g.M && k < g.K) ? __ldg(reinterpret_cast<const float4*>(A + (long long)m * g.lda + k))
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < W_IT; ++i) {
            const int f = tid + i * NT, row = f / (BK / 4), kq = f % (BK / 4);
            const int n = n0 + row, k = k0 + kq * 4;
            rw[i] = (n < g.N && k < g.K) ? __ldg(reinterpret_cast<const float4*>(W + (long long)n * g.ldw + k))
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < A_IT; ++i) {
            const int f = tid + i * NT, row = f / (BK / 4), kq = f % (BK / 4);
            As[buf][kq * 4 + 0][row] = ra[i].x;
            As[buf][kq * 4 + 1][row] = ra[i].y;
            As[buf][kq * 4 + 2][row] = ra[i].z;
            As[buf][kq * 4 + 3][row] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < W_IT; ++i) {
            const int f = tid + i * NT, row = f / (BK / 4), kq = f % (BK / 4);
            Ws[buf][kq * 4 + 0][row] = rw[i].x;
            Ws[buf][kq * 4 + 1][row] = rw[i].y;
            Ws[buf][kq * 4 + 2][row] = rw[i].z;
            Ws[buf][kq * 4 + 3][row] = rw[i].w;
        }
    };

    const int nk = (g.K + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
                const float4 v = *reinterpret_cast<const float4*>(&As[buf][k][(i / 4) * (BM / 2) + ty * 4]);
                a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
                const float4 v = *reinterpret_cast<const float4*>(&Ws[buf][k][(j / 4) * (BN / 2) + tx * 4]);
                b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            sstore(buf ^ 1);      // the other buffer was last read in iteration kt-1, fenced by its barrier
            __syncthreads();
        }
    }

    // epilogue
    const bool vec_ok = (g.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + (i / 4) * (BM / 2) + ty * 4 + (i % 4);
        if (m >= g.M) continue;
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
            const int n = n0 + (j / 4) * (BN / 2) + tx * 4;
            float v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float x = acc[i][j + q] * g.alpha;
                const int nn = n + q;
                if (nn < g.N) {
                    if (bias) x += __ldg(bias + nn);
                    if (g.act >= GVD_ACT_RELU) x = fmaxf(x, 0.f);
                    if (g.act == GVD_ACT_RELU_AFFINE_RELU) x = fmaxf(fmaf(x, __ldg(g.scale2 + nn), __ldg(g.shift2 + nn)), 0.f);
                }
                v[q] = x;
            }
            float* dst = C + (long long)m * g.ldc + n;
            if (vec_ok && n + 3 < g.N) {
                *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (n + q < g.N) dst[q] = v[q];
            }
        }
    }
}

template <int BM, int BN, int TM, int TN>
int launch(const GemmArgs& g, int batch, cudaStream_t stream) {
    dim3 grid(gvd_cdiv(g.N, BN), gvd_cdiv(g.M, BM), batch);
    gemm_nt_kernel<BM, BN, TM, TN><<<grid, (BM / TM) * (BN / TN), 0, stream>>>(g);
    GVD_CHECK_LAUNCH();
    return 0;
}

}  // namespace

int gvd_gemm_nt_tc(const GemmArgs& g, int batch, cudaStream_t stream);

int gvd_gemm_nt(const GemmArgs& g, int batch, cudaStream_t stream) {
    if (gvd_backend_on(BK_TC) && g.M >= 32 && batch % g.nh == 0) return gvd_gemm_nt_tc(g, batch, stream);
    GVD_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
    GVD_REQUIRE(g.K % 4 == 0 && g.lda % 4 == 0 && g.ldw % 4 == 0, "gemm: K/lda/ldw must be multiples of 4 (K=%d lda=%lld ldw=%lld)",
                g.K, g.lda, g.ldw);
    GVD_REQUIRE(((uintptr_t)g.A & 15) == 0 && ((uintptr_t)g.W & 15) == 0, "gemm: operands must be 16-byte aligned");
    GVD_REQUIRE(g.sAb % 4 == 0 && g.sAh % 4 == 0 && g.sWb % 4 == 0 && g.sWh % 4 == 0, "gemm: batch strides must be multiples of 4");
    GVD_REQUIRE(g.act != GVD_ACT_RELU_AFFINE_RELU || (g.scale2 && g.shift2), "gemm: act=2 needs scale2/shift2");
    GVD_REQUIRE(batch >= 1 && batch <= 65535 && g.nh >= 1, "gemm: bad batch %d", batch);
    // tile choice: fill 132 SMs; skinny problems take narrower N tiles
    const long long ctas_big = (long long)gvd_cdiv(g.M, 128) * gvd_cdiv(g.N, 128) * batch;
    if (g.M > 64 && ctas_big >= 132) return launch<128, 128, 8, 8>(g, batch, stream);
    if (g.M > 64) {
        const long long ctas_mid = (long long)gvd_cdiv(g.M, 128) * gvd_cdiv(g.N, 64) * batch;
        if (ctas_mid >= 120) return launch<128, 64, 8, 4>(g, batch, stream);
        return launch<128, 32, 8, 4>(g, batch, stream);
    }
    return launch<64, 64, 4, 4>(g, batch, stream);
}
