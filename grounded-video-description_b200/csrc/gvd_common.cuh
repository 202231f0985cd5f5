// gvd-b200: shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>

#define GVD_MIN_VALUE (-1e8f)   // misc/model.py:71, misc/AttModel.py:29,66

// ---------------------------------------------------------------- error plumbing (C-ABI: int status)
void gvd_set_error(const char* fmt, ...);
#define GVD_CHECK_CUDA(expr)                                                            \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            gvd_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            (void)cudaGetLastError();   /* reported: do not leave it for the next launch check */ \
            return 2;                                                                   \
        }                                                                               \
    } while (0)
void gvd_count_launch();
long long gvd_launch_count();                 // kernels launched so far (gvd_op_kernel_launches)
void gvd_launch_count_add(long long n);       // graph capture records launches without running them: callers correct the count
#define GVD_CHECK_LAUNCH()                  \
    do {                                    \
        gvd_count_launch();                 \
        GVD_CHECK_CUDA(cudaGetLastError()); \
    } while (0)
#define GVD_REQUIRE(cond, ...)                                                          \
    do {                                                                                \
        if (!(cond)) { gvd_set_error(__VA_ARGS__); return 1; }                          \
    } while (0)
#define GVD_TRY(expr)                                                                   \
    do { int _s = (expr); if (_s != 0) return _s; } while (0)

static inline int gvd_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------- warp / block reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// block-wide sum / max; `red` is >= 32 floats of shared memory; all threads get the result
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : 0.f;
    r = warp_sum(r);
    return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : -INFINITY;
    r = warp_max(r);
    return r;
}

// ---------------------------------------------------------------- accurate-enough transcendental
// tanh with ~2e-7 ABSOLUTE error from two MUFU ops (ex2 + rcp).  tanh.approx (2^-11 relative) is
// too coarse for the 1e-4 attention-logit bound; libm tanhf costs ~20 issue slots per element and
// the decode step evaluates (R+T)*A of them per clip.
__device__ __forceinline__ float tanh_mufu(float x) {
    const float ax = fminf(fabsf(x), 15.f);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * 2.8853900817779268f));  // exp(2|x|)
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.f));
    const float t = fmaf(-2.f, r, 1.f);
    return copysignf(t, x);
}
// round-to-nearest(-away) fp32 -> tf32 on the integer pipe (cvt.rna.tf32.f32 is emulated by ptxas in 5 instructions);
// x = hi + lo with hi exactly representable in tf32 is the operand split of every 3xTF32 tensor-core product here
__device__ __forceinline__ float tf32_rna(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }
__device__ __forceinline__ float ex2_approx(float x) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
    return e;
}
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------- counter-based random numbers (train-mode dropout, multinomial sampler)
// Philox4x32-10 (Salmon et al., SC'11): four 32-bit words from a 128-bit counter and a 64-bit key, no state.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// ---------------------------------------------------------------- fp16x3 operand image (gvd_wgmma.cu: skinny_f16_kernel, pre-split weights)
// A row of K fp32 values is stored as K 32-bit words: per 32-wide K slice 16 words of hi pairs (k = 2p, 2p + 1 in word p, low half = even k)
// followed by 16 words of lo pairs; hi = the value rounded to 11 significant bits (exact in fp16), lo = fp16(value - hi); values are
// multiplied by a power-of-two scale first.  word index of the hi pair of column k (even): (k / 32) * 32 + (k % 32) / 2, lo pair: + 16.
__device__ __forceinline__ uint32_t f16x3_pack_pair(float lo_elem, float hi_elem) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}
__device__ __forceinline__ void f16x3_split_pair(float x0, float x1, float scale, uint32_t& hi, uint32_t& lo) {
    x0 *= scale; x1 *= scale;
    const float a0 = __uint_as_float((__float_as_uint(x0) + 0x1000u) & 0xFFFFE000u), a1 = __uint_as_float((__float_as_uint(x1) + 0x1000u) & 0xFFFFE000u);
    hi = f16x3_pack_pair(a0, a1);
    lo = f16x3_pack_pair(x0 - a0, x1 - a1);
}
__device__ __forceinline__ long long f16x3_word(int k_even) { return (long long)(k_even >> 5) * 32 + ((k_even & 31) >> 1); }

// ---------------------------------------------------------------- programmatic dependent launch (decode loop, backend bit 6)
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor is still running:
// pdl_trigger() lets the NEXT kernel be scheduled early, pdl_wait() blocks until the predecessor has completed and its writes are
// visible.  Everything before pdl_wait() may only touch data that no kernel of the loop writes (weights, prologue features).
// Both are no-ops when the kernel was launched normally.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool gvd_pdl();

// ---------------------------------------------------------------- backend bits (gvd_set_backend; default 923, include/gvd_b200.h)
// Bits 2, 5 and 10 are inert: accepted so that stored flag values keep working, read by nothing.
enum GvdBackendBit : int {
    BK_TC = 1,                // bit 0: wgmma tensor cores for every GEMM-shaped stage (else fp32 CUDA cores)
    BK_FUSED_ATTN = 2,        // bit 1: fused self-attention pair of the region encoder
    BK_SPLITK = 8,            // bit 3: operand-swapped split-K decode products with the fused reduce + sampler
    BK_F16X3 = 16,            // bit 4: fp16x3 instead of 3xTF32 in the forward GEMMs (pre-split constant weights)
    BK_PDL = 64,              // bit 6: programmatic dependent launch in the decode loops
    BK_SS_GEMM = 128,         // bit 7: conversion-free prologue GEMMs (both operands as fp16x3 images straight from TMA)
    BK_ATT_F16 = 256,         // bit 8: fp16x3 images instead of tf32 planes in the fused self-attention pair
    BK_PACK_FUSION = 512,     // bit 9: the producer of a prologue activation stores the operand image the next GEMM streams
};
int gvd_backend();
static inline bool gvd_backend_on(int bits) { return (gvd_backend() & bits) == bits; }      // every bit of `bits` is set
// launch helper: <<<>>> or, with backend bit 6, cudaLaunchKernelEx + the programmatic-serialization attribute
template <typename... KArgs, typename... Args>
static inline cudaError_t gvd_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = gvd_pdl() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// ---------------------------------------------------------------- mbarrier + bulk-copy (TMA) PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// 1-D bulk async copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
