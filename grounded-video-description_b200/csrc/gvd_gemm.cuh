// gvd-b200: fp32 "NT" GEMM  C[M,N] = act(alpha * A[M,K] . W[N,K]^T + bias[N])  on the CUDA cores.
//
// Every dense contraction of the prologue (misc/model.py:510-565, misc/transformer.py:98-133)
// is an x @ weight.T with both operands K-contiguous, so one kernel family serves all of them;
// blockIdx.z walks a (batch, head) grid with independent strides for the per-clip / per-head
// contractions of the object-interaction attention.  fp32 accumulate in registers: greedy token
// ids must be bit-exact against an fp32 oracle, which plain TF32/BF16 tensor-core math is not
// (SURVEY.md section 7, "hard parts").
#pragma once
#include "gvd_common.cuh"

struct GemmArgs {
    const float* A; long long lda, sAb, sAh;
    const float* W; long long ldw, sWb, sWh;
    float* C;       long long ldc, sCb, sCh;
    const float* bias;     // [N] or nullptr
    long long sBb;         // bias stride per batch entry b (0: shared)
    const float* scale2;   // act==2: v = relu(relu(v) * scale2[n] + shift2[n])  (BatchNorm1d eval + ReLU)
    const float* shift2;
    int M, N, K;           // K % 4 == 0, lda % 4 == 0, ldw % 4 == 0, 16-byte aligned bases
    int nh;                // heads per batch entry (blockIdx.z = b * nh + h)
    int act;               // 0 none, 1 relu, 2 relu->affine->relu
    float alpha;
    int trans_c;           // tensor-core path only: store C transposed, C[n * ldc + m] (no bias / activation): the split-K partials of the
                           // operand-swapped skinny products come out batch-major, so every later pass reads them along the contiguous dimension
};

enum { GVD_ACT_NONE = 0, GVD_ACT_RELU = 1, GVD_ACT_RELU_AFFINE_RELU = 2 };

int gvd_gemm_nt(const GemmArgs& a, int batch, cudaStream_t stream);

// convenience: plain 2-D  C = act(A W^T + b)
static inline int gvd_linear(const float* A, long long lda, const float* W, long long ldw, const float* bias, float* C,
                             long long ldc, int M, int N, int K, int act, cudaStream_t stream) {
    GemmArgs g{};
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.C = C; g.ldc = ldc; g.bias = bias;
    g.M = M; g.N = N; g.K = K; g.nh = 1; g.act = act; g.alpha = 1.f;
    return gvd_gemm_nt(g, 1, stream);
}
