// Primitive set of the training step (gvd_b200/train.py; SURVEY 8 rows T7 / D1): the element-wise, row-wise and reduction
// kernels of the explicit backward.  The dense products go through the wgmma GEMM (gvd_op_linear / gvd_tr_gemm_nt_batched).
//
// Every function here has its
// mathematical definition in tests/ops_ref.py (same name) and a per-primitive device test in tests/test_gpu_zz_train.py.
// All tensors fp32, contiguous.  Reductions are deterministic (fixed summation order, no float atomics except cls_nll's scatter of
// equal addends).
#include <algorithm>

#include "../../include/gvd_b200.h"
#include "gvd_common.cuh"
#include "gvd_kernels.cuh"

namespace {

constexpr int TB = 256;

// ---------------------------------------------------------------- element-wise
enum { EW_ADD = 0, EW_MUL = 1, EW_SCALE = 2, EW_RELU = 3, EW_RELU_BWD = 4, EW_MASKED_FILL = 5 };
__global__ void ew_kernel(int op, const float* __restrict__ a, const float* __restrict__ b, const unsigned char* __restrict__ mask, float s,
                          float* __restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float v;
        switch (op) {
            case EW_ADD: v = a[i] + b[i]; break;
            case EW_MUL: v = a[i] * b[i]; break;
            case EW_SCALE: v = a[i] * s; break;
            case EW_RELU: v = fmaxf(a[i], 0.f); break;
            case EW_RELU_BWD: v = b[i] > 0.f ? a[i] : 0.f; break;       // a = dy, b = y
            default: v = mask[i] ? s : a[i]; break;                      // EW_MASKED_FILL
        }
        out[i] = v;
    }
}
// out[b,n,h] = a[b,n] * v[b,h]
__global__ void outer_rows_kernel(const float* __restrict__ a, const float* __restrict__ v, float* __restrict__ out, int N, int H, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int h = (int)(i % H);
        const long long bn = i / H;
        out[i] = a[bn] * v[(bn / N) * H + h];
    }
}

// acc[b,n,h] += a[b,n] * v[b,h]   (the attention backward's d(features): accumulated in place instead of outer + add)
__global__ void outer_rows_acc_kernel(const float* __restrict__ a, const float* __restrict__ v, float* __restrict__ acc, int N, int H, long long total4) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
        const int h4 = (int)(i % (H / 4));
        const long long bn = i / (H / 4);
        const float s = a[bn];
        const float4 x = *reinterpret_cast<const float4*>(v + (bn / N) * H + 4 * h4);
        float4 y = reinterpret_cast<float4*>(acc)[i];
        y.x = fmaf(s, x.x, y.x); y.y = fmaf(s, x.y, y.y); y.z = fmaf(s, x.z, y.z); y.w = fmaf(s, x.w, y.w);
        reinterpret_cast<float4*>(acc)[i] = y;
    }
}

// ---------------------------------------------------------------- reductions (deterministic)
// out[z][n] = sum_m x[z][m][n]: block (32, 8) per 32 columns; fixed order: each thread strides rows, then the 8 partials in order
// Tall matrices (the bias gradients: 10^5 rows) are summed in two deterministic phases: blockIdx.z owns a contiguous range of rows and
// writes one partial row, a second launch of the same kernel adds the partial rows (RB = gridDim.z row blocks, fixed order everywhere).
__global__ void colsum_kernel(const float* __restrict__ x, float* __restrict__ out, long long M, int N, long long rows_per_block, long long out_stride_z) {
    __shared__ float red[8][33];
    const int n = blockIdx.x * 32 + threadIdx.x;
    const float* xz = x + (long long)blockIdx.y * M * N;
    const long long m0 = (long long)blockIdx.z * rows_per_block, m1 = min(M, m0 + rows_per_block);
    float s = 0.f;
    if (n < N)
        for (long long m = m0 + threadIdx.y; m < m1; m += 8) s += xz[m * N + n];
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
        out[(long long)blockIdx.z * out_stride_z + (long long)blockIdx.y * N + n] = t;
    }
}
__global__ void rowsum_kernel(const float* __restrict__ x, float* __restrict__ out, int N) {
    __shared__ float red[32];
    const float* r = x + (long long)blockIdx.x * N;
    float s = 0.f;
    for (int j = threadIdx.x; j < N; j += blockDim.x) s += r[j];
    s = block_sum(s, red);
    if (threadIdx.x == 0) out[blockIdx.x] = s;
}
// one block: out[0] = sum x (double accumulation: gradient norms over up to 1e7 elements)
__global__ void sum_all_kernel(const float* __restrict__ x, float* __restrict__ out, long long n) {
    __shared__ double red[32];
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) s += (double)x[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
        out[0] = (float)t;
    }
}
// out[b,f] = mean_t x[b,t,f]
__global__ void mean_dim1_kernel(const float* __restrict__ x, float* __restrict__ out, int T, int F, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int f = (int)(i % F);
    const long long b = i / F;
    float s = 0.f;
    for (int t = 0; t < T; ++t) s += x[(b * T + t) * F + f];
    out[i] = s / (float)T;
}

// ---------------------------------------------------------------- row-wise (one block per row of n columns)
__global__ void ln_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int n) {
    __shared__ float red[32];
    const float* r = x + (long long)blockIdx.x * n;
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += r[j];
    const float mu = block_sum(s, red) / n;
    float q = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) { const float d = r[j] - mu; q += d * d; }
    const float inv = rsqrtf(block_sum(q, red) / n + 1e-5f);
    for (int j = threadIdx.x; j < n; j += blockDim.x) y[(long long)blockIdx.x * n + j] = (r[j] - mu) * inv;
}
// dx = (dy - mean(dy) - y mean(dy y)) / sigma
__global__ void ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ x, float* __restrict__ dx, int n) {
    __shared__ float red[32];
    const long long o = (long long)blockIdx.x * n;
    float s = 0.f, q = 0.f, a = 0.f, b = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += x[o + j];
    const float mu = block_sum(s, red) / n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) { const float d = x[o + j] - mu; q += d * d; a += dy[o + j]; b += dy[o + j] * y[o + j]; }
    const float inv = rsqrtf(block_sum(q, red) / n + 1e-5f);
    const float ma = block_sum(a, red) / n, mb = block_sum(b, red) / n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) dx[o + j] = (dy[o + j] - ma - y[o + j] * mb) * inv;
}
// y = gamma (x - mu) / (std_unbiased + 1e-6) + beta   (transformer.py:74-77)
__global__ void ln_star_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ be, float* __restrict__ y, int n) {
    __shared__ float red[32];
    const long long o = (long long)blockIdx.x * n;
    float s = 0.f, q = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += x[o + j];
    const float mu = block_sum(s, red) / n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) { const float d = x[o + j] - mu; q += d * d; }
    const float d = sqrtf(block_sum(q, red) / (n - 1)) + 1e-6f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) y[o + j] = g[j] * (x[o + j] - mu) / d + be[j];
}
// dx = (g - mean g)/d - xc (sum g xc) / (d^2 (n-1) std),  g = dy gamma;  tmp = dy xc / d  (column sums of tmp = dgamma)
__global__ void ln_star_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ gam, float* __restrict__ dx,
                                   float* __restrict__ tmp, int n) {
    __shared__ float red[32];
    const long long o = (long long)blockIdx.x * n;
    float s = 0.f, q = 0.f, a = 0.f, b = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += x[o + j];
    const float mu = block_sum(s, red) / n;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const float xc = x[o + j] - mu, g = dy[o + j] * gam[j];
        q += xc * xc; a += g; b += g * xc;
    }
    const float std = sqrtf(block_sum(q, red) / (n - 1)), d = std + 1e-6f;
    const float mg = block_sum(a, red) / n, sgx = block_sum(b, red);
    const float k = sgx / (d * d * (float)(n - 1) * std);
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const float xc = x[o + j] - mu;
        dx[o + j] = (dy[o + j] * gam[j] - mg) / d - xc * k;
        tmp[o + j] = dy[o + j] * xc / d;
    }
}
__global__ void softmax_fwd_kernel(const float* __restrict__ x, float scale, float* __restrict__ p, int n) {
    __shared__ float red[32];
    const long long o = (long long)blockIdx.x * n;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, x[o + j] * scale);
    m = block_max(m, red);
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += expf(x[o + j] * scale - m);
    const float inv = 1.f / block_sum(s, red);
    for (int j = threadIdx.x; j < n; j += blockDim.x) p[o + j] = expf(x[o + j] * scale - m) * inv;
}
__global__ void softmax_bwd_kernel(const float* __restrict__ dp, const float* __restrict__ p, float scale, float* __restrict__ dx, int n) {
    __shared__ float red[32];
    const long long o = (long long)blockIdx.x * n;
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += p[o + j] * dp[o + j];
    s = block_sum(s, red);
    for (int j = threadIdx.x; j < n; j += blockDim.x) dx[o + j] = scale * p[o + j] * (dp[o + j] - s);
}
// language-model NLL (utils.py:126-136): rowloss = -(logit[target] - lse) on counted rows; dlogits = (softmax - onehot) mask inv_n
__global__ void lm_nll_kernel(const float* __restrict__ logits, const long long* __restrict__ target, const unsigned char* __restrict__ mask,
                              const float* __restrict__ inv_ptr, float* __restrict__ rowloss, float* __restrict__ dlogits, int n) {
    __shared__ float red[32];
    const float inv_n = __ldg(inv_ptr);
    const long long o = (long long)blockIdx.x * n;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, logits[o + j]);
    m = block_max(m, red);
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += expf(logits[o + j] - m);
    const float lse = m + logf(block_sum(s, red));
    const long long t = target[blockIdx.x];
    const float w = mask[blockIdx.x] ? inv_n : 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) dlogits[o + j] = (expf(logits[o + j] - lse) - (j == t ? 1.f : 0.f)) * w;
    if (threadIdx.x == 0) rowloss[blockIdx.x] = mask[blockIdx.x] ? -(logits[o + t] - lse) : 0.f;
}
// -sum over the positives of a row of log_softmax(x); dx = (n_pos_row softmax - pos) inv_n   (utils.py:139,142)
__global__ void pos_nll_kernel(const float* __restrict__ x, const unsigned char* __restrict__ pos, const float* __restrict__ inv_ptr,
                               float* __restrict__ rowloss, float* __restrict__ dx, int n) {
    __shared__ float red[32];
    const float inv_n = __ldg(inv_ptr);
    const long long o = (long long)blockIdx.x * n;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, x[o + j]);
    m = block_max(m, red);
    float s = 0.f, c = 0.f, l = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += expf(x[o + j] - m);
    const float lse = m + logf(block_sum(s, red));
    for (int j = threadIdx.x; j < n; j += blockDim.x)
        if (pos[o + j]) { c += 1.f; l -= x[o + j] - lse; }
    const float npr = block_sum(c, red);
    l = block_sum(l, red);
    for (int j = threadIdx.x; j < n; j += blockDim.x) dx[o + j] = (expf(x[o + j] - lse) * npr - (pos[o + j] ? 1.f : 0.f)) * inv_n;
    if (threadIdx.x == 0) rowloss[blockIdx.x] = l;
}
// region-class loss on the region-major similarity simT [B,R,C] with targets [B,NB,R] (model.py:345-350): per (b,k,r) with t > 0:
// loss -= max(log p, -100); d simT[b,r,t] -= inv_n / p (not where clamped).  part[idx] = the loss term (summed afterwards).
__global__ void cls_nll_kernel(const float* __restrict__ simT, const int* __restrict__ target, const float* __restrict__ inv_ptr,
                               float* __restrict__ part, float* __restrict__ dsimT, int R, int NB, int C, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const float inv_n = __ldg(inv_ptr);
    const int r = (int)(idx % R);
    const long long b = idx / ((long long)R * NB);
    const int t = target[idx];
    float term = 0.f;
    if (t > 0) {
        const long long e = (b * R + r) * C + t;
        const float p = simT[e], lp = logf(p);
        term = -fmaxf(lp, -100.f);
        if (lp > -100.f) atomicAdd(dsimT + e, -inv_n / p);
    }
    part[idx] = term;
}
__global__ void class_target_kernel(const float* __restrict__ ov, const float* __restrict__ gt, int* __restrict__ target, int R, int NB, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // (b, k, r)
    if (idx >= total) return;
    const int r = (int)(idx % R), k = (int)((idx / R) % NB);
    const long long b = idx / ((long long)R * NB);
    target[idx] = ov[(b * R + r) * NB + k] > 0.5f ? (int)gt[(b * NB + k) * 6 + 5] : 0;
}

// inv_out[0] = 1 / #{i : data[i] != 0 (bytes) or data[i] > 0 (int32)}: the 1/n of a masked mean, kept on the device (no host round trip).
// An empty set gives +inf, and the mean over it 0 * inf = NaN like torch's mean over nothing (the reference's empty-positive-set quirk Q11).
__global__ void count_inv_kernel(const void* __restrict__ data, long long n, int elem_bytes, float* __restrict__ inv_out, float* __restrict__ scaled,
                                 const float* __restrict__ value) {
    __shared__ long long red[32];
    long long c = 0;
    if (elem_bytes == 1) { const unsigned char* d = (const unsigned char*)data; for (long long i = threadIdx.x; i < n; i += blockDim.x) c += d[i] != 0; }
    else { const int* d = (const int*)data; for (long long i = threadIdx.x; i < n; i += blockDim.x) c += d[i] > 0; }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
        const float inv = t > 0 ? 1.f / (float)t : __int_as_float(0x7fc00000);
        inv_out[0] = inv;
        if (scaled) scaled[0] = value[0] * inv;
    }
}
// out[0] = a[0] * b[0]
__global__ void scalar_mul_kernel(const float* a, const float* b, float* out) { out[0] = a[0] * b[0]; }

// ---------------------------------------------------------------- recurrent cells
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ gates, const float* __restrict__ c, float* __restrict__ h2, float* __restrict__ c2,
                                     float* __restrict__ act, int H, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int j = (int)(idx % H);
    const long long b = idx / H, g0 = b * 4 * H + j;
    const float i = sigmoid_acc(gates[g0]), f = sigmoid_acc(gates[g0 + H]), g = tanhf(gates[g0 + 2 * H]), o = sigmoid_acc(gates[g0 + 3 * H]);
    const float cc = f * c[idx] + i * g;
    c2[idx] = cc;
    h2[idx] = o * tanhf(cc);
    act[g0] = i; act[g0 + H] = f; act[g0 + 2 * H] = g; act[g0 + 3 * H] = o;
}
__global__ void lstm_cell_bwd_kernel(const float* __restrict__ dh2, const float* __restrict__ dc2in, const float* __restrict__ act,
                                     const float* __restrict__ c, const float* __restrict__ c2, float* __restrict__ dgates, float* __restrict__ dc,
                                     int H, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int j = (int)(idx % H);
    const long long b = idx / H, g0 = b * 4 * H + j;
    const float i = act[g0], f = act[g0 + H], g = act[g0 + 2 * H], o = act[g0 + 3 * H];
    const float tc = tanhf(c2[idx]);
    const float dc2 = dc2in[idx] + dh2[idx] * o * (1.f - tc * tc);
    dgates[g0] = dc2 * g * i * (1.f - i);
    dgates[g0 + H] = dc2 * c[idx] * f * (1.f - f);
    dgates[g0 + 2 * H] = dc2 * i * (1.f - g * g);
    dgates[g0 + 3 * H] = dh2[idx] * tc * o * (1.f - o);
    dc[idx] = dc2 * f;
}
__global__ void gru_cell_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh, const float* __restrict__ h, float* __restrict__ h2,
                                    float* __restrict__ r_, float* __restrict__ z_, float* __restrict__ n_, int G, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int j = (int)(idx % G);
    const long long b = idx / G, g0 = b * 3 * G + j;
    const float r = sigmoid_acc(gi[g0] + gh[g0]), z = sigmoid_acc(gi[g0 + G] + gh[g0 + G]);
    const float n = tanhf(gi[g0 + 2 * G] + r * gh[g0 + 2 * G]);
    h2[idx] = (1.f - z) * n + z * h[idx];
    r_[idx] = r; z_[idx] = z; n_[idx] = n;
}
__global__ void gru_cell_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ r_, const float* __restrict__ z_, const float* __restrict__ n_,
                                    const float* __restrict__ h, const float* __restrict__ ghn, float* __restrict__ dgi, float* __restrict__ dgh,
                                    float* __restrict__ dh_keep, int G, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int j = (int)(idx % G);
    const long long b = idx / G, g0 = b * 3 * G + j;
    const float r = r_[idx], z = z_[idx], n = n_[idx], d = dh[idx];
    const float dpn = d * (1.f - z) * (1.f - n * n);
    const float dpr = dpn * ghn[idx] * r * (1.f - r);
    const float dpz = d * (h[idx] - n) * z * (1.f - z);
    dgi[g0] = dpr; dgi[g0 + G] = dpz; dgi[g0 + 2 * G] = dpn;
    dgh[g0] = dpr; dgh[g0 + G] = dpz; dgh[g0 + 2 * G] = dpn * r;
    dh_keep[idx] = d * z;
}

// ---------------------------------------------------------------- additive attention scores: s[b,n] = w . tanh(p[b,n,:] + q[b,:]) + bias
__global__ void att_scores_fwd_kernel(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w, const float* __restrict__ bias,
                                      float* __restrict__ s, int N, int A, long long rows) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;      // one warp per (b, n)
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const long long b = row / N;
    float acc = 0.f;
    for (int a = lane; a < A; a += 32) acc += w[a] * tanhf(p[row * A + a] + q[b * A + a]);
    acc = warp_sum(acc);
    if (lane == 0) s[row] = acc + bias[0];
}
// dpre[b,n,a] = ds[b,n] w[a] (1 - t^2),  dst[b,n,a] = ds[b,n] t   (t recomputed)
__global__ void att_scores_bwd_kernel(const float* __restrict__ ds, const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w,
                                      float* __restrict__ dpre, float* __restrict__ dst, int N, int A, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int a = (int)(i % A);
        const long long row = i / A, b = row / N;
        const float t = tanhf(p[i] + q[b * A + a]), d = ds[row];
        dpre[i] = d * w[a] * (1.f - t * t);
        dst[i] = d * t;
    }
}

// multiplicative scores ('mix_mul', AttModel.py:81-82): s[b,n] = w . tanh(p[b,n,:] * q[b,:]) + bias
__global__ void att_scores_mul_fwd_kernel(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ w,
                                          const float* __restrict__ bias, float* __restrict__ s, int N, int A, long long rows) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;      // one warp per (b, n)
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const long long b = row / N;
    float acc = 0.f;
    for (int a = lane; a < A; a += 32) acc += w[a] * tanhf(p[row * A + a] * q[b * A + a]);
    acc = warp_sum(acc);
    if (lane == 0) s[row] = acc + bias[0];
}
// dpre = ds[b,n] w[a] (1 - t^2):  dp[b,n,a] = dpre q[b,a],  dqt[b,n,a] = dpre p[b,n,a],  dst[b,n,a] = ds[b,n] t   (t recomputed; the sums over
// n / rows are the colsum kernel's, so nothing here accumulates across threads)
__global__ void att_scores_mul_bwd_kernel(const float* __restrict__ ds, const float* __restrict__ p, const float* __restrict__ q,
                                          const float* __restrict__ w, float* __restrict__ dp, float* __restrict__ dqt, float* __restrict__ dst, int N,
                                          int A, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int a = (int)(i % A);
        const long long row = i / A, b = row / N;
        const float pv = p[i], qv = q[b * A + a], t = tanhf(pv * qv), d = ds[row];
        const float dpre = d * w[a] * (1.f - t * t);
        dp[i] = dpre * qv;
        dqt[i] = dpre * pv;
        dst[i] = d * t;
    }
}

// ---------------------------------------------------------------- embeddings
__global__ void gather_rows_kernel(const float* __restrict__ table, const long long* __restrict__ idx, float* __restrict__ out, int D, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        out[i] = table[idx[i / D] * D + (i % D)];
}
// out[r, :] = sum over the m with idx[m] == r of rows[m, :]   (one block per output row, ascending m: deterministic)
__global__ void index_add_rows_kernel(const long long* __restrict__ idx, const float* __restrict__ rows, float* __restrict__ out, int M, int D) {
    const long long r = blockIdx.x;
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float s = 0.f;
        for (int m = 0; m < M; ++m)
            if (idx[m] == r) s += rows[(long long)m * D + d];
        out[r * D + d] = s;
    }
}

// ---------------------------------------------------------------- BatchNorm1d (train mode) pieces and Adam
__global__ void bn_normalize_kernel(const float* __restrict__ e, const float* __restrict__ mu, const float* __restrict__ var, float* __restrict__ out,
                                    int N, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % N);
        out[i] = (e[i] - mu[n]) * rsqrtf(var[n] + 1e-5f);
    }
}
// de = (dxh - s1/M - e_hat s2/M) / sqrt(var + eps),  s1 = colsum(dxh), s2 = colsum(dxh e_hat)
__global__ void bn_bwd_kernel(const float* __restrict__ dxh, const float* __restrict__ e_hat, const float* __restrict__ var, const float* __restrict__ s1,
                              const float* __restrict__ s2, float inv_m, float* __restrict__ de, int N, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % N);
        de[i] = (dxh[i] - s1[n] * inv_m - e_hat[i] * s2[n] * inv_m) * rsqrtf(var[n] + 1e-5f);
    }
}
// first Adam step (exp_avg = exp_avg_sq = 0 before it) on clipped gradients, torch.optim.Adam arithmetic
__global__ void adam_first_step_kernel(const float* __restrict__ w, const float* __restrict__ g, float coef, float lr, float b1, float b2, float eps,
                                       float* __restrict__ out, long long n) {
    const float bc2 = sqrtf(1.f - b2);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gg = g[i] * coef;
        const float m = (1.f - b1) * gg, v = (1.f - b2) * gg * gg;
        out[i] = w[i] - (lr / (1.f - b1)) * m / (sqrtf(v) / bc2 + eps);
    }
}


// ---------------------------------------------------------------- flat-buffer optimiser (main.py:265-266,660-677)
// Global gradient norm of the flat fp32 gradient buffer, deterministic: fixed grid, per-block double partials, one finishing block.
constexpr int SQ_BLOCKS = 1056;      // 8 x 132 SMs
__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, long long n, double* __restrict__ part) {
    __shared__ double red[8];
    double s = 0.0;
    const long long n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = g4[i];
        s += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[(n4 << 2) + threadIdx.x]; s += (double)v * v; }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < 8; ++k) t += red[k];
        part[blockIdx.x] = t;
    }
}
// norm_out[0] = sqrt(sum), norm_out[1] = clip coefficient min(max_norm / (norm + 1e-6), 1)  (torch.nn.utils.clip_grad_norm_)
__global__ void __launch_bounds__(256) sumsq_finish_kernel(const double* __restrict__ part, int nparts, float max_norm, float* __restrict__ norm_out) {
    __shared__ double red[8];
    double s = 0.0;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) s += part[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int k = 0; k < 8; ++k) t += red[k];
        const float nrm = (float)sqrt(t);
        norm_out[0] = nrm;
        norm_out[1] = max_norm > 0.f ? fminf(max_norm / (nrm + 1e-6f), 1.f) : 1.f;
    }
}
// torch.optim.Adam (single-tensor arithmetic, amsgrad off) over the flat parameter buffer; segment s covers [seg_end[s-1], seg_end[s]) and
// carries its own learning rate (one param group per tensor, main.py:660-669); lr <= 0 marks a tensor that never receives a gradient
// (torch skips it: no state, no decay).  The clip coefficient is read from the device (no host round trip).  g is clipped in place,
// like clip_grad_norm_ does.
__global__ void __launch_bounds__(256) adam_flat_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                        long long n, const long long* __restrict__ seg_end, const float* __restrict__ seg_lr, int nseg,
                                                        const float* __restrict__ norm, float b1, float b2, float eps, float wd, float bc1,
                                                        float bc2_sqrt) {
    const float coef = norm ? norm[1] : 1.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = nseg - 1;                       // first segment whose end is > i
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (seg_end[mid] > i) hi = mid; else lo = mid + 1; }
        const float lr = seg_lr[lo];
        float gg = g[i] * coef;
        g[i] = gg;
        if (lr <= 0.f) continue;
        const float ww = w[i];
        if (wd != 0.f) gg = fmaf(wd, ww, gg);
        const float mm = b1 * m[i] + (1.f - b1) * gg;
        const float vv = b2 * v[i] + (1.f - b2) * gg * gg;
        m[i] = mm; v[i] = vv;
        const float denom = sqrtf(vv) / bc2_sqrt + eps;
        w[i] = ww - (lr / bc1) * (mm / denom);
    }
}
// torch.optim.SGD (momentum mu, dampening 0, nesterov off) over the flat buffers, same segment layout / lr rule / in-place clipping as
// adam_flat_kernel.  torch keeps the momentum buffer per parameter and creates it on the tensor's first step (buf = d); seg_step[s] = the
// steps segment s has taken before this one (advanced by seg_step_advance_kernel after this launch).
__global__ void __launch_bounds__(256) sgd_flat_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ buf, long long n,
                                                       const long long* __restrict__ seg_end, const float* __restrict__ seg_lr,
                                                       const int* __restrict__ seg_step, int nseg, const float* __restrict__ norm, float mu,
                                                       float wd) {
    const float coef = norm ? norm[1] : 1.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = nseg - 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (seg_end[mid] > i) hi = mid; else lo = mid + 1; }
        const float lr = seg_lr[lo];
        float d = g[i] * coef;
        g[i] = d;
        if (lr <= 0.f) continue;
        const float ww = w[i];
        if (wd != 0.f) d = fmaf(wd, ww, d);
        const float b = seg_step[lo] == 0 ? d : fmaf(mu, buf[i], d);
        buf[i] = b;
        w[i] = ww - lr * b;
    }
}
// torch.optim.Adamax (single-tensor arithmetic): exp_avg m = b1 m + (1 - b1) d, exp_inf u = max(b2 u, |d| + eps),
// w -= lr / (1 - b1^t) * m / u with t the segment's own step count (seg_step[s] + 1).  Layout and idle rule as adam_flat_kernel.
__global__ void __launch_bounds__(256) adamax_flat_kernel(float* __restrict__ w, float* __restrict__ g, float* __restrict__ m, float* __restrict__ u,
                                                          long long n, const long long* __restrict__ seg_end, const float* __restrict__ seg_lr,
                                                          const int* __restrict__ seg_step, int nseg, const float* __restrict__ norm, float b1,
                                                          float b2, float eps, float wd) {
    const float coef = norm ? norm[1] : 1.f;
    int cur = -1;
    float clr = 0.f;                                     // lr / (1 - b1^t) of segment `cur`
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = nseg - 1;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (seg_end[mid] > i) hi = mid; else lo = mid + 1; }
        const float lr = seg_lr[lo];
        float d = g[i] * coef;
        g[i] = d;
        if (lr <= 0.f) continue;
        if (lo != cur) {                                 // torch: bias_correction = 1 - beta1 ** step in double
            cur = lo;
            clr = (float)((double)lr / (1.0 - pow((double)b1, (double)(seg_step[lo] + 1))));
        }
        const float ww = w[i];
        if (wd != 0.f) d = fmaf(wd, ww, d);
        const float mm = b1 * m[i] + (1.f - b1) * d;
        const float uu = fmaxf(b2 * u[i], fabsf(d) + eps);
        m[i] = mm; u[i] = uu;
        w[i] = ww - clr * (mm / uu);
    }
}
// seg_step[s] += 1 for every segment that stepped (lr > 0): after the update launch, so that all of it read the old count
__global__ void seg_step_advance_kernel(int* __restrict__ seg_step, const float* __restrict__ seg_lr, int nseg) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < nseg && seg_lr[s] > 0.f) seg_step[s] += 1;
}

// ---------------------------------------------------------------- dropout: counter-based masks (Philox4x32-10), nothing stored
// Element i of a tensor at dropout site `site` in optimisation step `step` draws word (i & 3) of Philox(counter = (i >> 2, site, step_lo,
// step_hi), key = seed): the backward regenerates the same mask from the same (seed, site, step) — no mask tensor, no RNG state.
// y = keep ? x / (1 - p) : 0 with keep = uniform >= p, uniform = (word >> 8) * 2^-24   (nn.Dropout / F.dropout train-mode arithmetic)
__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float p, float inv_keep, uint32_t seed_lo,
                               uint32_t seed_hi, uint32_t site, uint32_t step_lo, uint32_t step_hi) {
    const long long nq = (n + 3) >> 2;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (long long)gridDim.x * blockDim.x) {
        uint32_t r[4];
        philox4x32_10((uint32_t)q, site, step_lo ^ (uint32_t)(q >> 32), step_hi, seed_lo, seed_hi, r);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const long long i = q * 4 + e;
            if (i < n) y[i] = ((float)(r[e] >> 8) * (1.f / 16777216.f) >= p) ? x[i] * inv_keep : 0.f;
        }
    }
}

inline unsigned grid_for(long long n) { return (unsigned)(n <= 0 ? 1 : (n + TB - 1) / TB); }   // exact: several kernels are one element per thread

}  // namespace

#define ST(s) ((cudaStream_t)(s))
#define LAUNCH_OK() do { GVD_CHECK_LAUNCH(); return 0; } while (0)

extern "C" {
GVD_API int gvd_tr_ew(int op, const float* a, const float* b, const unsigned char* mask, float s, float* out, long long n, void* st) {
    GVD_REQUIRE(a && out && op >= 0 && op <= 5 && (((op > EW_MUL) && (op != EW_RELU_BWD)) || b) && (op != EW_MASKED_FILL || mask), "tr_ew: bad arguments (op %d)", op);
    if (n > 0) ew_kernel<<<grid_for(n), TB, 0, ST(st)>>>(op, a, b, mask, s, out, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_outer_rows(const float* a, const float* v, float* out, int B, int N, int H, void* st) {
    const long long total = (long long)B * N * H;
    outer_rows_kernel<<<grid_for(total), TB, 0, ST(st)>>>(a, v, out, N, H, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_outer_rows_acc(const float* a, const float* v, float* acc, int B, int N, int H, void* st) {
    GVD_REQUIRE(a && v && acc && H % 4 == 0, "tr_outer_rows_acc: H must be a multiple of 4");
    const long long total4 = (long long)B * N * (H / 4);
    outer_rows_acc_kernel<<<(unsigned)std::min<long long>(132 * 16, (total4 + TB - 1) / TB), TB, 0, ST(st)>>>(a, v, acc, N, H, total4);
    LAUNCH_OK();
}
GVD_API int gvd_tr_colsum(const float* x, float* out, int batch, long long M, int N, void* st) {
    const int nb = gvd_cdiv(N, 32);
    long long RB = std::min<long long>(std::max<long long>(1, 1056 / ((long long)nb * batch)), std::max<long long>(1, M / 64));
    if (RB <= 1) {
        colsum_kernel<<<dim3(nb, batch, 1), dim3(32, 8), 0, ST(st)>>>(x, out, M, N, M, 0);
        LAUNCH_OK();
    }
    const long long rpb = (M + RB - 1) / RB;
    RB = (M + rpb - 1) / rpb;
    float* part = nullptr;                                              // [RB][batch][N], stream-ordered scratch
    GVD_CHECK_CUDA(cudaMallocAsync(&part, (size_t)RB * batch * N * sizeof(float), ST(st)));
    colsum_kernel<<<dim3(nb, batch, (unsigned)RB), dim3(32, 8), 0, ST(st)>>>(x, part, M, N, rpb, (long long)batch * N);
    GVD_CHECK_LAUNCH();
    // phase 2: the partial rows of batch entry z are rows z, z + batch, ... of part viewed as [RB, batch * N]: one more column sum
    colsum_kernel<<<dim3(gvd_cdiv((long long)batch * N, 32), 1, 1), dim3(32, 8), 0, ST(st)>>>(part, out, RB, batch * N, RB, 0);
    GVD_CHECK_LAUNCH();
    GVD_CHECK_CUDA(cudaFreeAsync(part, ST(st)));
    return 0;
}
GVD_API int gvd_tr_rowsum(const float* x, float* out, long long M, int N, void* st) {
    rowsum_kernel<<<(unsigned)M, TB, 0, ST(st)>>>(x, out, N);
    LAUNCH_OK();
}
GVD_API int gvd_tr_sum_all(const float* x, float* out, long long n, void* st) {
    sum_all_kernel<<<1, 1024, 0, ST(st)>>>(x, out, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_mean_dim1(const float* x, float* out, int B, int T, int F, void* st) {
    const long long total = (long long)B * F;
    mean_dim1_kernel<<<grid_for(total), TB, 0, ST(st)>>>(x, out, T, F, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_ln_fwd(const float* x, float* y, long long rows, int n, void* st) { ln_fwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(x, y, n); LAUNCH_OK(); }
GVD_API int gvd_tr_ln_bwd(const float* dy, const float* y, const float* x, float* dx, long long rows, int n, void* st) {
    ln_bwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(dy, y, x, dx, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_ln_star_fwd(const float* x, const float* g, const float* b, float* y, long long rows, int n, void* st) {
    ln_star_fwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(x, g, b, y, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_ln_star_bwd(const float* dy, const float* x, const float* g, float* dx, float* tmp, long long rows, int n, void* st) {
    ln_star_bwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(dy, x, g, dx, tmp, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_softmax_fwd(const float* x, float scale, float* p, long long rows, int n, void* st) {
    softmax_fwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(x, scale, p, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_softmax_bwd(const float* dp, const float* p, float scale, float* dx, long long rows, int n, void* st) {
    softmax_bwd_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(dp, p, scale, dx, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_count_inv(const void* data, long long n, int elem_bytes, float* inv_out, void* st) {
    GVD_REQUIRE(data && inv_out && (elem_bytes == 1 || elem_bytes == 4) && n >= 0, "tr_count_inv: bad arguments");
    count_inv_kernel<<<1, 1024, 0, ST(st)>>>(data, n, elem_bytes, inv_out, nullptr, nullptr);
    LAUNCH_OK();
}
GVD_API int gvd_tr_scalar_mul(const float* a, const float* b, float* out, void* st) {
    scalar_mul_kernel<<<1, 1, 0, ST(st)>>>(a, b, out);
    LAUNCH_OK();
}
GVD_API int gvd_tr_lm_nll(const float* logits, const int64_t* target, const unsigned char* mask, const float* inv_n, float* rowloss, float* dlogits,
                          long long rows, int n, void* st) {
    lm_nll_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(logits, (const long long*)target, mask, inv_n, rowloss, dlogits, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_pos_nll(const float* x, const unsigned char* pos, const float* inv_n, float* rowloss, float* dx, long long rows, int n, void* st) {
    pos_nll_kernel<<<(unsigned)rows, TB, 0, ST(st)>>>(x, pos, inv_n, rowloss, dx, n);
    LAUNCH_OK();
}
GVD_API int gvd_tr_cls_nll(const float* simT, const int* target, const float* inv_n, float* part, float* dsimT, int B, int R, int NB, int C, void* st) {
    const long long total = (long long)B * NB * R;
    GVD_CHECK_CUDA(cudaMemsetAsync(dsimT, 0, (size_t)B * R * C * sizeof(float), ST(st)));
    cls_nll_kernel<<<grid_for(total), TB, 0, ST(st)>>>(simT, target, inv_n, part, dsimT, R, NB, C, total);
    LAUNCH_OK();
}
// IoU + class targets + per-step RoI labels / frame masks of the teacher forcing (utils.py:293-328, model.py:345-347,436-440)
GVD_API int gvd_tr_targets(const float* ppls, const float* gt_boxes, const unsigned char* frm_mask, const unsigned char* pnt_mask,
                           const unsigned char* mask_boxes, int B, int R, int NB, int S, int L1, float* ov, int* cls_target,
                           unsigned char* labels, unsigned char* fm, void* st) {
    GVD_REQUIRE(ppls && gt_boxes && frm_mask && pnt_mask && mask_boxes && ov && cls_target && labels && fm, "tr_targets: null argument");
    GVD_TRY(gvd_bbox_overlaps(ppls, gt_boxes, frm_mask, pnt_mask, ov, B, R, NB, ST(st)));
    const long long total = (long long)B * NB * R;
    class_target_kernel<<<grid_for(total), TB, 0, ST(st)>>>(ov, gt_boxes, cls_target, R, NB, total);
    GVD_CHECK_LAUNCH();
    return gvd_step_targets(ov, mask_boxes, frm_mask, pnt_mask, labels, fm, B, S, R, NB, L1, ST(st));
}
GVD_API int gvd_tr_lstm_cell_fwd(const float* gates, const float* c, float* h2, float* c2, float* act, int B, int H, void* st) {
    const long long total = (long long)B * H;
    lstm_cell_fwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(gates, c, h2, c2, act, H, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_lstm_cell_bwd(const float* dh2, const float* dc2, const float* act, const float* c, const float* c2, float* dgates, float* dc,
                                 int B, int H, void* st) {
    const long long total = (long long)B * H;
    lstm_cell_bwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(dh2, dc2, act, c, c2, dgates, dc, H, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_gru_cell_fwd(const float* gi, const float* gh, const float* h, float* h2, float* r, float* z, float* n, int B, int G, void* st) {
    const long long total = (long long)B * G;
    gru_cell_fwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(gi, gh, h, h2, r, z, n, G, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_gru_cell_bwd(const float* dh, const float* r, const float* z, const float* n, const float* h, const float* ghn, float* dgi,
                                float* dgh, float* dh_keep, int B, int G, void* st) {
    const long long total = (long long)B * G;
    gru_cell_bwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(dh, r, z, n, h, ghn, dgi, dgh, dh_keep, G, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_att_scores_fwd(const float* p, const float* q, const float* w, const float* bias, float* s, int B, int N, int A, void* st) {
    const long long rows = (long long)B * N;
    att_scores_fwd_kernel<<<gvd_cdiv(rows * 32, TB), TB, 0, ST(st)>>>(p, q, w, bias, s, N, A, rows);
    LAUNCH_OK();
}
GVD_API int gvd_tr_att_scores_bwd(const float* ds, const float* p, const float* q, const float* w, float* dpre, float* dst, int B, int N, int A, void* st) {
    const long long total = (long long)B * N * A;
    att_scores_bwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(ds, p, q, w, dpre, dst, N, A, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_att_scores_mul_fwd(const float* p, const float* q, const float* w, const float* bias, float* s, int B, int N, int A, void* st) {
    GVD_REQUIRE(p && q && w && bias && s, "tr_att_scores_mul_fwd: null argument");
    const long long rows = (long long)B * N;
    att_scores_mul_fwd_kernel<<<gvd_cdiv(rows * 32, TB), TB, 0, ST(st)>>>(p, q, w, bias, s, N, A, rows);
    LAUNCH_OK();
}
GVD_API int gvd_tr_att_scores_mul_bwd(const float* ds, const float* p, const float* q, const float* w, float* dp, float* dqt, float* dst, int B, int N,
                                      int A, void* st) {
    GVD_REQUIRE(ds && p && q && w && dp && dqt && dst, "tr_att_scores_mul_bwd: null argument");
    const long long total = (long long)B * N * A;
    att_scores_mul_bwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(ds, p, q, w, dp, dqt, dst, N, A, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_gather_rows(const float* table, const int64_t* idx, float* out, long long M, int D, void* st) {
    const long long total = M * D;
    gather_rows_kernel<<<grid_for(total), TB, 0, ST(st)>>>(table, (const long long*)idx, out, D, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_index_add_rows(const int64_t* idx, const float* rows, float* out, int n_rows, int M, int D, void* st) {
    index_add_rows_kernel<<<n_rows, TB, 0, ST(st)>>>((const long long*)idx, rows, out, M, D);
    LAUNCH_OK();
}
GVD_API int gvd_tr_bn_normalize(const float* e, const float* mu, const float* var, float* out, long long M, int N, void* st) {
    const long long total = M * N;
    bn_normalize_kernel<<<grid_for(total), TB, 0, ST(st)>>>(e, mu, var, out, N, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_bn_bwd(const float* dxh, const float* e_hat, const float* var, const float* s1, const float* s2, float* de, long long M, int N,
                          void* st) {
    const long long total = M * N;
    bn_bwd_kernel<<<grid_for(total), TB, 0, ST(st)>>>(dxh, e_hat, var, s1, s2, 1.f / (float)M, de, N, total);
    LAUNCH_OK();
}
GVD_API int gvd_tr_adam_first_step(const float* w, const float* g, float coef, float lr, float b1, float b2, float eps, float* out, long long n,
                                   void* st) {
    adam_first_step_kernel<<<grid_for(n), TB, 0, ST(st)>>>(w, g, coef, lr, b1, b2, eps, out, n);
    LAUNCH_OK();
}


// Dropout with a regenerable mask (see dropout_kernel): y may alias x.  The same call on the upstream gradient is the backward.
GVD_API int gvd_tr_dropout(const float* x, float* y, long long n, float p, long long seed, int site, long long step, void* st) {
    GVD_REQUIRE(x && y && n >= 0 && p >= 0.f && p < 1.f, "tr_dropout: bad arguments (p = %f)", (double)p);
    if (n == 0) return 0;
    const unsigned grid = (unsigned)std::min<long long>(132 * 16, (((n + 3) >> 2) + TB - 1) / TB);
    dropout_kernel<<<grid, TB, 0, ST(st)>>>(x, y, n, p, 1.f / (1.f - p), (uint32_t)(seed & 0xffffffffll), (uint32_t)((unsigned long long)seed >> 32),
                                            (uint32_t)site, (uint32_t)(step & 0xffffffffll), (uint32_t)((unsigned long long)step >> 32));
    LAUNCH_OK();
}
// Global L2 norm of the flat gradient buffer + clip coefficient, on the device: norm_out[0] = ||g||, norm_out[1] = min(max_norm/(||g||+1e-6), 1)
// (torch.nn.utils.clip_grad_norm_, main.py:265).  scratch: >= gvd_tr_sumsq_scratch_bytes() bytes.
GVD_API size_t gvd_tr_sumsq_scratch_bytes(void) { return (size_t)SQ_BLOCKS * sizeof(double); }
GVD_API int gvd_tr_grad_norm(const float* g, long long n, float max_norm, void* scratch, float* norm_out, void* st) {
    GVD_REQUIRE(g && scratch && norm_out && n > 0 && ((uintptr_t)g & 15) == 0, "tr_grad_norm: bad arguments");
    sumsq_partial_kernel<<<SQ_BLOCKS, 256, 0, ST(st)>>>(g, n, (double*)scratch);
    GVD_CHECK_LAUNCH();
    sumsq_finish_kernel<<<1, 256, 0, ST(st)>>>((const double*)scratch, SQ_BLOCKS, max_norm, norm_out);
    LAUNCH_OK();
}
// One Adam step (step count t >= 1) on the flat buffers; see adam_flat_kernel.  norm = the output of gvd_tr_grad_norm (or null: no clipping).
GVD_API int gvd_tr_adam_flat(float* w, float* g, float* m, float* v, long long n, const int64_t* seg_end, const float* seg_lr, int nseg,
                             const float* norm, float b1, float b2, float eps, float weight_decay, int t, void* st) {
    GVD_REQUIRE(w && g && m && v && seg_end && seg_lr && nseg >= 1 && n > 0 && t >= 1, "tr_adam_flat: bad arguments");
    const float bc1 = (float)(1.0 - pow((double)b1, (double)t)), bc2s = (float)sqrt(1.0 - pow((double)b2, (double)t));
    adam_flat_kernel<<<132 * 8, 256, 0, ST(st)>>>(w, g, m, v, n, (const long long*)seg_end, seg_lr, nseg, norm, b1, b2, eps, weight_decay, bc1, bc2s);
    LAUNCH_OK();
}
// One SGD-with-momentum step on the flat buffers (see sgd_flat_kernel), then seg_step[s] += 1 for the segments with lr > 0.
GVD_API int gvd_tr_sgd_flat(float* w, float* g, float* buf, long long n, const int64_t* seg_end, const float* seg_lr, int* seg_step, int nseg,
                            const float* norm, float momentum, float weight_decay, void* st) {
    GVD_REQUIRE(w && g && buf && seg_end && seg_lr && seg_step && nseg >= 1 && n > 0, "tr_sgd_flat: bad arguments");
    sgd_flat_kernel<<<132 * 8, 256, 0, ST(st)>>>(w, g, buf, n, (const long long*)seg_end, seg_lr, seg_step, nseg, norm, momentum, weight_decay);
    GVD_CHECK_LAUNCH();
    seg_step_advance_kernel<<<gvd_cdiv(nseg, TB), TB, 0, ST(st)>>>(seg_step, seg_lr, nseg);
    LAUNCH_OK();
}
// One Adamax step on the flat buffers (see adamax_flat_kernel), then seg_step[s] += 1 for the segments with lr > 0.
GVD_API int gvd_tr_adamax_flat(float* w, float* g, float* m, float* u, long long n, const int64_t* seg_end, const float* seg_lr, int* seg_step,
                               int nseg, const float* norm, float b1, float b2, float eps, float weight_decay, void* st) {
    GVD_REQUIRE(w && g && m && u && seg_end && seg_lr && seg_step && nseg >= 1 && n > 0, "tr_adamax_flat: bad arguments");
    adamax_flat_kernel<<<132 * 8, 256, 0, ST(st)>>>(w, g, m, u, n, (const long long*)seg_end, seg_lr, seg_step, nseg, norm, b1, b2, eps, weight_decay);
    GVD_CHECK_LAUNCH();
    seg_step_advance_kernel<<<gvd_cdiv(nseg, TB), TB, 0, ST(st)>>>(seg_step, seg_lr, nseg);
    LAUNCH_OK();
}
// C[z] = A[z] W[z]^T  (A [batch, M, K], W [batch, N, K], C [batch, M, N]; row pitches lda / ldw / ldc, batch strides in elements)
GVD_API int gvd_tr_gemm_nt_batched(const float* A, long long lda, long long sA, const float* W, long long ldw, long long sW, float* C, long long ldc,
                                   long long sC, int M, int N, int K, int batch, void* st) {
    GVD_REQUIRE(A && W && C && batch >= 1, "tr_gemm_nt_batched: bad arguments");
    GemmArgs g{};
    g.A = A; g.lda = lda; g.sAb = sA; g.W = W; g.ldw = ldw; g.sWb = sW; g.C = C; g.ldc = ldc; g.sCb = sC;
    g.M = M; g.N = N; g.K = K; g.nh = 1; g.act = GVD_ACT_NONE; g.alpha = 1.f;
    return gvd_gemm_nt(g, batch, ST(st));
}
// out[z][c][r] = in[z][r][c]
GVD_API int gvd_tr_transpose(const float* in, float* out, int batch, int R, int C, void* st) { return gvd_transpose(in, out, batch, R, C, C, ST(st)); }
}  // extern "C"
