// Persistent bidirectional GRU layer (model.py:150-154,562: nn.GRU(H, H/2, 2, bidirectional=True); SURVEY 8 row P7).
//
// Run as launches per time step the recurrence needs thousands of launches per batch at the reference default T = 480.  Here ONE cooperative launch runs a
// whole layer (both directions): CTA (c, d) owns 8 hidden units of direction d and keeps its 24 rows of W_hh (r, z, n gates) in
// shared memory for all T steps; per step it computes gh = W_hh h(t-1) + b_hh for its units and every clip (fp32 FFMA, h staged through
// shared memory in K chunks), applies the gate math, writes h(t) to a ping-pong global buffer and the layer output row, then meets
// the other CTAs of ITS direction at a device-scope barrier (one counter per direction; the two directions never wait for each other).
#include <cooperative_groups.h>

#include "gvd_common.cuh"
#include "gvd_kernels.cuh"

namespace {

constexpr int GRU_UPC = 8;                  // hidden units per CTA
constexpr int GRU_ROWS = 3 * GRU_UPC;       // W_hh rows per CTA (gate-major: row = gate * UPC + unit)
constexpr int GRU_KC = 128;                 // K chunk of h staged in shared memory
constexpr int GRU_BT = 128;                 // clips per pass
constexpr int GRU_THREADS = 256;
constexpr int GRU_HP = GRU_KC + 4;          // padded row pitch of the h tile (conflict-free 128-bit reads)

struct GruArgs {
    const float* gi;            // [B, T, 6G]  W_ih x + b_ih, direction d at column offset d * 3G
    const float* whh;           // [2][3G][G]
    const float* bhh;           // [2][3G]
    float* hbuf;                // [2 parity][2 dir][B][G], zero-initialised
    float* out;                 // [B, T, 2G]
    const long long* sample_idx;   // optional [B, 2]: rows outside [lo, hi) are written as zeros (model.py:505-507,564)
    unsigned int* bar;          // [2] zero-initialised arrival counters (one per direction)
    int B, T, G;
};

__global__ void __launch_bounds__(GRU_THREADS, 1) gru_layer_kernel(const GruArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int G = a.G, B = a.B, T = a.T;
    const int WP = G + 4;                                    // pitch of the W rows
    float* Ws = sm;                                          // [24][WP]
    float* bs = Ws + GRU_ROWS * WP;                          // [24] (+8 pad)
    float* hs = bs + 32;                                     // [GRU_BT][GRU_HP]
    float* ghs = hs + 2 * GRU_BT * GRU_HP;                   // [GRU_BT][25]   (hs: two staging buffers)
    const int tid = threadIdx.x;
    const int d = blockIdx.y, u0 = blockIdx.x * GRU_UPC;
    const int nu = min(GRU_UPC, G - u0);
    const int ncta = gridDim.x;
    const float* whh = a.whh + (size_t)d * 3 * G * G;
    const float* bhh = a.bhh + (size_t)d * 3 * G;
    for (int i = tid; i < GRU_ROWS * (G / 4); i += GRU_THREADS) {
        const int r = i / (G / 4), k4 = i % (G / 4);
        const int gate = r / GRU_UPC, u = r % GRU_UPC;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (u < nu) v = __ldg(reinterpret_cast<const float4*>(whh + ((size_t)gate * G + u0 + u) * G) + k4);
        *reinterpret_cast<float4*>(Ws + r * WP + 4 * k4) = v;
    }
    if (tid < GRU_ROWS) {
        const int gate = tid / GRU_UPC, u = tid % GRU_UPC;
        bs[tid] = u < nu ? __ldg(bhh + gate * G + u0 + u) : 0.f;
    }
    __syncthreads();
    const int bl = tid & 63, q = tid >> 6;                   // this thread: clips bl and bl + 64 of the pass, rows [6q, 6q + 6)
    const size_t BG = (size_t)B * G;
    const int nchunk = (G + GRU_KC - 1) / GRU_KC;
    float* hs2[2] = {hs, hs + GRU_BT * GRU_HP};
    // asynchronous copy of one K chunk of h(t-1) for the clips [b0, b0 + nb): 16-byte cp.async.cg (L2 only: the rows were written by other SMs)
    auto stage = [&](const float* h_prev, int b0, int nb, int c, float* dst) {
        const int k0 = c * GRU_KC, kc4 = min(GRU_KC, G - k0) >> 2;
        for (int i = tid; i < nb * kc4; i += GRU_THREADS) {
            const int b = i / kc4, k4 = i % kc4;
            const unsigned sa = (unsigned)__cvta_generic_to_shared(dst + b * GRU_HP + 4 * k4);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(h_prev + (size_t)(b0 + b) * G + k0 + 4 * k4) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (int s = 0; s < T; ++s) {
        const int t = d ? (T - 1 - s) : s;
        const float* h_prev = a.hbuf + ((size_t)(s & 1) * 2 + d) * BG;
        float* h_new = a.hbuf + ((size_t)((s + 1) & 1) * 2 + d) * BG;
        for (int b0 = 0; b0 < B; b0 += GRU_BT) {
            const int nb = min(GRU_BT, B - b0);
            float acc0[6], acc1[6];
#pragma unroll
            for (int r = 0; r < 6; ++r) acc0[r] = acc1[r] = 0.f;
            if (s > 0) {                                     // h(-1) = 0: the first step's recurrent term is the bias alone
                __syncthreads();                             // the previous pass no longer reads the staging buffers
                stage(h_prev, b0, nb, 0, hs2[0]);
                for (int c = 0; c < nchunk; ++c) {
                    if (c + 1 < nchunk) {
                        stage(h_prev, b0, nb, c + 1, hs2[(c + 1) & 1]);          // next chunk in flight while this one is multiplied
                        asm volatile("cp.async.wait_group 1;" ::: "memory");
                    } else {
                        asm volatile("cp.async.wait_group 0;" ::: "memory");
                    }
                    __syncthreads();
                    const int k0 = c * GRU_KC, kc4 = min(GRU_KC, G - k0) >> 2;
                    const float* hA = hs2[c & 1] + bl * GRU_HP;
                    const float* hB = hs2[c & 1] + (bl + 64) * GRU_HP;
                    const float* wr = Ws + (6 * q) * WP + k0;
#pragma unroll 4
                    for (int k4 = 0; k4 < kc4; ++k4) {
                        const float4 x = *reinterpret_cast<const float4*>(hA + 4 * k4);
                        const float4 y = *reinterpret_cast<const float4*>(hB + 4 * k4);
#pragma unroll
                        for (int r = 0; r < 6; ++r) {
                            const float4 w = *reinterpret_cast<const float4*>(wr + r * WP + 4 * k4);   // warp-wide broadcast
                            acc0[r] = fmaf(x.x, w.x, acc0[r]); acc0[r] = fmaf(x.y, w.y, acc0[r]);
                            acc0[r] = fmaf(x.z, w.z, acc0[r]); acc0[r] = fmaf(x.w, w.w, acc0[r]);
                            acc1[r] = fmaf(y.x, w.x, acc1[r]); acc1[r] = fmaf(y.y, w.y, acc1[r]);
                            acc1[r] = fmaf(y.z, w.z, acc1[r]); acc1[r] = fmaf(y.w, w.w, acc1[r]);
                        }
                    }
                    __syncthreads();                         // chunk consumed: its buffer may be refilled two iterations later
                }
            }
            // rows of clips >= nb in the staging buffers hold stale data of earlier passes: their sums are never read below
#pragma unroll
            for (int r = 0; r < 6; ++r) {
                ghs[bl * 25 + 6 * q + r] = acc0[r] + bs[6 * q + r];
                ghs[(bl + 64) * 25 + 6 * q + r] = acc1[r] + bs[6 * q + r];
            }
            __syncthreads();
            // gate math: r, z, n order, b_hn inside the r product (torch.nn.GRU); one item = (clip, unit)
            for (int i = tid; i < nb * GRU_UPC; i += GRU_THREADS) {
                const int b = i / GRU_UPC, u = i % GRU_UPC;
                if (u >= nu) continue;
                const int bb = b0 + b, j = u0 + u;
                const float* gir = a.gi + ((size_t)bb * T + t) * (6 * G) + (size_t)d * 3 * G;
                const float g_r = __ldg(gir + j), g_z = __ldg(gir + G + j), g_n = __ldg(gir + 2 * G + j);
                const float hp = s > 0 ? __ldcg(h_prev + (size_t)bb * G + j) : 0.f;
                const float hr = ghs[b * 25 + u], hz = ghs[b * 25 + GRU_UPC + u], hn = ghs[b * 25 + 2 * GRU_UPC + u];
                const float rg = sigmoid_acc(g_r + hr);
                const float zg = sigmoid_acc(g_z + hz);
                const float ng = tanhf(g_n + rg * hn);
                const float h = (1.f - zg) * ng + zg * hp;
                h_new[(size_t)bb * G + j] = h;
                float o = h;
                if (a.sample_idx) {
                    const long long lo = a.sample_idx[2 * bb], hi = a.sample_idx[2 * bb + 1];
                    if (t < lo || t >= hi) o = 0.f;
                }
                a.out[((size_t)bb * T + t) * (2 * G) + (size_t)d * G + j] = o;
            }
        }
        if (s + 1 < T) {
            // barrier among the CTAs of this direction: h(t) of every unit is visible before anyone starts step t + 1
            // (CTA barrier, then ONE thread fences at device scope, arrives and polls: the cooperative-groups grid.sync pattern)
            __syncthreads();
            if (tid == 0) {
                __threadfence();
                atomicAdd(a.bar + d, 1u);
                const unsigned int target = (unsigned int)ncta * (unsigned int)(s + 1);
                unsigned int v;
                do {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.bar + d) : "memory");
                } while (v < target);
                __threadfence();
            }
            __syncthreads();
        }
    }
}

size_t gru_smem_bytes(int G) { return (size_t)(GRU_ROWS * (G + 4) + 32 + 2 * GRU_BT * GRU_HP + GRU_BT * 25) * sizeof(float); }

}  // namespace

// One bidirectional GRU layer in one cooperative launch.  Returns 1 (with the error text set) when the shape is not supported, so the
// caller can keep the per-step path: G % 4 == 0, shared memory for 24 rows of W_hh, all CTAs co-resident.
int gvd_gru_layer(const float* gi, const float* whh, const float* bhh, float* hbuf, float* out, const long long* sample_idx, unsigned int* bar,
                  int B, int T, int G, cudaStream_t st) {
    GVD_REQUIRE(gi && whh && bhh && hbuf && out && bar && B >= 1 && T >= 1 && G >= 4 && G % 4 == 0, "gru_layer: bad arguments");
    const size_t smem = gru_smem_bytes(G);
    GVD_REQUIRE(smem <= 227 * 1024, "gru_layer: G = %d needs %zu bytes of shared memory", G, smem);
    static int max_ctas = -1;
    GVD_CHECK_CUDA(cudaFuncSetAttribute(gru_layer_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (max_ctas < 0) {
        int dev = 0, sms = 0, per_sm = 0;
        GVD_CHECK_CUDA(cudaGetDevice(&dev));
        GVD_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        GVD_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gru_layer_kernel, GRU_THREADS, smem));
        max_ctas = sms * per_sm;
    }
    const int ncta = gvd_cdiv(G, GRU_UPC);
    GVD_REQUIRE(2 * ncta <= max_ctas, "gru_layer: %d CTAs cannot be co-resident (max %d)", 2 * ncta, max_ctas);
    GVD_CHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned int), st));
    GVD_CHECK_CUDA(cudaMemsetAsync(hbuf, 0, (size_t)2 * 2 * B * G * sizeof(float), st));
    GruArgs a{gi, whh, bhh, hbuf, out, sample_idx, bar, B, T, G};
    void* params[] = {(void*)&a};
    GVD_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)gru_layer_kernel, dim3(ncta, 2), dim3(GRU_THREADS), params, smem, st));
    gvd_count_launch();
    return 0;
}
