// gvd-b200: row-wise prologue kernels (means, LayerNorms, softmax over classes, transposes,
// GRU pointwise).  All HBM-bound, one pass over their inputs, coalesced along the feature dim.
#include <algorithm>

#include "gvd_kernels.cuh"

namespace {

// ---------------------------------------------------------------- mean over frames
// fc = mean_t segs_feat[b,t,:] over ALL T rows (model.py:508; padding rows included, quirk Q6)
__global__ void frame_mean_kernel(const float* __restrict__ segs, float* __restrict__ out, int T, int C) {
    const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float* p = segs + (long long)b * T * C + c;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int t = 0;
    for (; t + 3 < T; t += 4) {
        s0 += __ldg(p + (long long)(t + 0) * C);
        s1 += __ldg(p + (long long)(t + 1) * C);
        s2 += __ldg(p + (long long)(t + 2) * C);
        s3 += __ldg(p + (long long)(t + 3) * C);
    }
    for (; t < T; ++t) s0 += __ldg(p + (long long)t * C);
    out[(long long)b * C + c] = ((s0 + s1) + (s2 + s3)) / (float)T;
}

// ---------------------------------------------------------------- clip vector assembly
// xcat[b] = [ LN_C(fc) | LN_50(ReLU(W_seg . float(num[b,3:7]) + b_seg)) | 0-pad ]   (model.py:509-510)
// rows (optional): clip b's mean is fc_mean row rows[b] (video-indexed batches: one mean per video)
__global__ void clip_vector_kernel(const float* __restrict__ fc_mean, const long long* __restrict__ num,
                                   const float* __restrict__ Wseg, const float* __restrict__ bseg,
                                   float* __restrict__ xcat, int C, int S, int ld, const long long* __restrict__ rows) {
    __shared__ float red[32];
    __shared__ float seg[64];
    const int b = blockIdx.x;
    const float* x = fc_mean + (rows ? rows[b] : (long long)b) * C;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) s += x[c];
    const float mu = block_sum(s, red) / (float)C;
    float v = 0.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) { const float d = x[c] - mu; v += d * d; }
    const float rstd = 1.f / sqrtf(block_sum(v, red) / (float)C + 1e-5f);
    float* o = xcat + (long long)b * ld;
    for (int c = threadIdx.x; c < C; c += blockDim.x) o[c] = (x[c] - mu) * rstd;
    // segment-info embedding: num is int64 at this boundary, so the start/end fractions are
    // already truncated (main.py:572; quirk Q7)
    if (threadIdx.x < S) {
        float a = bseg[threadIdx.x];
#pragma unroll
        for (int q = 0; q < 4; ++q) a = fmaf(Wseg[threadIdx.x * 4 + q], (float)num[(long long)b * 7 + 3 + q], a);
        seg[threadIdx.x] = fmaxf(a, 0.f);
    }
    __syncthreads();
    const float sv = threadIdx.x < S ? seg[threadIdx.x] : 0.f;
    const float smu = block_sum(sv, red) / (float)S;
    const float sd = threadIdx.x < S ? (sv - smu) : 0.f;
    const float srstd = 1.f / sqrtf(block_sum(sd * sd, red) / (float)S + 1e-5f);
    if (threadIdx.x < S) o[C + threadIdx.x] = sd * srstd;
    for (int c = C + S + threadIdx.x; c < ld; c += blockDim.x) o[c] = 0.f;
}

// ---------------------------------------------------------------- region-class softmax
// rows of simT[(b,r), 0..NC) : masked proposal -> all -1e8 (model.py:278), softmax over classes (:535)
__global__ void sim_softmax_kernel(float* __restrict__ simT, const unsigned char* __restrict__ pnt_mask, int rows, int R,
                                   int NC, int ld) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int b = warp / R, r = warp % R;
    float* x = simT + (long long)warp * ld;
    const bool masked = pnt_mask[(long long)b * (R + 1) + 1 + r] != 0;
    float m = -INFINITY;
    for (int c = lane; c < NC; c += 32) m = fmaxf(m, masked ? GVD_MIN_VALUE : x[c]);
    m = warp_max(m);
    float s = 0.f;
    for (int c = lane; c < NC; c += 32) s += expf((masked ? GVD_MIN_VALUE : x[c]) - m);
    s = warp_sum(s);
    for (int c = lane; c < NC; c += 32) x[c] = expf((masked ? GVD_MIN_VALUE : x[c]) - m) / s;
}

// ---------------------------------------------------------------- batched transpose  in[b][r][c] -> out[b][c][r]
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int C, int ld_in) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < R && c < C) ? in[((long long)b * R + r) * ld_in + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < C) out[((long long)b * C + c) * R + r] = tile[threadIdx.x][i];
    }
}

// in[b][r][c] -> hi[b][c][r], lo[b][c][r]: the transposed operand already split into its tf32 planes (x = hi + lo), so the
// tensor-core kernels that stream it as the smem operand do no conversion work of their own
__global__ void transpose_split_kernel(const float* __restrict__ in, float* __restrict__ hi, float* __restrict__ lo, int R, int C, int ld_in) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < R && c < C) ? in[((long long)b * R + r) * ld_in + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < C) {
            const float x = tile[threadIdx.x][i], h = tf32_rna(x);
            const long long o = ((long long)b * C + c) * R + r;
            hi[o] = h;
            lo[o] = x - h;
        }
    }
}
// fp16x3 operand images for the fused self-attention (gvd_common.cuh):
// per (row, head) the hs (<= KH) columns of that head, padded with zeros to KH = 32-multiple words:  out[(row * nh + h) * KH + word]
__global__ void pack_heads_f16x3_kernel(const float* __restrict__ in, long long ld_in, long long rows, int nh, int hs_in, int hs, int KH, float scale,
                                        uint32_t* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;       // (row, head, pair)
    const int per = KH / 2;
    if (i >= rows * nh * per) return;
    const int pr = (int)(i % per), h = (int)((i / per) % nh);
    const long long r = i / ((long long)per * nh);
    const int k = 2 * pr;
    const float* src = in + r * ld_in + (long long)h * hs_in;
    uint32_t hi, lo;
    f16x3_split_pair(k < hs ? src[k] : 0.f, k + 1 < hs ? src[k + 1] : 0.f, scale, hi, lo);
    uint32_t* dst = out + (r * nh + h) * KH + (k >> 5) * 32 + ((k & 31) >> 1);
    dst[0] = hi; dst[16] = lo;
}
// in[b][r][c] -> image of the transposed matrix: out[(b * C + c) * Rp + word(r)], Rp = 32-multiple >= R (zero padded)
__global__ void transpose_pack_f16x3_kernel(const float* __restrict__ in, uint32_t* __restrict__ out, int R, int C, int ld_in, int Rp, float scale) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < R && c < C) ? in[((long long)b * R + r) * ld_in + c] : 0.f;
    }
    __syncthreads();
    const int lane = threadIdx.x, pr = lane & 15;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i;
        if (c < C) {
            uint32_t hi, lo;
            f16x3_split_pair(tile[2 * pr][i], tile[2 * pr + 1][i], scale, hi, lo);
            out[((long long)b * C + c) * Rp + r0 + lane] = lane < 16 ? hi : lo;       // one K slice: 16 hi words then 16 lo words
        }
    }
}
// rows x cols (cols % 4 == 0) -> tf32 hi / lo planes with the same row pitch
__global__ void split_hilo_kernel(const float* __restrict__ in, long long ld_in, float* __restrict__ hi, float* __restrict__ lo, long long ld_out,
                                  long long rows, int cols4) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols4) return;
    const long long r = i / cols4;
    const int c = (int)(i % cols4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(in + r * ld_in + c);
    float4 h, l;
    h.x = tf32_rna(v.x); h.y = tf32_rna(v.y); h.z = tf32_rna(v.z); h.w = tf32_rna(v.w);
    l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
    *reinterpret_cast<float4*>(hi + r * ld_out + c) = h;
    *reinterpret_cast<float4*>(lo + r * ld_out + c) = l;
}

// ---------------------------------------------------------------- region embedding input
// row (b,r): [ LN_F(g) | LN_300(ReLU(W_loc . loc_in + b_loc)) | LN_NC(simT row) | 0-pad ]   (model.py:537-544)
// loc_in = (x1,y1,x2,y2)/720, frame/num_sampled_frm
template <int NT>
__global__ void __launch_bounds__(NT)
pool_in_kernel(const float* __restrict__ g, const float* __restrict__ ppls, const float* __restrict__ simT,
               const float* __restrict__ Wloc, const float* __restrict__ bloc, float* __restrict__ out, int F, int NL,
               int NC, int ld_sim, int ld_out, float inv_frames, uint32_t* __restrict__ img, int ld_img, float img_scale) {
    __shared__ float red[32];
    __shared__ float loc_in[5];
    extern __shared__ __align__(16) float rowbuf[];             // the assembled row (ld_img >= ld_out floats): written once, then stored as fp32 and / or image
    const long long row = blockIdx.x;
    float* o = rowbuf;
    // --- LN over the fc7 feature
    const float* x = g + row * F;
    float s = 0.f;
    for (int c = threadIdx.x; c < F; c += NT) s += x[c];
    float mu = block_sum(s, red) / (float)F;
    float v = 0.f;
    for (int c = threadIdx.x; c < F; c += NT) { const float d = x[c] - mu; v += d * d; }
    float rstd = 1.f / sqrtf(block_sum(v, red) / (float)F + 1e-5f);
    for (int c = threadIdx.x; c < F; c += NT) o[c] = (x[c] - mu) * rstd;
    // --- location embedding
    if (threadIdx.x < 4) loc_in[threadIdx.x] = ppls[row * 7 + threadIdx.x] / 720.f;
    if (threadIdx.x == 4) loc_in[4] = ppls[row * 7 + 4] * inv_frames;
    __syncthreads();
    float lv[4];   // NL <= 4*NT
    s = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int j = threadIdx.x + q * NT;
        lv[q] = 0.f;
        if (j < NL) {
            float a = bloc[j];
#pragma unroll
            for (int k = 0; k < 5; ++k) a = fmaf(Wloc[j * 5 + k], loc_in[k], a);
            lv[q] = fmaxf(a, 0.f);
            s += lv[q];
        }
    }
    mu = block_sum(s, red) / (float)NL;
    v = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (threadIdx.x + q * NT < NL) { const float d = lv[q] - mu; v += d * d; }
    rstd = 1.f / sqrtf(block_sum(v, red) / (float)NL + 1e-5f);
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (threadIdx.x + q * NT < NL) o[F + threadIdx.x + q * NT] = (lv[q] - mu) * rstd;
    // --- LN over the class distribution
    const float* p = simT + row * ld_sim;
    s = 0.f;
    for (int c = threadIdx.x; c < NC; c += NT) s += p[c];
    mu = block_sum(s, red) / (float)NC;
    v = 0.f;
    for (int c = threadIdx.x; c < NC; c += NT) { const float d = p[c] - mu; v += d * d; }
    rstd = 1.f / sqrtf(block_sum(v, red) / (float)NC + 1e-5f);
    for (int c = threadIdx.x; c < NC; c += NT) o[F + NL + c] = (p[c] - mu) * rstd;
    const int ldmax = img ? ld_img : ld_out;
    for (int c = F + NL + NC + threadIdx.x; c < ldmax; c += NT) o[c] = 0.f;
    __syncthreads();
    if (out) {
        float* og = out + row * ld_out;
        for (int c = threadIdx.x * 4; c < ld_out; c += NT * 4) *reinterpret_cast<float4*>(og + c) = *reinterpret_cast<const float4*>(o + c);
    }
    if (img) {                                    // fp16x3 operand image of the row (A operand of the pool_embed GEMM): no separate packing pass
        uint32_t* ig = img + row * ld_img;
        for (int pr = threadIdx.x; 2 * pr < ld_img; pr += NT) {
            uint32_t hi, lo;
            f16x3_split_pair(o[2 * pr], o[2 * pr + 1], img_scale, hi, lo);
            const long long wd = f16x3_word(2 * pr);
            ig[wd] = hi; ig[wd + 16] = lo;
        }
    }
}

// ---------------------------------------------------------------- residual + custom LayerNorm
// y = gamma * (v - mean) / (std_unbiased + 1e-6) + beta,  v = x + a    (transformer.py:74-77,87-88)
template <int NT>
__global__ void __launch_bounds__(NT)
add_ln_star_kernel(const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ gamma,
                   const float* __restrict__ beta, float* __restrict__ y, int H, uint32_t* __restrict__ img, float img_scale) {
    __shared__ float red[32];
    extern __shared__ float vbuf[];
    const long long row = blockIdx.x;
    float s = 0.f;
    for (int c = threadIdx.x; c < H; c += NT) {
        const float v = x[row * H + c] + a[row * H + c];
        vbuf[c] = v;
        s += v;
    }
    const float mu = block_sum(s, red) / (float)H;
    float q = 0.f;
    for (int c = threadIdx.x; c < H; c += NT) { const float d = vbuf[c] - mu; q += d * d; }
    const float sd = sqrtf(block_sum(q, red) / (float)(H - 1));
    const float inv = 1.f / (sd + 1e-6f);
    if (!img) {
        for (int c = threadIdx.x; c < H; c += NT) y[row * H + c] = gamma[c] * (vbuf[c] - mu) * inv + beta[c];
        return;
    }
    __syncthreads();                               // every thread has finished reading vbuf for the variance
    for (int c = threadIdx.x; c < H; c += NT) {
        const float v = gamma[c] * (vbuf[c] - mu) * inv + beta[c];
        y[row * H + c] = v;
        vbuf[c] = v;
    }
    __syncthreads();
    uint32_t* ig = img + row * H;                  // fp16x3 operand image of the row (H % 32 == 0): A operand of the next GEMMs
    for (int pr = threadIdx.x; 2 * pr < H; pr += NT) {
        uint32_t hi, lo;
        f16x3_split_pair(vbuf[2 * pr], vbuf[2 * pr + 1], img_scale, hi, lo);
        const long long wd = f16x3_word(2 * pr);
        ig[wd] = hi; ig[wd + 16] = lo;
    }
}

// ---------------------------------------------------------------- softmax over rows with a scale
// obj_interact attention probabilities: softmax(S / sqrt(d_model)) over the key axis (transformer.py:98-105)
template <int NT>
__global__ void __launch_bounds__(NT)
scaled_softmax_rows_kernel(float* __restrict__ S, int cols, long long ld, float inv_scale) {
    __shared__ float red[32];
    float* x = S + (long long)blockIdx.x * ld;
    float m = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += NT) m = fmaxf(m, x[c] * inv_scale);
    m = block_max(m, red);
    float s = 0.f;
    for (int c = threadIdx.x; c < cols; c += NT) {
        const float e = expf(x[c] * inv_scale - m);
        x[c] = e;
        s += e;
    }
    s = block_sum(s, red);
    const float inv = 1.f / s;
    for (int c = threadIdx.x; c < cols; c += NT) x[c] *= inv;
}

// register-resident variant: one read + one write of S (cols <= NT * VPT)
template <int NT, int VPT>
__global__ void __launch_bounds__(NT)
scaled_softmax_rows_reg_kernel(float* __restrict__ S, int cols, long long ld, float inv_scale) {
    __shared__ float red[32];
    float* x = S + (long long)blockIdx.x * ld;
    float v[VPT];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + i * NT;
        v[i] = c < cols ? x[c] * inv_scale : -INFINITY;
        m = fmaxf(m, v[i]);
    }
    m = block_max(m, red);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        v[i] = expf(v[i] - m);            // exp(-inf) = 0 for the padding lanes
        s += v[i];
    }
    s = block_sum(s, red);
    const float inv = 1.f / s;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + i * NT;
        if (c < cols) x[c] = v[i] * inv;
    }
}

// ---------------------------------------------------------------- GRU pointwise (both directions)
// r,z,n gate order, b_hn inside the r product (torch.nn.GRU); gi = W_ih x + b_ih for all t (precomputed),
// gh = W_hh h_{prev} + b_hh.  Writes the new state and the layer output row (optionally zeroed
// outside [sample_idx[b,0], sample_idx[b,1]) : model.py:505-507,564).
__global__ void gru_pointwise_kernel(const float* __restrict__ gi, const float* __restrict__ gh, const float* __restrict__ h_prev,
                                     float* __restrict__ h_new, float* __restrict__ out, const long long* __restrict__ sample_idx,
                                     int B, int T, int G, int step) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int d = blockIdx.y;
    if (idx >= B * G) return;
    const int b = idx / G, j = idx % G;
    const int t = d ? (T - 1 - step) : step;
    const float* gir = gi + ((long long)b * T + t) * (6 * G) + (long long)d * 3 * G;
    const float* ghr = gh + ((long long)d * B + b) * (3 * G);
    const float hp = h_prev[((long long)d * B + b) * G + j];
    const float r = sigmoid_acc(gir[j] + ghr[j]);
    const float z = sigmoid_acc(gir[G + j] + ghr[G + j]);
    const float n = tanhf(gir[2 * G + j] + r * ghr[2 * G + j]);
    const float h = (1.f - z) * n + z * hp;
    h_new[((long long)d * B + b) * G + j] = h;
    float o = h;
    if (sample_idx) {
        const long long lo = sample_idx[2 * b], hi = sample_idx[2 * b + 1];
        if (t < lo || t >= hi) o = 0.f;
    }
    out[((long long)b * T + t) * (2 * G) + (long long)d * G + j] = o;
}

}  // namespace

// ---------------------------------------------------------------- host launchers
int gvd_frame_mean(const float* segs, float* out, int B, int T, int C, cudaStream_t st) {
    dim3 grid(gvd_cdiv(C, 256), B);
    frame_mean_kernel<<<grid, 256, 0, st>>>(segs, out, T, C);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_clip_vector(const float* fc_mean, const long long* num, const float* Wseg, const float* bseg, float* xcat, int B,
                    int C, int S, int ld, cudaStream_t st, const long long* rows) {
    GVD_REQUIRE(S <= 64 && S <= 256, "clip_vector: seg_info_size %d too large", S);
    clip_vector_kernel<<<B, 256, 0, st>>>(fc_mean, num, Wseg, bseg, xcat, C, S, ld, rows);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_sim_softmax(float* simT, const unsigned char* pnt_mask, int B, int R, int NC, int ld, cudaStream_t st) {
    const int rows = B * R;
    sim_softmax_kernel<<<gvd_cdiv(rows, 8), 256, 0, st>>>(simT, pnt_mask, rows, R, NC, ld);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_transpose(const float* in, float* out, int B, int R, int C, int ld_in, cudaStream_t st) {
    dim3 grid(gvd_cdiv(C, 32), gvd_cdiv(R, 32), B), block(32, 8);
    transpose_kernel<<<grid, block, 0, st>>>(in, out, R, C, ld_in);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_transpose_split(const float* in, float* hi, float* lo, int B, int R, int C, int ld_in, cudaStream_t st) {
    dim3 grid(gvd_cdiv(C, 32), gvd_cdiv(R, 32), B), block(32, 8);
    transpose_split_kernel<<<grid, block, 0, st>>>(in, hi, lo, R, C, ld_in);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_pack_heads_f16x3(const float* in, long long ld_in, long long rows, int nh, int hs_in, int hs, int KH, float scale, float* out, cudaStream_t st) {
    GVD_REQUIRE(in && out && KH % 32 == 0 && KH >= hs && nh >= 1, "pack_heads_f16x3: bad arguments");
    const long long n = rows * nh * (KH / 2);
    pack_heads_f16x3_kernel<<<(unsigned)gvd_cdiv(n, 256), 256, 0, st>>>(in, ld_in, rows, nh, hs_in, hs, KH, scale, reinterpret_cast<uint32_t*>(out));
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_transpose_pack_f16x3(const float* in, float* out, int B, int R, int C, int ld_in, int Rp, float scale, cudaStream_t st) {
    GVD_REQUIRE(in && out && Rp % 32 == 0 && Rp >= R, "transpose_pack_f16x3: bad arguments");
    dim3 grid(gvd_cdiv(C, 32), Rp / 32, B), block(32, 8);
    transpose_pack_f16x3_kernel<<<grid, block, 0, st>>>(in, reinterpret_cast<uint32_t*>(out), R, C, ld_in, Rp, scale);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_split_hilo(const float* in, long long ld_in, float* hi, float* lo, long long ld_out, long long rows, int cols, cudaStream_t st) {
    GVD_REQUIRE(cols % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0, "split_hilo: cols / pitches must be multiples of 4");
    const long long n = rows * (cols / 4);
    split_hilo_kernel<<<(unsigned)gvd_cdiv(n, 256), 256, 0, st>>>(in, ld_in, hi, lo, ld_out, rows, cols / 4);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_pool_in(const float* g, const float* ppls, const float* simT, const float* Wloc, const float* bloc, float* out,
                long long rows, int F, int NL, int NC, int ld_sim, int ld_out, int num_frames, cudaStream_t st, float* img, int ld_img) {
    GVD_REQUIRE(NL <= 4 * 128, "pool_in: loc size %d too large", NL);
    GVD_REQUIRE(ld_out % 4 == 0 && (!img || (ld_img % 32 == 0 && ld_img >= ld_out)), "pool_in: pitches");
    const size_t smem = (size_t)std::max(ld_out, img ? ld_img : 0) * sizeof(float);
    pool_in_kernel<128><<<(unsigned)rows, 128, smem, st>>>(g, ppls, simT, Wloc, bloc, out, F, NL, NC, ld_sim, ld_out,
                                                         1.f / (float)num_frames, reinterpret_cast<uint32_t*>(img), ld_img, GVD_F16_SA);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_add_ln_star(const float* x, const float* a, const float* gamma, const float* beta, float* y, long long rows, int H,
                    cudaStream_t st, float* img) {
    GVD_REQUIRE(!img || H % 32 == 0, "add_ln_star: the operand image needs H %% 32 == 0");
    add_ln_star_kernel<256><<<(unsigned)rows, 256, H * sizeof(float), st>>>(x, a, gamma, beta, y, H, reinterpret_cast<uint32_t*>(img), GVD_F16_SA);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_scaled_softmax_rows(float* S, long long rows, int cols, long long ld, float inv_scale, cudaStream_t st) {
    GVD_REQUIRE(rows < (1ll << 31), "softmax: too many rows");
    if (cols <= 1024) scaled_softmax_rows_reg_kernel<256, 4><<<(unsigned)rows, 256, 0, st>>>(S, cols, ld, inv_scale);
    else if (cols <= 2048) scaled_softmax_rows_reg_kernel<256, 8><<<(unsigned)rows, 256, 0, st>>>(S, cols, ld, inv_scale);
    else scaled_softmax_rows_kernel<256><<<(unsigned)rows, 256, 0, st>>>(S, cols, ld, inv_scale);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_gru_pointwise(const float* gi, const float* gh, const float* h_prev, float* h_new, float* out,
                      const long long* sample_idx, int B, int T, int G, int step, cudaStream_t st) {
    dim3 grid(gvd_cdiv((long long)B * G, 256), 2);
    gru_pointwise_kernel<<<grid, 256, 0, st>>>(gi, gh, h_prev, h_new, out, sample_idx, B, T, G, step);
    GVD_CHECK_LAUNCH();
    return 0;
}
