// gvd-b200: teacher-forced side of the hot path — IoU, per-step RoI labels / frame masks, the four
// losses and the GRD argmax outputs (reference: misc/bbox_transform.py:224-269, misc/utils.py:117-152,
// 293-328, misc/model.py:317-350,431-440,464-489).  All reductions are two-stage with a fixed
// order (per-row partials -> one block), so losses are run-to-run deterministic.
#include "gvd_kernels.cuh"

namespace {

// overlaps[b,r,k] = IoU(+1 pixel convention) * (1 - (frm_mask[b,r,k] | pnt_mask[b,r+1])); zero-area GT -> 0,
// zero-area proposal -> -1   (bbox_transform.py:224-269 3-D branch, call site model.py:317-318)
__global__ void bbox_overlaps_kernel(const float* __restrict__ ppls, const float* __restrict__ gt, const unsigned char* __restrict__ frm_mask,
                                     const unsigned char* __restrict__ pnt_mask, float* __restrict__ ov, int B, int R, int NB) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * R * NB) return;
    const int k = idx % NB, r = (idx / NB) % R, b = idx / ((long long)NB * R);
    const float* a = ppls + ((long long)b * R + r) * 7;
    const float* g = gt + ((long long)b * NB + k) * 6;
    const float aw = a[2] - a[0] + 1.f, ah = a[3] - a[1] + 1.f;
    const float gw = g[2] - g[0] + 1.f, gh = g[3] - g[1] + 1.f;
    float iw = fminf(a[2], g[2]) - fmaxf(a[0], g[0]) + 1.f;
    float ih = fminf(a[3], g[3]) - fmaxf(a[1], g[1]) + 1.f;
    iw = iw < 0.f ? 0.f : iw;
    ih = ih < 0.f ? 0.f : ih;
    const float inter = iw * ih;
    const float ua = aw * ah + gw * gh - inter;
    float o = inter / ua;
    const bool masked = frm_mask[idx] != 0 || pnt_mask[(long long)b * (R + 1) + 1 + r] != 0;
    o *= masked ? 0.f : 1.f;
    if (gw == 1.f && gh == 1.f) o = 0.f;
    if (aw == 1.f && ah == 1.f) o = -1.f;
    ov[idx] = o;
}

// sim_target[b,k,r] = (ov > 0.5) * cls_k (utils.py:299-305); pred[b,r] = argmax_c sim (model.py:354);
// per-(b,k) partial sums of clamp(log sim[b, cls, r], -100) over positives (BCE vs ones, model.py:348-350)
__global__ void __launch_bounds__(128) cls_target_kernel(const float* __restrict__ ov, const float* __restrict__ gt, const float* __restrict__ simT,
                                                         int* __restrict__ target, float* __restrict__ part_sum, int* __restrict__ part_cnt,
                                                         int R, int NB, int NC, int ld_sim) {
    __shared__ float red[32];
    const int b = blockIdx.x / NB, k = blockIdx.x % NB;
    const int cls = (int)gt[((long long)b * NB + k) * 6 + 5];
    float s = 0.f, c = 0.f;
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        const int t = ov[((long long)b * R + r) * NB + k] > 0.5f ? cls : 0;
        target[((long long)b * NB + k) * R + r] = t;
        if (t > 0) {
            s += fmaxf(logf(simT[((long long)b * R + r) * ld_sim + t]), -100.f);
            c += 1.f;
        }
    }
    s = block_sum(s, red);
    c = block_sum(c, red);
    if (threadIdx.x == 0) { part_sum[blockIdx.x] = s; part_cnt[blockIdx.x] = (int)c; }
}

__global__ void class_argmax_kernel(const float* __restrict__ simT, int* __restrict__ pred, long long rows, int NC, int ld) {
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float* x = simT + warp * ld;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < NC; c += 32) {
        const float v = x[c];
        if (v > bv || (v == bv && c < bi)) { bv = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov_ = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov_ > bv || (ov_ == bv && oi < bi)) { bv = ov_; bi = oi; }
    }
    if (lane == 0) pred[warp] = bi;
}

// per (b, i, r): labels (utils.py:307-328: max over boxes tied to word i+1 of IoU > 0.5) and the frame mask
// (model.py:436-440: proposal has no tied box on its frame, or is masked); fm[b,i,0] = 0 (legacy column)
__global__ void step_targets_kernel(const float* __restrict__ ov, const unsigned char* __restrict__ mask_boxes,
                                    const unsigned char* __restrict__ frm_mask, const unsigned char* __restrict__ pnt_mask,
                                    unsigned char* __restrict__ labels, unsigned char* __restrict__ fm, int B, int S, int R, int NB, int L1) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * S * R) return;
    const int r = idx % R, i = (idx / R) % S, b = idx / ((long long)R * S);
    float mx = -INFINITY;
    int active = 0;
    for (int k = 0; k < NB; ++k) {
        const bool bm = mask_boxes[((long long)b * NB + k) * L1 + i + 1] != 0;       // 0 = box tied to the target word
        const float o = bm ? 0.f : ov[((long long)b * R + r) * NB + k];
        mx = fmaxf(mx, o);
        active += (!bm && frm_mask[((long long)b * R + r) * NB + k] == 0) ? 1 : 0;
    }
    labels[idx] = mx > 0.5f ? 1 : 0;
    const bool m = (active <= 0) || pnt_mask[(long long)b * (R + 1) + 1 + r] != 0;
    fm[((long long)b * S + i) * (R + 1) + 1 + r] = m ? 1 : 0;
    if (r == 0) fm[((long long)b * S + i) * (R + 1)] = pnt_mask[(long long)b * (R + 1)];
}

// rows of vis_relu gathered by class index: emb[b,i,:] = ReLU(vis_embed)[clamp(word - V, 0)]  (model.py:469-470)
__global__ void gather_class_rows_kernel(const float* __restrict__ vis_relu, const long long* __restrict__ input_cls, float* __restrict__ emb,
                                         int* __restrict__ cls_idx, int S, int L1, int V, int D2, int NC) {
    const int row = blockIdx.x, b = row / S, i = row % S;
    long long c = input_cls[(long long)b * L1 + i + 1] - V;
    c = c < 0 ? 0 : (c >= NC ? NC - 1 : c);              // upper clamp: stay inside the table (the Python shim rejects such ids)
    if (threadIdx.x == 0) cls_idx[row] = (int)c;
    for (int d = threadIdx.x * 4; d < D2; d += blockDim.x * 4)
        *reinterpret_cast<float4*>(emb + (long long)row * D2 + d) = *reinterpret_cast<const float4*>(vis_relu + c * D2 + d);
}

// G[b,i,r] = dot + bias[cls] + z[b,i,r], then -1e8 where masked (model.py:472-486, _grounder :267-278).  cls_bias NULL: the module has no
// class bias (transfer_mode 'none', model.py:475-476), G = dot + z
__global__ void grounding_finish_kernel(float* __restrict__ G, const float* __restrict__ z, const float* __restrict__ cls_bias,
                                        const int* __restrict__ cls_idx, const unsigned char* __restrict__ mask, long long mask_stride_row,
                                        int mask_per_step, int S, int R, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int r = idx % R;
    const long long row = idx / R;                 // b*S + i
    const long long b = row / S;
    const unsigned char m = mask_per_step ? mask[row * mask_stride_row + 1 + r] : mask[b * mask_stride_row + 1 + r];
    if (m) { G[idx] = GVD_MIN_VALUE; return; }
    float g = G[idx];
    if (cls_bias) g += cls_bias[cls_idx[row]];
    G[idx] = g + z[idx];
}

// per (b,i): nll = -(logit[target] - lse) and whether the position counts (utils.py:126-136)
__global__ void __launch_bounds__(256) lm_nll_kernel(const float* __restrict__ logits, long long ld, const long long* __restrict__ seq, int S,
                                                     int L1, int V, float* __restrict__ part_sum, int* __restrict__ part_cnt) {
    __shared__ float red[32];
    const int row = blockIdx.x, b = row / S, i = row % S;
    const float* x = logits + (long long)row * ld;
    float m = -INFINITY;
    for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, x[v]);
    m = block_max(m, red);
    float s = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(x[v] - m);
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        const long long tgt = seq[(long long)b * L1 + i + 1];
        const bool counts = (i == 0) || (seq[(long long)b * L1 + i] > 0);       // mask shifted right with a leading 1
        const float xt = (tgt >= 0 && tgt < V) ? x[tgt] : __int_as_float(0x7fc00000);   // out-of-range target: NaN loss, no stray read
        part_sum[row] = counts ? -(xt - (m + logf(s))) : 0.f;
        part_cnt[row] = counts ? 1 : 0;
    }
}

// per (b,i): sum over positive RoIs of log_softmax_r(x) and their count (utils.py:139,142)
__global__ void __launch_bounds__(256) att_nll_kernel(const float* __restrict__ x_all, const unsigned char* __restrict__ labels, int R,
                                                      float* __restrict__ part_sum, int* __restrict__ part_cnt) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const float* x = x_all + row * R;
    const unsigned char* lab = labels + row * R;
    float m = -INFINITY;
    for (int r = threadIdx.x; r < R; r += blockDim.x) m = fmaxf(m, x[r]);
    m = block_max(m, red);
    float s = 0.f;
    for (int r = threadIdx.x; r < R; r += blockDim.x) s += expf(x[r] - m);
    s = block_sum(s, red);
    const float lse = m + logf(s);
    float acc = 0.f, cnt = 0.f;
    for (int r = threadIdx.x; r < R; r += blockDim.x)
        if (lab[r]) { acc += x[r] - lse; cnt += 1.f; }
    acc = block_sum(acc, red);
    cnt = block_sum(cnt, red);
    if (threadIdx.x == 0) { part_sum[row] = acc; part_cnt[row] = (int)cnt; }
}

// out = -(sum of partials) / (count)  in a fixed order; empty set -> NaN like torch.mean of an empty tensor (quirk Q11)
__global__ void __launch_bounds__(256) finish_mean_kernel(const float* __restrict__ part_sum, const int* __restrict__ part_cnt, int n, float sign,
                                                          float* __restrict__ out) {
    __shared__ double sh_s[256];
    __shared__ long long sh_c[256];
    double s = 0.0;
    long long c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { s += (double)part_sum[i]; c += part_cnt[i]; }
    sh_s[threadIdx.x] = s;
    sh_c[threadIdx.x] = c;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { sh_s[threadIdx.x] += sh_s[threadIdx.x + o]; sh_c[threadIdx.x] += sh_c[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sh_c[0] > 0 ? (float)(sign * sh_s[0] / (double)sh_c[0]) : __int_as_float(0x7fc00000);
}

// argmax over the proposals of each frame (model.py:487-489)
__global__ void frame_argmax_kernel(const float* __restrict__ x, long long* __restrict__ out, long long rows, int NF, int P) {
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows * NF) return;
    const float* p = x + warp * P;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < P; c += 32) {
        const float v = p[c];
        if (v > bv || (v == bv && c < bi)) { bv = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov_ = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov_ > bv || (ov_ == bv && oi < bi)) { bv = ov_; bi = oi; }
    }
    if (lane == 0) out[warp] = bi;
}

// boxes[b, j, f, :] = ppls[b, f*P + idx[b, j, f], :]  (main.py:367-370: the proposal each generated word attends to in every frame)
__global__ void grounding_gather_kernel(const float* __restrict__ ppls, const long long* __restrict__ idx, float* __restrict__ boxes,
                                        long long n, int L, int NF, int P, int C) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // one thread per (b, j, f, c)
    if (t >= n) return;
    const int c = (int)(t % C);
    const long long e = t / C;                                                   // (b, j, f)
    const int f = (int)(e % NF);
    const long long b = e / ((long long)NF * L);
    const long long r = (long long)f * P + idx[e];
    boxes[t] = ppls[(b * NF * P + r) * C + c];
}

// Localisation hit test of the grounding evaluator (eval_grd_anet_entities.py:95-102, scripts/utils.py:75-128): one warp per word,
// lanes over the (frame, annotation) pairs.  The arithmetic is written with the non-contracting intrinsics in the reference's
// operation order (iw*ih / (a_area + g_area - iw*ih)) so that the `> thresh` decision is bit-identical to the fp32 CPU result.
__global__ void grounding_eval_kernel(const float* __restrict__ pred, const float* __restrict__ ref, const int* __restrict__ nref,
                                      float* __restrict__ max_iou, unsigned char* __restrict__ hit, int N, int F, int K, float thresh) {
    const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (w >= N) return;
    const int k_valid = min(nref[w], K);
    float best = -INFINITY;
    for (int t = lane; t < F * k_valid; t += 32) {
        const int f = t / k_valid, k = t % k_valid;
        const float* a = pred + ((long long)w * F + f) * 5;
        const float* g = ref + ((long long)w * K + k) * 5;
        const float aw = __fadd_rn(__fsub_rn(a[2], a[0]), 1.f), ah = __fadd_rn(__fsub_rn(a[3], a[1]), 1.f);
        const float gw = __fadd_rn(__fsub_rn(g[2], g[0]), 1.f), gh = __fadd_rn(__fsub_rn(g[3], g[1]), 1.f);
        float iw = __fadd_rn(__fsub_rn(fminf(a[2], g[2]), fmaxf(a[0], g[0])), 1.f);
        float ih = __fadd_rn(__fsub_rn(fminf(a[3], g[3]), fmaxf(a[1], g[1])), 1.f);
        iw = iw < 0.f ? 0.f : iw;
        ih = ih < 0.f ? 0.f : ih;
        const float inter = __fmul_rn(iw, ih);
        const float ua = __fsub_rn(__fadd_rn(__fmul_rn(aw, ah), __fmul_rn(gw, gh)), inter);
        float o = __fmul_rn(__fdiv_rn(inter, ua), a[4] != g[4] ? 0.f : 1.f);      // different frames never overlap
        if (gw == 1.f && gh == 1.f) o = 0.f;
        if (aw == 1.f && ah == 1.f) o = -1.f;
        best = fmaxf(best, o);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) {
        if (k_valid <= 0) best = -1.f;                                            // nothing annotated for this word
        max_iou[w] = best;
        hit[w] = best > thresh ? 1 : 0;
    }
}

}  // namespace

int gvd_grounding_eval_hits(const float* pred, const float* ref, const int* nref, float* max_iou, unsigned char* hit, int N, int F, int K,
                            float thresh, cudaStream_t st) {
    grounding_eval_kernel<<<gvd_cdiv((long long)N * 32, 256), 256, 0, st>>>(pred, ref, nref, max_iou, hit, N, F, K, thresh);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_grounding_gather(const float* ppls, const long long* idx, float* boxes, int B, int L, int NF, int P, int C, cudaStream_t st) {
    const long long n = (long long)B * L * NF * C;
    grounding_gather_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(ppls, idx, boxes, n, L, NF, P, C);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_bbox_overlaps(const float* ppls, const float* gt, const unsigned char* frm_mask, const unsigned char* pnt_mask, float* ov, int B, int R,
                      int NB, cudaStream_t st) {
    const long long n = (long long)B * R * NB;
    bbox_overlaps_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(ppls, gt, frm_mask, pnt_mask, ov, B, R, NB);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_cls_target(const float* ov, const float* gt, const float* simT, int* target, float* part_sum, int* part_cnt, int B, int R, int NB,
                   int NC, int ld_sim, cudaStream_t st) {
    cls_target_kernel<<<B * NB, 128, 0, st>>>(ov, gt, simT, target, part_sum, part_cnt, R, NB, NC, ld_sim);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_class_argmax(const float* simT, int* pred, long long rows, int NC, int ld, cudaStream_t st) {
    class_argmax_kernel<<<gvd_cdiv(rows, 8), 256, 0, st>>>(simT, pred, rows, NC, ld);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_step_targets(const float* ov, const unsigned char* mask_boxes, const unsigned char* frm_mask, const unsigned char* pnt_mask,
                     unsigned char* labels, unsigned char* fm, int B, int S, int R, int NB, int L1, cudaStream_t st) {
    const long long n = (long long)B * S * R;
    step_targets_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(ov, mask_boxes, frm_mask, pnt_mask, labels, fm, B, S, R, NB, L1);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_gather_class_rows(const float* vis_relu, const long long* input_cls, float* emb, int* cls_idx, int B, int S, int L1, int V, int D2, int NC,
                          cudaStream_t st) {
    gather_class_rows_kernel<<<B * S, 256, 0, st>>>(vis_relu, input_cls, emb, cls_idx, S, L1, V, D2, NC);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_grounding_finish(float* G, const float* z, const float* cls_bias, const int* cls_idx, const unsigned char* mask, long long mask_stride_row,
                         int mask_per_step, int B, int S, int R, cudaStream_t st) {
    const long long n = (long long)B * S * R;
    grounding_finish_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(G, z, cls_bias, cls_idx, mask, mask_stride_row, mask_per_step, S, R, n);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_lm_nll(const float* logits, long long ld, const long long* seq, int B, int S, int L1, int V, float* part_sum, int* part_cnt,
               cudaStream_t st) {
    lm_nll_kernel<<<B * S, 256, 0, st>>>(logits, ld, seq, S, L1, V, part_sum, part_cnt);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_att_nll(const float* x, const unsigned char* labels, long long rows, int R, float* part_sum, int* part_cnt, cudaStream_t st) {
    att_nll_kernel<<<(unsigned)rows, 256, 0, st>>>(x, labels, R, part_sum, part_cnt);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_finish_mean(const float* part_sum, const int* part_cnt, int n, float sign, float* out, cudaStream_t st) {
    finish_mean_kernel<<<1, 256, 0, st>>>(part_sum, part_cnt, n, sign, out);
    GVD_CHECK_LAUNCH();
    return 0;
}
int gvd_frame_argmax(const float* x, long long* out, long long rows, int NF, int P, cudaStream_t st) {
    frame_argmax_kernel<<<gvd_cdiv(rows * NF, 8), 256, 0, st>>>(x, out, rows, NF, P);
    GVD_CHECK_LAUNCH();
    return 0;
}
