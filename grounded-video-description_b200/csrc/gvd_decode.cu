// gvd-b200: decode-step kernels — TopDownCore.forward (misc/AttModel.py:134-164) rebuilt for sm_90a.
//
//   lstm_step_kernel     : both LSTMCells (AttModel.py:139,160): gate GEMM over up to three
//                          K-segments (no concat is ever materialised; the token embedding is
//                          gathered inside the operand loader) + the i,f,g,o pointwise, fused.
//   attn_partial_kernel  : Attention (AttModel.py:33-53) and Attention2 (AttModel.py:71-108):
//                          each CTA owns one (clip, row-chunk); a producer warp streams the
//                          chunk's projected rows and then its feature rows HBM -> shared memory
//                          with 1-D bulk TMA copies through a 6-stage mbarrier ring; 8 consumer
//                          warps do  w.tanh(p+q)  (warp-shuffle reduce), the chunk softmax
//                          numerators and the weighted feature sum.  Every feature byte is read
//                          from HBM exactly once per step.
//                          att_input_mode 'featmap' (AttModel.py:145-146): the region chunks stop
//                          after the scores, so the region features are not read at all.
//                          'dual_region' (AttModel.py:153-156): both region attentions share one
//                          pass over the region rows (two scores per p_pool row, two weighted
//                          sums per pool row); the merging CTA applies the dual_pointer gate.
//                          region_attn_mode (AttModel.py:79-96) is a template parameter of the
//                          region chunks' score: ADD w.tanh(p+q)+b ('mix'), MUL w.tanh(p*q)+b
//                          ('mix_mul') or DOT p.q ('dp': no alpha_net, w / b never read).  The
//                          temporal chunks are additive in every mode.
//                          Video-indexed batches (AttnArgs::vid): a clip's temporal chunks stream only its window's rows of
//                          the video's unmasked features; the first one adds the closed-form out-of-window softmax term.
//   attn_group_kernel    : the same attention for up to 8 rows that share a clip's features (sampled captions, beam rows) per CTA: each
//                          chunk is streamed once and scored against every query of the group.  Bit-identical to attn_partial_kernel
//                          per row; measured slower than it on shared features (L2 serves the per-row kernel's repeated reads), so the
//                          decode does not select it (gvd_attn_partial_path, DESIGN §3).
//   attn_combine_kernel  : merges the chunk partials (flash-decoding style) into att + att2.
//   greedy_pick_kernel   : log_softmax + top-2 + UNK rule (misc/model.py:590-594,615).
#include "../../include/gvd_b200.h"
#include "gvd_kernels.cuh"

namespace {

// =====================================================================================
// LSTM step
// =====================================================================================
constexpr int L_BM = 128, L_UJ = 8, L_BN = 4 * L_UJ, L_BK = 16, L_NT = 256, L_PAD = 4;

__global__ void __launch_bounds__(L_NT) lstm_step_kernel(LstmArgs a) {
    __shared__ __align__(16) float As[2][L_BK][L_BM + L_PAD];
    __shared__ __align__(16) float Ws[2][L_BK][L_BN + L_PAD];
    __shared__ float gates[L_BM][L_BN + 1];

    const int tid = threadIdx.x;
    const int tx = tid % 8, ty = tid / 8;          // 4 columns x 4 rows per thread
    const int j0 = blockIdx.x * L_UJ, m0 = blockIdx.y * L_BM;
    const int H = a.H;

    int tiles_in[3];
    int ntiles = 0;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
        tiles_in[s] = (s < a.nseg) ? (a.seg[s].K + L_BK - 1) / L_BK : 0;
        ntiles += tiles_in[s];
    }

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    float4 ra[2], rw;
    auto gload = [&](int tile) {
        int s = 0;
        while (tile >= tiles_in[s]) { tile -= tiles_in[s]; ++s; }
        const LstmSeg& sg = a.seg[s];
        const int k0 = tile * L_BK;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int f = tid + i * L_NT, row = f >> 2, kq = f & 3;
            const int b = m0 + row, k = k0 + kq * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (b < a.B && k < sg.K) {
                const long long r = sg.gather ? sg.gather[b] : (long long)b;
                v = __ldg(reinterpret_cast<const float4*>(sg.x + r * sg.ldx + k));
                if (sg.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            }
            ra[i] = v;
        }
        rw = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tid < 128) {
            const int n = tid >> 2, kq = tid & 3;
            const int gate = n / L_UJ, j = j0 + (n % L_UJ), k = k0 + kq * 4;
            if (j < H && k < sg.K) rw = __ldg(reinterpret_cast<const float4*>(sg.w + ((long long)gate * H + j) * sg.ldw + k));
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int f = tid + i * L_NT, row = f >> 2, kq = f & 3;
            As[buf][kq * 4 + 0][row] = ra[i].x;
            As[buf][kq * 4 + 1][row] = ra[i].y;
            As[buf][kq * 4 + 2][row] = ra[i].z;
            As[buf][kq * 4 + 3][row] = ra[i].w;
        }
        if (tid < 128) {
            const int n = tid >> 2, kq = tid & 3;
            Ws[buf][kq * 4 + 0][n] = rw.x;
            Ws[buf][kq * 4 + 1][n] = rw.y;
            Ws[buf][kq * 4 + 2][n] = rw.z;
            Ws[buf][kq * 4 + 3][n] = rw.w;
        }
    };

    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < ntiles; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < ntiles) gload(kt + 1);
#pragma unroll
        for (int k = 0; k < L_BK; ++k) {
            const float4 av = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 bv = *reinterpret_cast<const float4*>(&Ws[buf][k][tx * 4]);
            const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
        }
        if (kt + 1 < ntiles) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) gates[ty * 4 + i][tx * 4 + j] = acc[i][j];
    __syncthreads();

    // pointwise: rows ordered i,f,g,o (torch.nn.LSTMCell)
    for (int idx = tid; idx < L_BM * L_UJ; idx += L_NT) {
        const int bl = idx / L_UJ, jj = idx % L_UJ;
        const int b = m0 + bl, j = j0 + jj;
        if (b >= a.B || j >= H) continue;
        float g4[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float v = gates[bl][q * L_UJ + jj];
            const long long col = (long long)q * H + j;
            if (a.pre) v += a.pre[(long long)(a.pre_div > 1 ? b / a.pre_div : b) * 4 * H + col];
            if (a.bias1) v += a.bias1[col];
            if (a.bias2) v += a.bias2[col];
            g4[q] = v;
        }
        const float ig = sigmoid_acc(g4[0]), fg = sigmoid_acc(g4[1]), gg = tanhf(g4[2]), og = sigmoid_acc(g4[3]);
        const float c = fg * a.c_prev[(long long)b * H + j] + ig * gg;
        a.c_out[(long long)b * H + j] = c;
        a.h_out[(long long)b * H + j] = og * tanhf(c);
    }
}

// =====================================================================================
// attention partials
// =====================================================================================
constexpr int ATT_STAGE_BYTES = 16384;
constexpr int ATT_NST = 6;
constexpr int ATT_MAXC = 128;
constexpr int ATT_CWARPS = 8;
constexpr int ATT_THREADS = (ATT_CWARPS + 1) * 32;

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(ATT_CWARPS * 32) : "memory"); }

template <int F> struct FormTag { static constexpr int value = F; };

// one term of a row's score in form F (GVD_REGION_ATTN_*): acc + w tanh(p + q), acc + w tanh(p q), or acc + p q (w unused)
template <int F>
__device__ __forceinline__ float att_term(float w, float p, float q, float acc) {
    if (F == GVD_REGION_ATTN_MIX) return fmaf(w, tanh_mufu(p + q), acc);
    if (F == GVD_REGION_ATTN_MIX_MUL) return fmaf(w, tanh_mufu(p * q), acc);
    return fmaf(p, q, acc);
}

// att_input_mode 'dual_region', consumer warps of one region chunk: attention2 (query slot 1, w2 / b2) and attention2_dual (query slot 0,
// w1 / b1) over the same stream of p_pool / pool rows and the same masks; the returned logits (z_out) are attention2's.  Shared memory
// after the generic query area: q1[A] w1[A] q2[A] w2[A] z2[MAXC] e2[MAXC] ml2[4].  Both attentions score in form F (DOT: w1 / w2 / b1 / b2
// are not read).
template <int F>
__device__ __forceinline__ void attn_dual_consumer(const AttnArgs& a, int nch_r, int b, int fb, int c, int r0, int nrows, int n_pa, int n_pb,
                                                int rows_pa, int rows_pb, unsigned char* smem, uint64_t* full, uint64_t* empty, float* z_s,
                                                float* e_s, float* ml, float* qs) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int A = a.A, H = a.H;
    float* ws = qs + A;
    float* qd = ws + A;
    float* wd = qd + A;
    float* zd_s = wd + A;
    float* ed_s = zd_s + ATT_MAXC;
    float* mld = ed_s + ATT_MAXC;
    for (int i = tid; i < 2 * A; i += ATT_CWARPS * 32) {
        float v;
        if (a.q) {
            v = a.q[(long long)b * 2 * A + i];
        } else {
            v = __ldg(a.q_bias + i);
            for (int s = 0; s < a.q_S; ++s) v += __ldcg(a.q_part + s * a.q_plane + (long long)b * 2 * A + i);
        }
        if (i < A) qd[i] = v; else qs[i - A] = v;
    }
    if (F != GVD_REGION_ATTN_DP)
        for (int i = tid; i < A; i += ATT_CWARPS * 32) { ws[i] = a.w2[i]; wd[i] = a.w1[i]; }
    consumer_bar();
    const float bias = F == GVD_REGION_ATTN_DP ? 0.f : __ldg(a.b2), bias_d = F == GVD_REGION_ATTN_DP ? 0.f : __ldg(a.b1);

    // phase A: both score vectors from one read of each projected row
    for (int i = 0; i < n_pa; ++i) {
        const int s = i % ATT_NST;
        const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
        mbar_wait(&full[s], ph);
        const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
        const int row0 = i * rows_pa, nr = min(rows_pa, nrows - row0);
        for (int rr = warp; rr < nr; rr += ATT_CWARPS) {
            const float* pr = st + (long long)rr * A;
            float sum = 0.f, sum_d = 0.f;
            for (int a0 = lane * 4; a0 < A; a0 += 128) {
                const float4 v = *reinterpret_cast<const float4*>(pr + a0);
                const float4 qv = *reinterpret_cast<const float4*>(qs + a0), wv = *reinterpret_cast<const float4*>(ws + a0);
                const float4 qv2 = *reinterpret_cast<const float4*>(qd + a0), wv2 = *reinterpret_cast<const float4*>(wd + a0);
                sum = att_term<F>(wv.x, v.x, qv.x, sum);
                sum = att_term<F>(wv.y, v.y, qv.y, sum);
                sum = att_term<F>(wv.z, v.z, qv.z, sum);
                sum = att_term<F>(wv.w, v.w, qv.w, sum);
                sum_d = att_term<F>(wv2.x, v.x, qv2.x, sum_d);
                sum_d = att_term<F>(wv2.y, v.y, qv2.y, sum_d);
                sum_d = att_term<F>(wv2.z, v.z, qv2.z, sum_d);
                sum_d = att_term<F>(wv2.w, v.w, qv2.w, sum_d);
            }
            sum = warp_sum(sum);
            sum_d = warp_sum(sum_d);
            if (lane == 0) {
                float z = sum + bias, zd = sum_d + bias_d;
                const int rl = row0 + rr;
                const long long mi = (long long)fb * (a.R + 1) + 1 + r0 + rl;
                const long long oi = a.out_mask_stride ? (long long)fb * a.out_mask_stride + 1 + r0 + rl : mi;
                const bool am = a.att_mask[mi] != 0, om = a.out_mask[oi] != 0;
                if (am) { z = GVD_MIN_VALUE; zd = GVD_MIN_VALUE; }                      // AttModel.py:99, both attentions
                a.z_out[(long long)b * a.z_stride_b + r0 + rl] = (am || om) ? GVD_MIN_VALUE : z;
                z_s[rl] = z;
                zd_s[rl] = zd;
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    consumer_bar();
    if (warp < 2) {
        const float* zz = warp ? zd_s : z_s;
        float* ee = warp ? ed_s : e_s;
        float m = -INFINITY;
        for (int r = lane; r < nrows; r += 32) m = fmaxf(m, zz[r]);
        m = warp_max(m);
        float l = 0.f;
        for (int r = lane; r < nrows; r += 32) {
            const float e = expf(zz[r] - m);
            ee[r] = e;
            l += e;
        }
        l = warp_sum(l);
        if (lane == 0) { (warp ? mld : ml)[0] = m; (warp ? mld : ml)[1] = l; }
    }
    consumer_bar();

    // phase B: both unnormalised weighted sums from one read of each feature row
    const int h0 = tid * 4;
    const bool active = h0 < H;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f), acc_d = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < n_pb; ++j) {
        const int i = n_pa + j, s = i % ATT_NST;
        const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
        mbar_wait(&full[s], ph);
        const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
        const int row0 = j * rows_pb, nr = min(rows_pb, nrows - row0);
        if (active) {
            for (int rr = 0; rr < nr; ++rr) {
                const float e = e_s[row0 + rr], ed = ed_s[row0 + rr];
                const float4 v = *reinterpret_cast<const float4*>(st + (long long)rr * H + h0);
                acc.x = fmaf(e, v.x, acc.x); acc.y = fmaf(e, v.y, acc.y); acc.z = fmaf(e, v.z, acc.z); acc.w = fmaf(e, v.w, acc.w);
                acc_d.x = fmaf(ed, v.x, acc_d.x); acc_d.y = fmaf(ed, v.y, acc_d.y); acc_d.z = fmaf(ed, v.z, acc_d.z); acc_d.w = fmaf(ed, v.w, acc_d.w);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    const int nrec = 2 * nch_r;
    float* out = a.partial + ((long long)b * nrec + c) * (H + 4);
    float* out_d = a.partial + ((long long)b * nrec + nch_r + c) * (H + 4);
    if (tid == 0) { out[0] = ml[0]; out[1] = ml[1]; out_d[0] = mld[0]; out_d[1] = mld[1]; }
    if (active) {
        *reinterpret_cast<float4*>(out + 4 + h0) = acc;
        *reinterpret_cast<float4*>(out_d + 4 + h0) = acc_d;
    }
    // ---- fused merge by the last chunk CTA of the row (fixed chunk order), then the gate
    __threadfence();
    consumer_bar();
    int* flag = reinterpret_cast<int*>(ml + 2);
    if (tid == 0) *flag = (atomicAdd(a.ticket + b, 1) == nch_r - 1) ? 1 : 0;
    consumer_bar();
    if (*flag == 0) return;
    __threadfence();
    // g = sigmoid(dual_pointer(h_att)) (AttModel.py:155): per-thread partial dot, warp sums, the 8 warp sums added in warp order
    float gd = 0.f;
    if (active) {
        const float4 hv = *reinterpret_cast<const float4*>(a.gate_h + (long long)b * a.gate_ld + h0);
        const float4 wv = __ldg(reinterpret_cast<const float4*>(a.gate_w + h0));
        gd = fmaf(wv.x, hv.x, gd); gd = fmaf(wv.y, hv.y, gd); gd = fmaf(wv.z, hv.z, gd); gd = fmaf(wv.w, hv.w, gd);
    }
    gd = warp_sum(gd);
    if (lane == 0) zd_s[warp] = gd;
    consumer_bar();
    float glogit = __ldg(a.gate_b);
    for (int wv = 0; wv < ATT_CWARPS; ++wv) glogit += zd_s[wv];
    const float g = sigmoid_acc(glogit);
    const float* base = a.partial + (long long)b * nrec * (H + 4);
    if (active) {
        float4 r[2];
#pragma unroll
        for (int part = 0; part < 2; ++part) {                 // attention2 chunks, then attention2_dual chunks
            const int c0 = part * nch_r, c1 = c0 + nch_r;
            float M = -INFINITY;
            for (int cc = c0; cc < c1; ++cc) M = fmaxf(M, __ldcg(base + (long long)cc * (H + 4)));
            float L = 0.f;
            float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int cc = c0; cc < c1; ++cc) {
                const float* pc = base + (long long)cc * (H + 4);
                const float sc = expf(__ldcg(pc) - M);
                L = fmaf(__ldcg(pc + 1), sc, L);
                const float4 v = __ldcg(reinterpret_cast<const float4*>(pc + 4 + h0));
                s4.x = fmaf(v.x, sc, s4.x); s4.y = fmaf(v.y, sc, s4.y); s4.z = fmaf(v.z, sc, s4.z); s4.w = fmaf(v.w, sc, s4.w);
            }
            r[part] = make_float4(s4.x / L, s4.y / L, s4.z / L, s4.w / L);
        }
        const float h = 1.f - g;                               // dual_p * att2 + (1 - dual_p) * att2_dual (AttModel.py:156)
        const float4 res = make_float4(g * r[0].x + h * r[1].x, g * r[0].y + h * r[1].y, g * r[0].z + h * r[1].z, g * r[0].w + h * r[1].w);
        *reinterpret_cast<float4*>(a.x_out + (long long)b * (a.x_ld ? a.x_ld : H) + h0) = res;
        if (a.x_pk) {
            uint32_t hi0, lo0, hi1, lo1;
            f16x3_split_pair(res.x, res.y, GVD_F16_SA, hi0, lo0);
            f16x3_split_pair(res.z, res.w, GVD_F16_SA, hi1, lo1);
            uint32_t* d = reinterpret_cast<uint32_t*>(a.x_pk) + (long long)b * a.x_pk_ld + f16x3_word(h0);
            *reinterpret_cast<uint2*>(d) = make_uint2(hi0, hi1);
            *reinterpret_cast<uint2*>(d + 16) = make_uint2(lo0, lo1);
        }
    }
    if (tid == 0) a.ticket[b] = 0;
}

// one warp's score sum of the projected row pr (before the warp reduction), form F
template <int AJ, int F>
__device__ __forceinline__ float att_row_sum(const float* pr, const float4* q4, const float4* w4, const float* qs, const float* ws, int A,
                                             int lane) {
    float sum = 0.f;
    if (AJ > 0) {
#pragma unroll
        for (int j = 0; j < AJ; ++j) {
            const float4 v = *reinterpret_cast<const float4*>(pr + lane * 4 + 128 * j);
            sum = att_term<F>(w4[j].x, v.x, q4[j].x, sum);
            sum = att_term<F>(w4[j].y, v.y, q4[j].y, sum);
            sum = att_term<F>(w4[j].z, v.z, q4[j].z, sum);
            sum = att_term<F>(w4[j].w, v.w, q4[j].w, sum);
        }
    } else {
        for (int a0 = lane * 4; a0 < A; a0 += 128) {
            const float4 v = *reinterpret_cast<const float4*>(pr + a0);
            const float4 qv = *reinterpret_cast<const float4*>(qs + a0);
            const float4 wv = F == GVD_REGION_ATTN_DP ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(ws + a0);
            sum = att_term<F>(wv.x, v.x, qv.x, sum);
            sum = att_term<F>(wv.y, v.y, qv.y, sum);
            sum = att_term<F>(wv.z, v.z, qv.z, sum);
            sum = att_term<F>(wv.w, v.w, qv.w, sum);
        }
    }
    return sum;
}

// AJ = A/128 when A is 128*{1..4}: queries/weights live in registers; 0 = generic (shared memory).
// FORM = GVD_REGION_ATTN_* of the region chunks (the temporal chunks are always additive).  The shared-memory ring allows 2 CTAs per SM; the
// mul / dp instantiations say so (minBlocks 2, up to 113 registers), which keeps ptxas from spilling their second phase-A loop; mix keeps
// the bounds it always had.
template <int AJ, int FORM>
__global__ void __launch_bounds__(ATT_THREADS, FORM == GVD_REGION_ATTN_MIX ? 0 : 2) attn_partial_kernel(AttnArgs a, int nch_r, int nch_t) {
    extern __shared__ __align__(128) unsigned char smem[];
    float* z_s = reinterpret_cast<float*>(smem + ATT_NST * ATT_STAGE_BYTES);
    float* e_s = z_s + ATT_MAXC;
    float* ml = e_s + ATT_MAXC;                  // [0] = chunk max, [1] = chunk sum
    uint64_t* full = reinterpret_cast<uint64_t*>(ml + 4);
    uint64_t* empty = full + ATT_NST;
    float* qs = reinterpret_cast<float*>(empty + ATT_NST);   // generic path only: q[A], w[A]
    float* ws = qs + a.A;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nch = nch_r + nch_t;
    const int b = blockIdx.x / nch, c = blockIdx.x % nch;      // b = sequence row; fb = the clip whose features it attends over
    const int fb = a.feat_div > 1 ? b / a.feat_div : b;
    const bool region = c < nch_r;
    const int N = region ? a.R : a.T;
    const int chunk = region ? a.RC : a.TC;
    int r0 = region ? c * chunk : (c - nch_r) * chunk;
    int nrows = min(chunk, N - r0);
    long long frow = fb;                                       // feature row block: the clip, or its video
    int n_out = 0;                                             // out-of-window rows this chunk's record stands for (video rows only)
    if (a.vid && !region) {
        const long long lo = max(a.win[2 * fb], 0ll), hi = min(a.win[2 * fb + 1], (long long)N);
        const int wlo = (int)min(lo, (long long)N), whi = (int)max(hi, (long long)wlo);     // window ∩ [0,T), empty -> wlo == whi
        const int c0 = max(r0, wlo), c1 = min(r0 + nrows, whi);
        frow = a.vid[fb];
        if (c == nch_r) n_out = N - (whi - wlo);
        r0 = c0;
        nrows = max(c1 - c0, 0);
    }
    const int A = a.A, H = a.H;
    const float* p_rows = (region ? a.p_pool : a.p_conv) + (frow * N + r0) * A;
    const float* f_rows = (region ? a.pool : a.conv) + (frow * N + r0) * H;
    const int rows_pa = ATT_STAGE_BYTES / (A * 4), rows_pb = ATT_STAGE_BYTES / (H * 4);
    const bool featmap = a.mode == GVD_ATT_INPUT_FEATMAP, dual = a.mode == GVD_ATT_INPUT_DUAL_REGION;
    // featmap: a region chunk's weighted sum never reaches the language LSTM, so its feature rows are not streamed (phase B is empty)
    const int n_pa = (nrows + rows_pa - 1) / rows_pa, n_pb = (featmap && region) ? 0 : (nrows + rows_pb - 1) / rows_pb;

    if (tid == 0) {
        for (int s = 0; s < ATT_NST; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], ATT_CWARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (tid == 0) pdl_trigger();
    if (warp == ATT_CWARPS) {
        // ------------------------------------------------------------ producer: bulk TMA stream (prologue features: constant during the loop,
        // so with programmatic dependent launch the pipeline fills while the query projection before this kernel is still finishing)
        if (lane == 0) {
            for (int i = 0; i < n_pa + n_pb; ++i) {
                const int s = i % ATT_NST;
                const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
                mbar_wait(&empty[s], ph ^ 1u);
                const float* src;
                uint32_t bytes;
                if (i < n_pa) {
                    const int row0 = i * rows_pa, nr = min(rows_pa, nrows - row0);
                    src = p_rows + (long long)row0 * A;
                    bytes = (uint32_t)nr * A * 4u;
                } else {
                    const int row0 = (i - n_pa) * rows_pb, nr = min(rows_pb, nrows - row0);
                    src = f_rows + (long long)row0 * H;
                    bytes = (uint32_t)nr * H * 4u;
                }
                mbar_expect_tx(&full[s], bytes);
                bulk_g2s(smem + (size_t)s * ATT_STAGE_BYTES, src, bytes, &full[s]);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    pdl_wait();                                       // queries come from the predecessor kernel
    if (dual) {
        attn_dual_consumer<FORM>(a, nch_r, b, fb, c, r0, nrows, n_pa, n_pb, rows_pa, rows_pb, smem, full, empty, z_s, e_s, ml, qs);
        return;
    }
    const float* w = region ? a.w2 : a.w1;
    const bool has_w = !(FORM == GVD_REGION_ATTN_DP && region);      // dp: the region attention has no alpha_net (w2 / b2 are NULL)
    const float bias = region ? (FORM == GVD_REGION_ATTN_DP ? 0.f : __ldg(a.b2)) : __ldg(a.b1);
    float4 q4[AJ > 0 ? AJ : 1], w4[AJ > 0 ? AJ : 1];
    const float* q = a.q ? a.q + (long long)b * 2 * A + (region ? A : 0) : qs;
    if (!a.q) {
        // the query projection arrives as split-K partials: this CTA sums its A columns once (no separate reduction launch)
        const float* p0 = a.q_part + (long long)b * 2 * A + (region ? A : 0);
        for (int i = tid; i < A; i += ATT_CWARPS * 32) {
            float v = __ldg(a.q_bias + (region ? A : 0) + i);
            for (int s = 0; s < a.q_S; ++s) v += __ldcg(p0 + s * a.q_plane + i);
            qs[i] = v;
        }
        consumer_bar();
    }
    if (AJ > 0) {
#pragma unroll
        for (int j = 0; j < AJ; ++j) {
            q4[j] = *reinterpret_cast<const float4*>(q + lane * 4 + 128 * j);
            w4[j] = has_w ? __ldg(reinterpret_cast<const float4*>(w + lane * 4 + 128 * j)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    } else {
        if (a.q) { for (int i = tid; i < A; i += ATT_CWARPS * 32) qs[i] = q[i]; }
        if (has_w) for (int i = tid; i < A; i += ATT_CWARPS * 32) ws[i] = w[i];
        consumer_bar();
    }

    // phase A: scores  z_r = w . tanh(p_r + q) + bias  (region chunks: w . tanh(p_r * q) + bias or p_r . q in the other forms).  One loop
    // per form a CTA can run: the form is uniform over the CTA, so no row pays for the other one
    auto phase_a = [&](auto form) {
        constexpr int F = decltype(form)::value;
        for (int i = 0; i < n_pa; ++i) {
            const int s = i % ATT_NST;
            const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
            mbar_wait(&full[s], ph);
            const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
            const int row0 = i * rows_pa, nr = min(rows_pa, nrows - row0);
            for (int rr = warp; rr < nr; rr += ATT_CWARPS) {
                const float* pr = st + (long long)rr * A;
                float sum = att_row_sum<AJ, F>(pr, q4, w4, qs, ws, A, lane);
                sum = warp_sum(sum);
                if (lane == 0) {
                    float z = sum + bias;
                    const int rl = row0 + rr;
                    if (region) {
                        const long long mi = (long long)fb * (a.R + 1) + 1 + r0 + rl;
                        const long long oi = a.out_mask_stride ? (long long)fb * a.out_mask_stride + 1 + r0 + rl : mi;
                        const bool am = a.att_mask[mi] != 0, om = a.out_mask[oi] != 0;
                        if (am) z = GVD_MIN_VALUE;                               // AttModel.py:99
                        a.z_out[(long long)b * a.z_stride_b + r0 + rl] = (am || om) ? GVD_MIN_VALUE : z;   // AttModel.py:100,103
                    }
                    z_s[rl] = z;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    };
    if (FORM != GVD_REGION_ATTN_MIX && region) phase_a(FormTag<FORM>{});
    else phase_a(FormTag<GVD_REGION_ATTN_MIX>{});
    consumer_bar();
    if (warp == 0) {
        float m = -INFINITY, s0 = -INFINITY;
        if (n_out > 0) s0 = warp_sum(att_row_sum<AJ, GVD_REGION_ATTN_MIX>(a.ctx_bias, q4, w4, qs, ws, A, lane)) + bias;   // p_conv row = ctx_bias
        for (int r = lane; r < nrows; r += 32) m = fmaxf(m, z_s[r]);
        m = fmaxf(warp_max(m), s0);
        float l = 0.f;
        for (int r = lane; r < nrows; r += 32) {
            const float e = expf(z_s[r] - m);
            e_s[r] = e;
            l += e;
        }
        l = warp_sum(l);
        if (n_out > 0) l = fmaf((float)n_out, expf(s0 - m), l);
        if (lane == 0) { ml[0] = m; ml[1] = l; }
    }
    consumer_bar();

    // phase B: unnormalised weighted feature sum
    const int h0 = tid * 4;
    const bool active = h0 < H;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < n_pb; ++j) {
        const int i = n_pa + j, s = i % ATT_NST;
        const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
        mbar_wait(&full[s], ph);
        const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
        const int row0 = j * rows_pb, nr = min(rows_pb, nrows - row0);
        if (active) {
            for (int rr = 0; rr < nr; ++rr) {
                const float e = e_s[row0 + rr];
                const float4 v = *reinterpret_cast<const float4*>(st + (long long)rr * H + h0);
                acc.x = fmaf(e, v.x, acc.x);
                acc.y = fmaf(e, v.y, acc.y);
                acc.z = fmaf(e, v.z, acc.z);
                acc.w = fmaf(e, v.w, acc.w);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    float* out = a.partial + ((long long)b * nch + c) * (H + 4);
    if (tid == 0) { out[0] = ml[0]; out[1] = ml[1]; }
    // (featmap region chunks: no weighted sum to store; a video row's temporal chunk outside its window stores its zero sum)
    if (active && !(featmap && region)) *reinterpret_cast<float4*>(out + 4 + h0) = acc;
    if (a.ticket == nullptr) return;
    // ---- fused combine: the last CTA of this row to finish merges all chunk partials (flash-decoding style).
    // Fixed merge order (chunk index), so the result does not depend on which CTA happens to be last.
    __threadfence();                                   // publish this CTA's partial before taking a ticket
    consumer_bar();
    int* flag = reinterpret_cast<int*>(ml + 2);
    if (tid == 0) *flag = (atomicAdd(a.ticket + b, 1) == nch - 1) ? 1 : 0;
    consumer_bar();
    if (*flag == 0) return;
    __threadfence();
    const float* base = a.partial + (long long)b * nch * (H + 4);
    if (active) {
        float4 res = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int part = 0; part < 2; ++part) {
            if (part == 1 && featmap) break;                               // featmap: x = att
            const int c0 = part ? 0 : nch_r, c1 = part ? nch_r : nch;      // temporal chunks, then region chunks
            float M = -INFINITY;
            for (int cc = c0; cc < c1; ++cc) M = fmaxf(M, __ldcg(base + (long long)cc * (H + 4)));
            float L = 0.f;
            float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int cc = c0; cc < c1; ++cc) {
                const float* pc = base + (long long)cc * (H + 4);
                const float sc = expf(__ldcg(pc) - M);
                L = fmaf(__ldcg(pc + 1), sc, L);
                const float4 v = __ldcg(reinterpret_cast<const float4*>(pc + 4 + h0));
                s4.x = fmaf(v.x, sc, s4.x); s4.y = fmaf(v.y, sc, s4.y); s4.z = fmaf(v.z, sc, s4.z); s4.w = fmaf(v.w, sc, s4.w);
            }
            res.x += s4.x / L; res.y += s4.y / L; res.z += s4.z / L; res.w += s4.w / L;
        }
        *reinterpret_cast<float4*>(a.x_out + (long long)b * (a.x_ld ? a.x_ld : H) + h0) = res;
        if (a.x_pk) {
            uint32_t hi0, lo0, hi1, lo1;
            f16x3_split_pair(res.x, res.y, GVD_F16_SA, hi0, lo0);
            f16x3_split_pair(res.z, res.w, GVD_F16_SA, hi1, lo1);
            uint32_t* d = reinterpret_cast<uint32_t*>(a.x_pk) + (long long)b * a.x_pk_ld + f16x3_word(h0);
            *reinterpret_cast<uint2*>(d) = make_uint2(hi0, hi1);
            *reinterpret_cast<uint2*>(d + 16) = make_uint2(lo0, lo1);
        }
    }
    if (tid == 0) a.ticket[b] = 0;                       // ready for the next step
}

// =====================================================================================
// row-grouped attention partials: up to ATT_GMAX rows that attend over one clip's features (sampled captions, beam rows) per CTA
// =====================================================================================
// ATT_GMAX = ATT_CWARPS: one softmax warp per row of the group, and at A = 512 the group's queries (G * A floats, twice in dual_region) and
// score vectors still fit next to the 96 KB ring in one CTA's shared memory (up to ~150 KB); phase B keeps G (dual: 2 G) float4 accumulators
// per thread in registers.  The decode does not select this kernel (gvd_attn_partial, DESIGN §3: slower than the per-row kernel on the same
// shared features at the measured rows per clip); gvd_op_attention_path runs it.
constexpr int ATT_GMAX = ATT_CWARPS;

// att_row_sum with the query in shared memory (the row group's queries do not fit in registers).  The same terms in the same order as
// att_row_sum on register queries: AJ > 0 takes the projected row from v4 (registers, loaded once for every query of the group).
template <int AJ, int F>
__device__ __forceinline__ float att_row_sum_sq(const float4* v4, const float* pr, const float* qg, const float4* w4, const float* ws, int A,
                                                int lane) {
    float sum = 0.f;
    if (AJ > 0) {
#pragma unroll
        for (int j = 0; j < AJ; ++j) {
            const float4 qv = *reinterpret_cast<const float4*>(qg + lane * 4 + 128 * j);
            sum = att_term<F>(w4[j].x, v4[j].x, qv.x, sum);
            sum = att_term<F>(w4[j].y, v4[j].y, qv.y, sum);
            sum = att_term<F>(w4[j].z, v4[j].z, qv.z, sum);
            sum = att_term<F>(w4[j].w, v4[j].w, qv.w, sum);
        }
    } else {
        for (int a0 = lane * 4; a0 < A; a0 += 128) {
            const float4 v = *reinterpret_cast<const float4*>(pr + a0);
            const float4 qv = *reinterpret_cast<const float4*>(qg + a0);
            const float4 wv = F == GVD_REGION_ATTN_DP ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4*>(ws + a0);
            sum = att_term<F>(wv.x, v.x, qv.x, sum);
            sum = att_term<F>(wv.y, v.y, qv.y, sum);
            sum = att_term<F>(wv.z, v.z, qv.z, sum);
            sum = att_term<F>(wv.w, v.w, qv.w, sum);
        }
    }
    return sum;
}

// sum_c acc_c e^{m_c - M} / sum_c l_c e^{m_c - M} over the chunk records [c0, c1) of one row: attn_partial_kernel's merge, chunk for chunk
__device__ __forceinline__ float4 merge_part(const float* base, int c0, int c1, int H, int h0) {
    float M = -INFINITY;
    for (int cc = c0; cc < c1; ++cc) M = fmaxf(M, __ldcg(base + (long long)cc * (H + 4)));
    float L = 0.f;
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int cc = c0; cc < c1; ++cc) {
        const float* pc = base + (long long)cc * (H + 4);
        const float sc = expf(__ldcg(pc) - M);
        L = fmaf(__ldcg(pc + 1), sc, L);
        const float4 v = __ldcg(reinterpret_cast<const float4*>(pc + 4 + h0));
        s4.x = fmaf(v.x, sc, s4.x); s4.y = fmaf(v.y, sc, s4.y); s4.z = fmaf(v.z, sc, s4.z); s4.w = fmaf(v.w, sc, s4.w);
    }
    return make_float4(s4.x / L, s4.y / L, s4.z / L, s4.w / L);
}

__device__ __forceinline__ void store_x(const AttnArgs& a, int b, int h0, float4 res) {
    *reinterpret_cast<float4*>(a.x_out + (long long)b * (a.x_ld ? a.x_ld : a.H) + h0) = res;
    if (a.x_pk) {
        uint32_t hi0, lo0, hi1, lo1;
        f16x3_split_pair(res.x, res.y, GVD_F16_SA, hi0, lo0);
        f16x3_split_pair(res.z, res.w, GVD_F16_SA, hi1, lo1);
        uint32_t* d = reinterpret_cast<uint32_t*>(a.x_pk) + (long long)b * a.x_pk_ld + f16x3_word(h0);
        *reinterpret_cast<uint2*>(d) = make_uint2(hi0, hi1);
        *reinterpret_cast<uint2*>(d + 16) = make_uint2(lo0, lo1);
    }
}

// Every row of the group equals attn_partial_kernel's result for that row bit for bit: the same chunks, the same lane -> element mapping of
// the scores (att_row_sum_sq), the same warp_sum trees, the same per-row softmax and weighted-sum order, the same merge.  Grid: (clip, row
// group, chunk); the group's rows b0 .. b0 + G - 1 share the clip's features, masks and (video rows) window, so each chunk's projected and
// feature rows are streamed once for all G queries.  The group's last chunk CTA (ticket of row b0) merges all its rows.
template <int AJ, int FORM>
__global__ void __launch_bounds__(ATT_THREADS, 1) attn_group_kernel(AttnArgs a, int nch_r, int nch_t, int ngroups) {
    extern __shared__ __align__(128) unsigned char smem[];
    const bool featmap = a.mode == GVD_ATT_INPUT_FEATMAP, dual = a.mode == GVD_ATT_INPUT_DUAL_REGION;
    const int nq = dual ? 2 : 1;                                // score vectors per row
    const int A = a.A, H = a.H;
    float* z_s = reinterpret_cast<float*>(smem + ATT_NST * ATT_STAGE_BYTES);   // [nq][GMAX][MAXC] (dual: attention2, then attention2_dual)
    float* e_s = z_s + nq * ATT_GMAX * ATT_MAXC;                               // [nq][GMAX][MAXC]
    float* ml = e_s + nq * ATT_GMAX * ATT_MAXC;                                // [nq][GMAX][2] + merge flag
    float* red = ml + 2 * nq * ATT_GMAX + 4;                                   // [GMAX][CWARPS] gate partial sums
    uint64_t* full = reinterpret_cast<uint64_t*>(red + ATT_GMAX * ATT_CWARPS);
    uint64_t* empty = full + ATT_NST;
    float* qs = reinterpret_cast<float*>(empty + ATT_NST);     // [nq][GMAX][A] (dual: attention2 queries, then the dual ones)
    float* ws = qs + nq * ATT_GMAX * A;                         // [nq][A]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nch = nch_r + nch_t;
    const int c = blockIdx.x % nch, grp = (blockIdx.x / nch) % ngroups, fb = blockIdx.x / nch / ngroups;
    const int div = a.feat_div > 1 ? a.feat_div : 1;
    const int g0 = grp * ATT_GMAX, G = min(ATT_GMAX, div - g0), b0 = fb * div + g0;
    const bool region = c < nch_r;
    const int N = region ? a.R : a.T;
    const int chunk = region ? a.RC : a.TC;
    int r0 = region ? c * chunk : (c - nch_r) * chunk;
    int nrows = min(chunk, N - r0);
    long long frow = fb;
    int n_out = 0;
    if (a.vid && !region) {
        const long long lo = max(a.win[2 * fb], 0ll), hi = min(a.win[2 * fb + 1], (long long)N);
        const int wlo = (int)min(lo, (long long)N), whi = (int)max(hi, (long long)wlo);
        const int c0 = max(r0, wlo), c1 = min(r0 + nrows, whi);
        frow = a.vid[fb];
        if (c == nch_r) n_out = N - (whi - wlo);
        r0 = c0;
        nrows = max(c1 - c0, 0);
    }
    const float* p_rows = (region ? a.p_pool : a.p_conv) + (frow * N + r0) * A;
    const float* f_rows = (region ? a.pool : a.conv) + (frow * N + r0) * H;
    const int rows_pa = ATT_STAGE_BYTES / (A * 4), rows_pb = ATT_STAGE_BYTES / (H * 4);
    const int n_pa = (nrows + rows_pa - 1) / rows_pa, n_pb = (featmap && region) ? 0 : (nrows + rows_pb - 1) / rows_pb;

    if (tid == 0) {
        for (int s = 0; s < ATT_NST; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], ATT_CWARPS);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (tid == 0) pdl_trigger();
    if (warp == ATT_CWARPS) {
        if (lane == 0) {
            for (int i = 0; i < n_pa + n_pb; ++i) {
                const int s = i % ATT_NST;
                const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
                mbar_wait(&empty[s], ph ^ 1u);
                const float* src;
                uint32_t bytes;
                if (i < n_pa) {
                    const int row0 = i * rows_pa, nr = min(rows_pa, nrows - row0);
                    src = p_rows + (long long)row0 * A;
                    bytes = (uint32_t)nr * A * 4u;
                } else {
                    const int row0 = (i - n_pa) * rows_pb, nr = min(rows_pb, nrows - row0);
                    src = f_rows + (long long)row0 * H;
                    bytes = (uint32_t)nr * H * 4u;
                }
                mbar_expect_tx(&full[s], bytes);
                bulk_g2s(smem + (size_t)s * ATT_STAGE_BYTES, src, bytes, &full[s]);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    pdl_wait();
    // the group's queries: row b's slice q[b, off .. off + A) (or its split-K partials summed onto the bias in plane order); dual_region
    // keeps attention2's query (second half) in slot 0 and the dual query (first half) in slot 1
    for (int qi = 0; qi < nq; ++qi) {
        const int off = dual ? (qi == 0 ? A : 0) : (region ? A : 0);
        for (int i = tid; i < G * A; i += ATT_CWARPS * 32) {
            const int g = i / A, k = i - g * A;
            const long long at = (long long)(b0 + g) * 2 * A + off + k;
            float v;
            if (a.q) {
                v = a.q[at];
            } else {
                v = __ldg(a.q_bias + off + k);
                for (int s = 0; s < a.q_S; ++s) v += __ldcg(a.q_part + s * a.q_plane + at);
            }
            qs[(qi * ATT_GMAX + g) * A + k] = v;
        }
    }
    const bool has_w = !(FORM == GVD_REGION_ATTN_DP && (region || dual));
    const float* w = dual ? a.w2 : (region ? a.w2 : a.w1);
    const float bias = has_w ? __ldg(dual ? a.b2 : (region ? a.b2 : a.b1)) : 0.f;
    const float bias_d = dual && has_w ? __ldg(a.b1) : 0.f;
    if (has_w) {
        for (int i = tid; i < A; i += ATT_CWARPS * 32) ws[i] = w[i];
        if (dual) for (int i = tid; i < A; i += ATT_CWARPS * 32) ws[A + i] = a.w1[i];
    }
    float4 w4[AJ > 0 ? AJ : 1];
    if (AJ > 0 && !dual) {
#pragma unroll
        for (int j = 0; j < AJ; ++j) w4[j] = has_w ? __ldg(reinterpret_cast<const float4*>(w + lane * 4 + 128 * j)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    consumer_bar();

    // phase A: the scores of every streamed row against each of the group's queries
    auto phase_a = [&](auto form) {
        constexpr int F = decltype(form)::value;
        for (int i = 0; i < n_pa; ++i) {
            const int s = i % ATT_NST;
            const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
            mbar_wait(&full[s], ph);
            const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
            const int row0 = i * rows_pa, nr = min(rows_pa, nrows - row0);
            for (int rr = warp; rr < nr; rr += ATT_CWARPS) {
                const float* pr = st + (long long)rr * A;
                const int rl = row0 + rr;
                bool am = false, om = false;
                if (region && lane == 0) {
                    const long long mi = (long long)fb * (a.R + 1) + 1 + r0 + rl;
                    const long long oi = a.out_mask_stride ? (long long)fb * a.out_mask_stride + 1 + r0 + rl : mi;
                    am = a.att_mask[mi] != 0;
                    om = a.out_mask[oi] != 0;
                }
                if (dual) {
                    // attn_dual_consumer's generic loop: both scores from one read of each element
                    for (int g = 0; g < G; ++g) {
                        const float* q2 = qs + g * A;
                        const float* qd = qs + (ATT_GMAX + g) * A;
                        float sum = 0.f, sum_d = 0.f;
                        for (int a0 = lane * 4; a0 < A; a0 += 128) {
                            const float4 v = *reinterpret_cast<const float4*>(pr + a0);
                            const float4 qv = *reinterpret_cast<const float4*>(q2 + a0), wv = *reinterpret_cast<const float4*>(ws + a0);
                            const float4 qv2 = *reinterpret_cast<const float4*>(qd + a0), wv2 = *reinterpret_cast<const float4*>(ws + A + a0);
                            sum = att_term<F>(wv.x, v.x, qv.x, sum);
                            sum = att_term<F>(wv.y, v.y, qv.y, sum);
                            sum = att_term<F>(wv.z, v.z, qv.z, sum);
                            sum = att_term<F>(wv.w, v.w, qv.w, sum);
                            sum_d = att_term<F>(wv2.x, v.x, qv2.x, sum_d);
                            sum_d = att_term<F>(wv2.y, v.y, qv2.y, sum_d);
                            sum_d = att_term<F>(wv2.z, v.z, qv2.z, sum_d);
                            sum_d = att_term<F>(wv2.w, v.w, qv2.w, sum_d);
                        }
                        sum = warp_sum(sum);
                        sum_d = warp_sum(sum_d);
                        if (lane == 0) {
                            float z = sum + bias, zd = sum_d + bias_d;
                            if (am) { z = GVD_MIN_VALUE; zd = GVD_MIN_VALUE; }
                            a.z_out[(long long)(b0 + g) * a.z_stride_b + r0 + rl] = (am || om) ? GVD_MIN_VALUE : z;
                            z_s[g * ATT_MAXC + rl] = z;
                            z_s[(ATT_GMAX + g) * ATT_MAXC + rl] = zd;
                        }
                    }
                } else {
                    float4 v4[AJ > 0 ? AJ : 1];
                    if (AJ > 0) {
#pragma unroll
                        for (int j = 0; j < AJ; ++j) v4[j] = *reinterpret_cast<const float4*>(pr + lane * 4 + 128 * j);
                    }
                    for (int g = 0; g < G; ++g) {
                        float sum = att_row_sum_sq<AJ, F>(v4, pr, qs + g * A, w4, ws, A, lane);
                        sum = warp_sum(sum);
                        if (lane == 0) {
                            float z = sum + bias;
                            if (region) {
                                if (am) z = GVD_MIN_VALUE;
                                a.z_out[(long long)(b0 + g) * a.z_stride_b + r0 + rl] = (am || om) ? GVD_MIN_VALUE : z;
                            }
                            z_s[g * ATT_MAXC + rl] = z;
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    };
    if (FORM != GVD_REGION_ATTN_MIX && (region || dual)) phase_a(FormTag<FORM>{});
    else phase_a(FormTag<GVD_REGION_ATTN_MIX>{});
    consumer_bar();
    // one warp per (score vector, row): the chunk softmax numerators, max and sum (the out-of-window term with that row's query)
    for (int k = warp; k < nq * G; k += ATT_CWARPS) {
        const int qi = k / G, g = k - qi * G;
        const float* zz = z_s + (qi * ATT_GMAX + g) * ATT_MAXC;
        float* ee = e_s + (qi * ATT_GMAX + g) * ATT_MAXC;
        float m = -INFINITY, s0 = -INFINITY;
        if (n_out > 0) {
            float4 v4[AJ > 0 ? AJ : 1];
            if (AJ > 0) {
#pragma unroll
                for (int j = 0; j < AJ; ++j) v4[j] = *reinterpret_cast<const float4*>(a.ctx_bias + lane * 4 + 128 * j);
            }
            s0 = warp_sum(att_row_sum_sq<AJ, GVD_REGION_ATTN_MIX>(v4, a.ctx_bias, qs + g * A, w4, ws, A, lane)) + bias;
        }
        for (int r = lane; r < nrows; r += 32) m = fmaxf(m, zz[r]);
        m = fmaxf(warp_max(m), s0);
        float l = 0.f;
        for (int r = lane; r < nrows; r += 32) {
            const float e = expf(zz[r] - m);
            ee[r] = e;
            l += e;
        }
        l = warp_sum(l);
        if (n_out > 0) l = fmaf((float)n_out, expf(s0 - m), l);
        if (lane == 0) { ml[2 * k] = m; ml[2 * k + 1] = l; }
    }
    consumer_bar();

    // phase B: each row's unnormalised weighted sum from one read of each feature row
    const int h0 = tid * 4;
    const bool active = h0 < H;
    float4 acc[ATT_GMAX], acc_d[ATT_GMAX];
#pragma unroll
    for (int g = 0; g < ATT_GMAX; ++g) { acc[g] = make_float4(0.f, 0.f, 0.f, 0.f); acc_d[g] = acc[g]; }
    for (int j = 0; j < n_pb; ++j) {
        const int i = n_pa + j, s = i % ATT_NST;
        const uint32_t ph = (uint32_t)(i / ATT_NST) & 1u;
        mbar_wait(&full[s], ph);
        const float* st = reinterpret_cast<const float*>(smem + (size_t)s * ATT_STAGE_BYTES);
        const int row0 = j * rows_pb, nr = min(rows_pb, nrows - row0);
        if (active) {
            for (int rr = 0; rr < nr; ++rr) {
                const float4 v = *reinterpret_cast<const float4*>(st + (long long)rr * H + h0);
#pragma unroll
                for (int g = 0; g < ATT_GMAX; ++g) {
                    if (g < G) {
                        const float e = e_s[g * ATT_MAXC + row0 + rr];
                        acc[g].x = fmaf(e, v.x, acc[g].x); acc[g].y = fmaf(e, v.y, acc[g].y);
                        acc[g].z = fmaf(e, v.z, acc[g].z); acc[g].w = fmaf(e, v.w, acc[g].w);
                        if (dual) {
                            const float ed = e_s[(ATT_GMAX + g) * ATT_MAXC + row0 + rr];
                            acc_d[g].x = fmaf(ed, v.x, acc_d[g].x); acc_d[g].y = fmaf(ed, v.y, acc_d[g].y);
                            acc_d[g].z = fmaf(ed, v.z, acc_d[g].z); acc_d[g].w = fmaf(ed, v.w, acc_d[g].w);
                        }
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }
    const int nrec = dual ? 2 * nch_r : nch;
#pragma unroll
    for (int g = 0; g < ATT_GMAX; ++g) {
        if (g < G) {
            float* out = a.partial + ((long long)(b0 + g) * nrec + c) * (H + 4);
            if (tid == 0) { out[0] = ml[2 * g]; out[1] = ml[2 * g + 1]; }
            if (active && !(featmap && region)) *reinterpret_cast<float4*>(out + 4 + h0) = acc[g];
            if (dual) {
                float* out_d = a.partial + ((long long)(b0 + g) * nrec + nch_r + c) * (H + 4);
                if (tid == 0) { out_d[0] = ml[2 * (G + g)]; out_d[1] = ml[2 * (G + g) + 1]; }
                if (active) *reinterpret_cast<float4*>(out_d + 4 + h0) = acc_d[g];
            }
        }
    }
    if (a.ticket == nullptr) return;
    // ---- fused merge by the group's last chunk CTA, row by row in attn_partial_kernel's fixed chunk order
    __threadfence();
    consumer_bar();
    int* flag = reinterpret_cast<int*>(ml + 2 * nq * ATT_GMAX);
    if (tid == 0) *flag = (atomicAdd(a.ticket + b0, 1) == nch - 1) ? 1 : 0;
    consumer_bar();
    if (*flag == 0) return;
    __threadfence();
    if (dual) {
        // g = sigmoid(dual_pointer(h_att)) per row: per-thread partial dot, warp sums, the 8 warp sums added in warp order
        for (int g = 0; g < G; ++g) {
            float gd = 0.f;
            if (active) {
                const float4 hv = *reinterpret_cast<const float4*>(a.gate_h + (long long)(b0 + g) * a.gate_ld + h0);
                const float4 wv = __ldg(reinterpret_cast<const float4*>(a.gate_w + h0));
                gd = fmaf(wv.x, hv.x, gd); gd = fmaf(wv.y, hv.y, gd); gd = fmaf(wv.z, hv.z, gd); gd = fmaf(wv.w, hv.w, gd);
            }
            gd = warp_sum(gd);
            if (lane == 0) red[g * ATT_CWARPS + warp] = gd;
        }
        consumer_bar();
    }
    for (int g = 0; g < G; ++g) {
        const int b = b0 + g;
        const float* base = a.partial + (long long)b * nrec * (H + 4);
        if (dual) {
            float glogit = __ldg(a.gate_b);
            for (int wv = 0; wv < ATT_CWARPS; ++wv) glogit += red[g * ATT_CWARPS + wv];
            const float gt = sigmoid_acc(glogit);
            if (active) {
                const float4 r0v = merge_part(base, 0, nch_r, H, h0), r1v = merge_part(base, nch_r, 2 * nch_r, H, h0);
                const float h = 1.f - gt;
                store_x(a, b, h0, make_float4(gt * r0v.x + h * r1v.x, gt * r0v.y + h * r1v.y, gt * r0v.z + h * r1v.z, gt * r0v.w + h * r1v.w));
            }
        } else if (active) {
            float4 res = make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 t = merge_part(base, nch_r, nch, H, h0);                  // temporal chunks, then region chunks
            res.x += t.x; res.y += t.y; res.z += t.z; res.w += t.w;
            if (!featmap) {
                const float4 r = merge_part(base, 0, nch_r, H, h0);
                res.x += r.x; res.y += r.y; res.z += r.z; res.w += r.w;
            }
            store_x(a, b, h0, res);
        }
    }
    if (tid == 0) a.ticket[b0] = 0;
}

// merge chunk partials: att = sum_c acc_c e^{m_c - M} / sum_c l_c e^{m_c - M}; x = att(temporal) + att2(region) (featmap: att only)
__global__ void __launch_bounds__(256) attn_combine_kernel(const float* __restrict__ partial, float* __restrict__ x_out, int H,
                                                           int nch_r, int nch_t, int nparts) {
    const int b = blockIdx.x, nch = nch_r + nch_t;
    const float* base = partial + (long long)b * nch * (H + 4);
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
        float res = 0.f;
        for (int part = 0; part < nparts; ++part) {
            const int c0 = part ? 0 : nch_r, c1 = part ? nch_r : nch;   // part 0: temporal chunks, part 1: region chunks
            float M = -INFINITY;
            for (int c = c0; c < c1; ++c) M = fmaxf(M, base[(long long)c * (H + 4)]);
            float L = 0.f, acc = 0.f;
            for (int c = c0; c < c1; ++c) {
                const float* pc = base + (long long)c * (H + 4);
                const float sc = expf(pc[0] - M);
                L = fmaf(pc[1], sc, L);
                acc = fmaf(pc[4 + h], sc, acc);
            }
            res += acc / L;
        }
        x_out[(long long)b * H + h] = res;
    }
}

// =====================================================================================
// greedy sampler
// =====================================================================================
struct Top2 { float v1, v2; int i1, i2; };
__device__ __forceinline__ void top2_insert(Top2& t, float v, int i) {
    if (v > t.v1 || (v == t.v1 && i < t.i1)) { t.v2 = t.v1; t.i2 = t.i1; t.v1 = v; t.i1 = i; }
    else if (v > t.v2 || (v == t.v2 && i < t.i2)) { t.v2 = v; t.i2 = i; }
}

__global__ void __launch_bounds__(256) greedy_pick_kernel(const float* __restrict__ logits, long long ld, int V, int unk_idx,
                                                          long long* __restrict__ it_out, long long* __restrict__ seq_out,
                                                          float* __restrict__ logp_out, long long out_stride,
                                                          const float* __restrict__ embed, float* __restrict__ xt, int E, long long ld_xt) {
    __shared__ float red[32];
    __shared__ Top2 wtop[8];
    __shared__ int tok_s;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* x = logits + (long long)b * ld;
    Top2 t{-INFINITY, -INFINITY, 0x7fffffff, 0x7fffffff};
    for (int i = threadIdx.x; i < V; i += blockDim.x) top2_insert(t, x[i], i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov1 = __shfl_xor_sync(0xffffffffu, t.v1, o), ov2 = __shfl_xor_sync(0xffffffffu, t.v2, o);
        const int oi1 = __shfl_xor_sync(0xffffffffu, t.i1, o), oi2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
        top2_insert(t, ov1, oi1);
        top2_insert(t, ov2, oi2);
    }
    if (lane == 0) wtop[warp] = t;
    __syncthreads();
    t = wtop[0];
    for (int wv = 1; wv < 8; ++wv) { top2_insert(t, wtop[wv].v1, wtop[wv].i1); top2_insert(t, wtop[wv].v2, wtop[wv].i2); }
    const float m = t.v1;
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x) s += expf(x[i] - m);
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        const float lse = m + logf(s);
        const bool keep = t.i1 != unk_idx;                       // misc/model.py:590-594
        int it = keep ? t.i1 : t.i2;
        if ((unsigned)it >= (unsigned)V) it = 0;                 // every logit NaN: no comparison succeeded; stay inside the embedding table
        const float lp = (keep ? t.v1 : t.v2) - lse;
        it_out[b] = it;
        if (seq_out) seq_out[(long long)b * out_stride] = it;
        if (logp_out) logp_out[(long long)b * out_stride] = lp;
        tok_s = it;
    }
    if (xt) {                                   // next step's input xt = ReLU(embed[token]) (model.py:79-82,605): saves a launch
        __syncthreads();
        const float* row = embed + (long long)tok_s * E;
        for (int e = threadIdx.x; e < E; e += blockDim.x) xt[(long long)b * ld_xt + e] = fmaxf(row[e], 0.f);
    }
}

__global__ void tanh_test_kernel(const float* x, float* y, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = tanh_mufu(x[i]);
}

}  // namespace

// =====================================================================================
// host launchers
// =====================================================================================
int gvd_lstm_step(const LstmArgs& a, cudaStream_t st) {
    GVD_REQUIRE(a.nseg >= 1 && a.nseg <= 3, "lstm: nseg=%d", a.nseg);
    GVD_REQUIRE(a.H % 4 == 0, "lstm: H must be a multiple of 4");
    for (int s = 0; s < a.nseg; ++s)
        GVD_REQUIRE(a.seg[s].K % 4 == 0 && a.seg[s].ldx % 4 == 0 && a.seg[s].ldw % 4 == 0 && a.seg[s].K > 0,
                    "lstm: segment %d K/ldx/ldw must be multiples of 4", s);
    dim3 grid(gvd_cdiv(a.H, L_UJ), gvd_cdiv(a.B, L_BM));
    lstm_step_kernel<<<grid, L_NT, 0, st>>>(a);
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_attn_chunks(int R, int T, int RC, int TC, int* nch_r, int* nch_t) {
    *nch_r = gvd_cdiv(R, RC);
    *nch_t = gvd_cdiv(T, TC);
    return 0;
}

static size_t attn_smem_bytes(int A, bool dual) {
    return (size_t)ATT_NST * ATT_STAGE_BYTES + (2 * ATT_MAXC + 4) * sizeof(float) + 2 * ATT_NST * sizeof(uint64_t) +
           2 * (size_t)A * sizeof(float) + 16 + (dual ? (2 * (size_t)A + 2 * ATT_MAXC + 4) * sizeof(float) : 0);
}

// the row-grouped kernel: the ring, [nq][GMAX][MAXC] scores and numerators, [nq][GMAX][2] records + flag, the gate sums, the barriers,
// [nq][GMAX][A] queries and [nq][A] alpha_net weights (nq = 2 score vectors per row in dual_region)
static size_t attn_group_smem_bytes(int A, bool dual) {
    const size_t nq = dual ? 2 : 1;
    return (size_t)ATT_NST * ATT_STAGE_BYTES + (2 * nq * ATT_GMAX * ATT_MAXC + 2 * nq * ATT_GMAX + 4 + ATT_GMAX * ATT_CWARPS) * sizeof(float) +
           2 * ATT_NST * sizeof(uint64_t) + (nq * ATT_GMAX + nq) * (size_t)A * sizeof(float);
}

// The decode runs the per-row kernel at every rows-per-clip: on the same shared features it measured faster than the row-grouped kernel
// at 2, 3, 5, 16 and 32 rows per clip and within 3 % either way at 8 (DESIGN §3, tools/sample_n_bench.py --part paths)
int gvd_attn_partial(const AttnArgs& a, cudaStream_t st) { return gvd_attn_partial_path(a, 0, st); }

int gvd_attn_partial_path(const AttnArgs& a, int path, cudaStream_t st) {
    GVD_REQUIRE(a.mode == GVD_ATT_INPUT_BOTH || a.mode == GVD_ATT_INPUT_FEATMAP || a.mode == GVD_ATT_INPUT_DUAL_REGION,
                "attn: unknown att_input_mode %d", a.mode);
    const bool dual = a.mode == GVD_ATT_INPUT_DUAL_REGION;
    GVD_REQUIRE(!dual || (a.ticket && a.gate_w && a.gate_b && a.gate_h && a.gate_ld >= a.H), "attn: dual_region needs the fused merge and the gate");
    GVD_REQUIRE(a.form == GVD_REGION_ATTN_MIX || a.form == GVD_REGION_ATTN_MIX_MUL || a.form == GVD_REGION_ATTN_DP,
                "attn: unknown region_attn_mode %d", a.form);
    const bool region_w = a.form != GVD_REGION_ATTN_DP;                // dp: no region alpha_net
    GVD_REQUIRE((dual ? (!region_w || (a.w1 && a.b1)) : (a.w1 && a.b1)) && (!region_w || (a.w2 && a.b2)), "attn: missing alpha_net weights");
    GVD_REQUIRE(a.A % 4 == 0 && a.H % 4 == 0, "attn: A and H must be multiples of 4");
    GVD_REQUIRE(a.A * 4 <= ATT_STAGE_BYTES && a.H * 4 <= ATT_STAGE_BYTES, "attn: row larger than a pipeline stage");
    GVD_REQUIRE(a.H <= ATT_CWARPS * 32 * 4, "attn: H=%d > %d not supported", a.H, ATT_CWARPS * 32 * 4);
    GVD_REQUIRE(a.RC >= 1 && a.RC <= ATT_MAXC && a.TC >= 1 && a.TC <= ATT_MAXC, "attn: chunk rows must be in [1,%d]", ATT_MAXC);
    GVD_REQUIRE(!a.vid || (a.win && a.ctx_bias && ((uintptr_t)a.ctx_bias & 15) == 0),
                "attn: video rows need the windows and a 16-byte aligned ctx2att bias");
    int nch_r, nch_t;
    gvd_attn_chunks(a.R, a.T, a.RC, a.TC, &nch_r, &nch_t);
    if (dual) nch_t = 0;                         // no temporal attention (AttModel.py:126-128: the frame features are dummies)
    GVD_REQUIRE(path == 0 || path == 1, "attn: unknown path %d", path);
    const bool grouped = path == 1;
    const int div = a.feat_div > 1 ? a.feat_div : 1;
    GVD_REQUIRE(!grouped || a.B % div == 0, "attn: B=%d rows is not a multiple of feat_div=%d", a.B, div);
    const int ngroups = gvd_cdiv(div, ATT_GMAX);
    const size_t smem = grouped ? attn_group_smem_bytes(a.A, dual) : attn_smem_bytes(a.A, dual);
    GVD_REQUIRE(smem <= 227 * 1024, "attn: A=%d needs %zu bytes of shared memory", a.A, smem);
    const unsigned grid = grouped ? (unsigned)(a.B / div) * (unsigned)ngroups * (unsigned)(nch_r + nch_t) : (unsigned)a.B * (unsigned)(nch_r + nch_t);
    const int aj = (a.A % 128 == 0 && a.A / 128 <= 4) ? a.A / 128 : 0;
#define GVD_ATT_LAUNCH(AJ, F)                                                                                                   \
    do {                                                                                                                        \
        if (grouped) {                                                                                                          \
            GVD_CHECK_CUDA(cudaFuncSetAttribute(attn_group_kernel<AJ, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            GVD_CHECK_CUDA(gvd_launch(attn_group_kernel<AJ, F>, dim3(grid), dim3(ATT_THREADS), smem, st, a, nch_r, nch_t, ngroups)); \
        } else {                                                                                                                \
            GVD_CHECK_CUDA(cudaFuncSetAttribute(attn_partial_kernel<AJ, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            GVD_CHECK_CUDA(gvd_launch(attn_partial_kernel<AJ, F>, dim3(grid), dim3(ATT_THREADS), smem, st, a, nch_r, nch_t));    \
        }                                                                                                                       \
    } while (0)
#define GVD_ATT_FORMS(AJ)                                                                   \
    do {                                                                                    \
        if (a.form == GVD_REGION_ATTN_MIX_MUL) GVD_ATT_LAUNCH(AJ, GVD_REGION_ATTN_MIX_MUL); \
        else if (a.form == GVD_REGION_ATTN_DP) GVD_ATT_LAUNCH(AJ, GVD_REGION_ATTN_DP);      \
        else GVD_ATT_LAUNCH(AJ, GVD_REGION_ATTN_MIX);                                       \
    } while (0)
    switch (aj) {
        case 1: GVD_ATT_FORMS(1); break;
        case 2: GVD_ATT_FORMS(2); break;
        case 3: GVD_ATT_FORMS(3); break;
        case 4: GVD_ATT_FORMS(4); break;
        default: GVD_ATT_FORMS(0); break;
    }
#undef GVD_ATT_FORMS
#undef GVD_ATT_LAUNCH
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_attn_combine(const float* partial, float* x_out, int B, int H, int nch_r, int nch_t, int mode, cudaStream_t st) {
    attn_combine_kernel<<<B, 256, 0, st>>>(partial, x_out, H, nch_r, nch_t, mode == GVD_ATT_INPUT_FEATMAP ? 1 : 2);
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_greedy_pick(const float* logits, long long ld, int B, int V, int unk_idx, long long* it_out, long long* seq_out,
                    float* logp_out, long long out_stride, const float* embed, float* xt, int E, cudaStream_t st, long long ld_xt) {
    GVD_REQUIRE(V >= 2, "pick: vocabulary must have >= 2 entries");
    greedy_pick_kernel<<<B, 256, 0, st>>>(logits, ld, V, unk_idx, it_out, seq_out, logp_out, out_stride, embed, xt, E, ld_xt ? ld_xt : E);
    GVD_CHECK_LAUNCH();
    return 0;
}

int gvd_tanh_test(const float* x, float* y, int n, cudaStream_t st) {
    tanh_test_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(x, y, n);
    GVD_CHECK_LAUNCH();
    return 0;
}
