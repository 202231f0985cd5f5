// gvd-b200: host launchers of the hot-path kernels (internal; the C-ABI is include/gvd_b200.h).
#pragma once
#include "gvd_common.cuh"
#include "gvd_gemm.cuh"

// ---- row-wise prologue kernels (gvd_rowops.cu)
int gvd_frame_mean(const float* segs, float* out, int B, int T, int C, cudaStream_t st);
int gvd_clip_vector(const float* fc_mean, const long long* num, const float* Wseg, const float* bseg, float* xcat, int B,
                    int C, int S, int ld, cudaStream_t st, const long long* rows = nullptr);
int gvd_sim_softmax(float* simT, const unsigned char* pnt_mask, int B, int R, int NC, int ld, cudaStream_t st);
int gvd_transpose(const float* in, float* out, int B, int R, int C, int ld_in, cudaStream_t st);
int gvd_transpose_split(const float* in, float* hi, float* lo, int B, int R, int C, int ld_in, cudaStream_t st);          // + tf32 hi/lo planes
int gvd_split_hilo(const float* in, long long ld_in, float* hi, float* lo, long long ld_out, long long rows, int cols, cudaStream_t st);
int gvd_pool_in(const float* g, const float* ppls, const float* simT, const float* Wloc, const float* bloc, float* out,
                long long rows, int F, int NL, int NC, int ld_sim, int ld_out, int num_frames, cudaStream_t st, float* img = nullptr, int ld_img = 0);
int gvd_add_ln_star(const float* x, const float* a, const float* gamma, const float* beta, float* y, long long rows, int H,
                    cudaStream_t st, float* img = nullptr);
int gvd_scaled_softmax_rows(float* S, long long rows, int cols, long long ld, float inv_scale, cudaStream_t st);
int gvd_gru_pointwise(const float* gi, const float* gh, const float* h_prev, float* h_new, float* out,
                      const long long* sample_idx, int B, int T, int G, int step, cudaStream_t st);

// ---- decode-step kernels (gvd_decode.cu)
struct LstmSeg {
    const float* x;            // [B, K] activations (or an embedding table when gather != nullptr)
    long long ldx;
    const long long* gather;   // optional: row b reads x + gather[b] * ldx   (embedding lookup)
    int relu;                  // apply ReLU to the gathered row (embed = Embedding + ReLU, model.py:79-82)
    const float* w;            // [4H, K] slice of the LSTM weight, row stride ldw
    long long ldw;
    int K;
};
struct LstmArgs {
    LstmSeg seg[3];
    int nseg;
    const float* pre;          // optional [B / pre_div, 4H] additive term (constant part of the gates incl. biases)
    int pre_div;               // rows sharing one `pre` row (beam rows of a clip); 0/1 = one per row
    const float* bias1;        // optional [4H]
    const float* bias2;        // optional [4H]
    const float* c_prev;       // [B, H]
    float* h_out;              // [B, H]
    float* c_out;              // [B, H] (may alias c_prev)
    int B, H;
};
int gvd_lstm_step(const LstmArgs& a, cudaStream_t st);

struct AttnArgs {
    const float* p_pool; const float* pool;     // [B,R,A], [B,R,H]
    const float* p_conv; const float* conv;     // [B,T,A], [B,T,H]
    const float* q;                             // [B, 2A] : temporal query | region query (h2att outputs)
    const float* q_part; int q_S; long long q_plane; const float* q_bias;   // or (q == nullptr) its split-K partials [S][B][2A] + bias: summed here
    const float* w1; const float* b1;           // core.attention.alpha_net   [A], [1]
    const float* w2; const float* b2;           // core.attention2.alpha_net  [A], [1] (NULL in region_attn_mode 'dp')
    const unsigned char* att_mask;              // [B, R+1] softmax mask (leading legacy column)
    const unsigned char* out_mask;              // [B, R+1] additionally applied to the returned logits
    long long out_mask_stride;                  // row stride of out_mask in bytes (0 = R+1): per-step slices of a [B,S,R+1] mask
    float* z_out; long long z_stride_b;         // masked region logits: z_out[b * z_stride_b + r]
    float* partial;                             // [B, nch_r + nch_t, H + 4] : m, l, -, -, acc[H]
    int* ticket;                                // optional [B] zero-initialised counters: the last chunk CTA of a row merges the partials
    float* x_out;                               //   ... into x_out[b * x_ld + h] = att + att2 (saves the separate combine launch)
    long long x_ld;                             //   row pitch of x_out (0 = H): the language LSTM's concatenated input when the split-K path runs
    float* x_pk; long long x_pk_ld;             //   optional fp16x3 operand image of the same row (gvd_common.cuh), scale GVD_F16_SA
    int B, R, T, A, H;
    int RC, TC;                                 // rows per region / temporal chunk (<= 128)
    int feat_div;                               // rows sharing one clip's features/masks (beam rows); 0/1 = one per row
    int mode;                                   // GVD_ATT_INPUT_* (include/gvd_b200.h): BOTH x = att + att2; FEATMAP x = att, the region
                                                //   chunks compute their masked logits (z_out) only and never read `pool`; DUAL_REGION: no
                                                //   temporal chunks, each region chunk scores its rows against both region queries (q = [dual
                                                //   query | attention2 query], w1/b1 = attention2_dual.alpha_net) in ONE pass over p_pool / pool,
                                                //   records [B, 2 * nch_r, H + 4] (attention2 chunks, then the dual ones); the merge writes
                                                //   x = g att2 + (1 - g) att2_dual, g = sigmoid(gate_w . gate_h[b] + gate_b)
    const float* gate_w; const float* gate_b;   // DUAL_REGION: core.dual_pointer.0  [H], [1]
    const float* gate_h; long long gate_ld;     //   h_att rows (pitch gate_ld)
    int form;                                   // GVD_REGION_ATTN_* (include/gvd_b200.h): the region attentions' score (the temporal one is
                                                //   additive in every mode); DP reads no region alpha_net (w2 / b2, and w1 / b1 in DUAL_REGION)
    // Video-indexed frame features (NULL vid: p_conv / conv are per clip).  Clip k attends over video vid[k]'s rows of the UNMASKED
    // p_conv / conv [V,T,A|H], only inside its window [win[2k], win[2k+1]) ∩ [0,T).  The T - n_in rows outside hold zero features and
    // p_conv = ctx_bias in the per-clip path, so they share one score s0 = w1 . tanh(ctx_bias + q) + b1 and add nothing to the weighted
    // sum: the first temporal chunk folds (s0, T - n_in, 0) into its (max, sum, acc) record and no chunk streams an out-of-window row.
    const long long* vid;                       // [B / feat_div] video of each clip
    const long long* win;                       // [B / feat_div, 2] sample_idx
    const float* ctx_bias;                      // [A] ctx2att.bias
};
int gvd_attn_chunks(int R, int T, int RC, int TC, int* nch_r, int* nch_t);
int gvd_attn_partial(const AttnArgs& a, cudaStream_t st);
// path 0 = attn_partial_kernel (one CTA per row and chunk, what gvd_attn_partial runs), 1 = attn_group_kernel (one CTA per group of up to 8
// of a clip's feat_div rows and chunk); both give the same bits per row
int gvd_attn_partial_path(const AttnArgs& a, int path, cudaStream_t st);
int gvd_attn_combine(const float* partial, float* x_out, int B, int H, int nch_r, int nch_t, int mode, cudaStream_t st);
int gvd_greedy_pick(const float* logits, long long ld, int B, int V, int unk_idx, long long* it_out, long long* seq_out,
                    float* logp_out, long long out_stride, const float* embed, float* xt, int E, cudaStream_t st, long long ld_xt = 0);
int gvd_tanh_test(const float* x, float* y, int n, cudaStream_t st);

// ---- beam bookkeeping kernels (gvd_beam.cu)
struct BeamBufs {
    int *seq, *att, *parent, *att_ind, *done_flag, *done_slot, *topi, *done_seq;   // seq/att: [B][L][K]; topi: [B*K][K]
    float *lp, *sums, *topv, *done_lp;                                              // lp: [B][L][K]; sums: [B][K]; topv: [B*K][K]
    long long* tokens;                                                              // [B*K]
    int *parent_hist, *done_step;      // optional (NULL: not kept): every step's parent [L][B*K]; the step at which done_slot finished [B]
};
int gvd_beam_topk(const float* logits, long long ld, int rows, int V, int K, float* topv, int* topi, cudaStream_t st);
int gvd_beam_update(const BeamBufs& bb, int B, int K, int L, int t, cudaStream_t st);
int gvd_beam_gather_rows(const float* src, float* dst, const int* parent, int B, int K, int H, cudaStream_t st);
int gvd_row_argmax(const float* z, long long ld, int rows, int R, int* out, cudaStream_t st);
int gvd_beam_finish(const BeamBufs& bb, const int* bos_att, int B, int K, int L, long long* seq_out, float* lp_out, long long* att_out,
                    cudaStream_t st);
int gvd_beam_backtrack(const BeamBufs& bb, const float* hist, long long step_stride, int B, int K, int L, int R, float* out, cudaStream_t st);

// ---- wgmma / TMA GEMM (gvd_wgmma.cu)
// operand-swapped split-K path for the skinny decode-step products (gvd_skinny.cu; backend bit 3)
int gvd_skinny_splits(int Nw, int Ktot, int B);
int gvd_skinny_splitk(const float* W, int Nw, int Ktot, const float* X, long long ldx, int B, int S, float* part, int ldp, cudaStream_t st);
int gvd_reduce_lstm(const float* part, int S, int ldp, const float* pre, int pre_div, const float* bias1, const float* bias2, const float* c_prev,
                    float* c_out, float* h0, long long ldh0, float* h1, long long ldh1, float* h2, long long ldh2, int B, int H, cudaStream_t st,
                    float* pk1 = nullptr, long long ldpk1 = 0, float* pk2 = nullptr, long long ldpk2 = 0);
// conversion-free fp16x3 product of two operand images (gvd_wgmma.cu: MODE_TRANS with split K)
int gvd_skinny_f16(const float* Wp, long long ldw, int Nw, const float* Xp, long long ldx, int B, int Ktot, int S, float* part, int ldp,
                   cudaStream_t st);
int gvd_reduce_bias(const float* part, int S, int Nw, int ldp, const float* bias, float* out, long long ld_out, int B, cudaStream_t st);
int gvd_reduce_pick(const float* part, int S, int ldp, const float* bias, int B, int V, int unk_idx, long long* it_out, long long* seq_out,
                    float* logp_out, long long out_stride, const float* embed, float* xt, long long ld_xt, int E, float* logits_out,
                    long long ld_logits, cudaStream_t st, float* xt_pk = nullptr, long long ld_xt_pk = 0);
// parameter block of the multinomial sampler, device-resident (a captured decode loop replays with a new seed / temperature)
struct GvdSampleParams { uint32_t seed_lo, seed_hi; float temperature; uint32_t pad; };
int gvd_reduce_sample(const float* part, int S, int ldp, const float* bias, int B, int V, const GvdSampleParams* params, int step,
                      long long* it_out, long long* seq_out, float* logp_out, long long out_stride, const float* embed, float* xt,
                      long long ld_xt, int E, cudaStream_t st, float* xt_pk = nullptr, long long ld_xt_pk = 0);
// Vocabulary head tail for any V (gvd_skinny.cu): one CTA per (row, slice of VOCAB_SLICE words) writes a record of its slice, the last CTA
// of the row merges the records in a fixed order and writes the outputs.  Same destinations as reduce_pick / reduce_sample, plus the
// transformer head's logits copy and teacher-forced nll.
enum { VOCAB_GREEDY = 0, VOCAB_SAMPLE = 1, VOCAB_ARGMAX = 2 };
constexpr int VOCAB_SLICE = 1024;
struct VocabTailArgs {
    const float* part; int S; long long plane; int ldp;      // S planes [B][ldp], plane stride in floats
    const float* bias; int B, V;                             // bias [V] or NULL
    int mode, unk_idx;                                       // VOCAB_GREEDY: top-2 + UNK rule; VOCAB_ARGMAX: first maximum
    const GvdSampleParams* par; int step;                    // VOCAB_SAMPLE: seed, temperature and decode step of the noise
    long long *it_out, *seq_out; float* logp_out; long long out_stride;
    const float* embed; float* xt; long long ld_xt; int E; float* xt_pk; long long ld_xt_pk;
    float* logits_out; long long ld_logits;                  // row b's logits at logits_out + b * ld_logits
    const long long* target; long long target_stride;        // nll[b] = lse - logit[target[b]] (0 unless 0 < target < V)
    float* nll; long long nll_stride;
    float* rec; int* ticket;                                 // [B][gvd_vocab_slices(V)] records; [B] tickets, zero before the first launch
};
inline int gvd_vocab_slices(int V) { return (V + VOCAB_SLICE - 1) / VOCAB_SLICE; }
inline size_t gvd_vocab_rec_floats(int B, int V) { return (size_t)B * gvd_vocab_slices(V) * 8; }
int gvd_vocab_tail(const VocabTailArgs& a, cudaStream_t st);
int gvd_gemm_nt_tc(const GemmArgs& g, int batch, cudaStream_t stream);
int gvd_gemm_nt_astat(const GemmArgs& g, int batch, cudaStream_t stream);   // short-K (<= 192), one K pass
// self-attention pair (W operands pre-split into tf32 hi / lo planes): softmax-numerator scores + group factors F, then (F (.) E) V
int gvd_attn_scores_tc(const GemmArgs& g, const float* W_lo, float* F, float smx_scale, int batch, cudaStream_t stream, int f16 = 0);
int gvd_attn_pv_tc(const GemmArgs& g, const float* W_lo, const float* F, int batch, cudaStream_t stream, int f16 = 0);
int gvd_lstm_step_tc(const LstmArgs& a, cudaStream_t stream);
// fused self-attention (gvd_attn.cu): O[b, r, h] = softmax(Q_h K_h^T * scale) V_h for every clip and head in one launch.  Q fp32 (row b * R + r,
// head h at column h * hs), the key image of gvd_pack_heads_f16x3 (KH = hs rounded up to 32), the V^T image of gvd_transpose_pack_f16x3 (HP
// columns per clip, Rp = R rounded up to 32); O as fp32 (out, pitch ldo) or, when img is given, as the fp16x3 operand image of the next GEMM
int gvd_self_attn_fused(const float* q, long long ldq, const float* k_img, const float* vt_img, int B, int R, int nh, int hs, int HP, float scale,
                        float* out, long long ldo, float* img, long long img_ld, cudaStream_t st);
int gvd_logit_pick_tc(const float* h, long long ldh, const float* W, long long ldw, const float* bias, int B, int V, int K, int unk_idx,
                      float* part, int* ticket, long long* it_out, long long* seq_out, float* logp_out, long long out_stride,
                      const float* embed, float* xt, int E, cudaStream_t stream);

// ---- teacher-forced losses / GRD outputs (gvd_losses.cu)
int gvd_bbox_overlaps(const float* ppls, const float* gt, const unsigned char* frm_mask, const unsigned char* pnt_mask, float* ov, int B, int R,
                      int NB, cudaStream_t st);
int gvd_cls_target(const float* ov, const float* gt, const float* simT, int* target, float* part_sum, int* part_cnt, int B, int R, int NB,
                   int NC, int ld_sim, cudaStream_t st);
int gvd_class_argmax(const float* simT, int* pred, long long rows, int NC, int ld, cudaStream_t st);
int gvd_step_targets(const float* ov, const unsigned char* mask_boxes, const unsigned char* frm_mask, const unsigned char* pnt_mask,
                     unsigned char* labels, unsigned char* fm, int B, int S, int R, int NB, int L1, cudaStream_t st);
int gvd_gather_class_rows(const float* vis_relu, const long long* input_cls, float* emb, int* cls_idx, int B, int S, int L1, int V, int D2, int NC,
                          cudaStream_t st);
int gvd_grounding_finish(float* G, const float* z, const float* cls_bias, const int* cls_idx, const unsigned char* mask, long long mask_stride_row,
                         int mask_per_step, int B, int S, int R, cudaStream_t st);
int gvd_lm_nll(const float* logits, long long ld, const long long* seq, int B, int S, int L1, int V, float* part_sum, int* part_cnt,
               cudaStream_t st);
int gvd_att_nll(const float* x, const unsigned char* labels, long long rows, int R, float* part_sum, int* part_cnt, cudaStream_t st);
int gvd_finish_mean(const float* part_sum, const int* part_cnt, int n, float sign, float* out, cudaStream_t st);
int gvd_grounding_eval_hits(const float* pred, const float* ref, const int* nref, float* max_iou, unsigned char* hit, int N, int F, int K,
                            float thresh, cudaStream_t st);
int gvd_grounding_gather(const float* ppls, const long long* idx, float* boxes, int B, int L, int NF, int P, int C, cudaStream_t st);
int gvd_frame_argmax(const float* x, long long* out, long long rows, int NF, int P, cudaStream_t st);

int gvd_gru_layer_f16(const float* gi, const float* Whh_img, const float* bhh, float* hstate, float* h_img, float* out, const long long* sample_idx, int B,
                      int T, int G, cudaStream_t st);

// power-of-two scales of the fp16x3 operands of the self-attention (queries, keys, probabilities, values)
#define GVD_ATT_SQ 4.f
#define GVD_ATT_SK 16.f
#define GVD_ATT_SP 1024.f
#define GVD_ATT_SV 16.f
// fp16x3 operand images for the self-attention: per-head key image (scale GVD_ATT_SK), transposed value image (GVD_ATT_SV)
int gvd_pack_heads_f16x3(const float* in, long long ld_in, long long rows, int nh, int hs_in, int hs, int KH, float scale, float* out, cudaStream_t st);
int gvd_transpose_pack_f16x3(const float* in, float* out, int B, int R, int C, int ld_in, int Rp, float scale, cudaStream_t st);

// fp16x3 precision scope (backend bit 4): inside a scope the wgmma GEMMs launched by this thread may use the fp16 hi/lo split
// (kind::f16, half the MMAs of 3xTF32).  Only forward inference stages with O(1) operands open a scope (prologue, decode step);
// gradient products stay on 3xTF32 (fp16's exponent range is too narrow for unscaled gradients).
bool gvd_gemm_f16();
void gvd_f16_scope(int delta);
#define GVD_F16_SA 4.f          // power-of-two operand scales of the fp16x3 variant: |activation| <= 16376, |weight| <= 255
#define GVD_F16_SW 256.f
// registry of pre-split constant weights (filled by gvd_model_finalize): fp32 weight pointer -> packed image (gvd_pack_f16x3)
int gvd_pack_f16x3(const float* W, long long ldw, int N, int K, float* out, long long Kp, cudaStream_t st, float scale = GVD_F16_SW);
// conversion-free GEMM on two operand images (gvd_wgmma.cu: ss_gemm_kernel)
// Q|K|V projection epilogue of the region encoder (ss_gemm_kernel): Q as fp32, K as the per-head fp16x3 image, V as the image of V^T per clip
struct GvdQkvImages { int HP, HS, KH, nh, R, Rp; float *k_img, *vt_img; float sk, sv; };
int gvd_gemm_f16ss(const float* Ap, long long lda, const float* Wp, long long ldw, const float* bias, const float* scale2, const float* shift2, int act,
                   float* C, long long ldc, int M, int N, int K, cudaStream_t st, float* img = nullptr, long long ld_img = 0,
                   const GvdQkvImages* qkv = nullptr);
bool gvd_packed_lookup(const float* W, long long ldw, int N, int K, const float** packed, long long* ld_packed);
struct GvdF16Scope { GvdF16Scope() { gvd_f16_scope(1); } ~GvdF16Scope() { gvd_f16_scope(-1); } };
