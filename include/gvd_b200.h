/* gvd-b200 C-ABI: H100-native caption-decode hot path of grounded-video-description.
 *
 * The reference has NO native interface: its boundary for this path is the Python nn.Module
 * surface misc/AttModel.py:167-171 (TopDownModel(opt)) / misc/model.py:227-234 (forward) /
 * the state_dict contract (main.py:638).  This header is the C ABI a binding for that surface
 * loads (ctypes stub in INTEGRATION.md; the in-repo binding is
 * grounded-video-description_b200/capi.py).  Plain pointers and sizes only; every entry point
 * returns 0 on success, non-zero on error with the message in gvd_last_error() (the Python shim
 * re-raises, mirroring the reference's assert / exception behaviour, SURVEY.md 8b "Errors").
 *
 * Device pointers are fp32 unless stated; masks are uint8; indices are int64 (the dtypes
 * main.py:564-573 allocates).  `stream` is a cudaStream_t passed as void*.  All calls are
 * re-entrant per (model, workspace) pair; no global mutable state except the error string
 * (thread-local).
 */
#ifndef GVD_B200_H
#define GVD_B200_H
#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define GVD_API __attribute__((visibility("default")))
#else
#define GVD_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* opt fields that size the model (misc/model.py:31-58, opts.py:38-52) */
typedef struct gvd_dims {
    int vocab_size;          /* V   opt.vocab_size                                   */
    int detect_size;         /* D   opt.detect_size (classes, background excluded)   */
    int input_encoding_size; /* E   opt.input_encoding_size                          */
    int rnn_size;            /* H   opt.rnn_size            (multiple of 4, <= 1024) */
    int att_hid_size;        /* A   opt.att_hid_size        (multiple of 4)          */
    int seq_length;          /* L   opt.seq_length                                   */
    int num_sampled_frm;     /* frames with proposals (10)                           */
    int num_prop_per_frm;    /* proposals per frame (100); R = frames * props        */
    int att_feat_size;       /* fc6 width, 2048                                      */
    int fc_feat_size;        /* frame feature width, 3072 = 2048 rgb + 1024 motion   */
    int obj_interact;        /* opt.obj_interact: 2-layer 6-head region self-attention */
    int unk_idx;             /* int(opt.wtoi['UNK'])  (misc/model.py:53)             */
} gvd_dims_t;

typedef struct gvd_model gvd_model_t;

GVD_API const char* gvd_last_error(void);
GVD_API const char* gvd_version(void);

/* ---- model / weights: replaces nn.Module construction + load_state_dict (main.py:616,638) */
GVD_API int gvd_model_create(const gvd_dims_t* dims, gvd_model_t** out);   /* att_input_mode 'both' */
/* opt.att_input_mode of the top-down captioner (opts.py:58-59, AttModel.py:140-156): what the language LSTM reads next to h_att.
 *   BOTH    (0) att + att2: temporal attention over the frame features plus region attention over the proposals;
 *   FEATMAP (1) att only: the region attention still yields its masked logits (the returned att2 weights, the grounding and the
 *               attention / grounding losses), but its weighted sum over the region features is never formed, so the decode step does
 *               not read them.  Same parameters (state_dict) as BOTH.
 *   DUAL_REGION (2) g att2 + (1 - g) att2_dual, g = sigmoid(dual_pointer(h_att)): two region attentions over the same features and
 *               masks, read in one pass; the returned logits are the first one's.  No temporal attention: the prologue skips the frame
 *               branch (att_embed, BatchNorm, bi-GRU, ctx2att).  The parameter list gains core.attention2_dual.{h2att,alpha_net}.* and
 *               core.dual_pointer.0.* (after core.attention2.*, before core.i2h_2.*).
 *   REGION  (3) only with enable_BUTD through gvd_model_create_opts: the transformer captioner's encoder reads the region features alone;
 *               the top-down captioner does not run 'region' (every top-down decode and teacher-forced entry point rejects such a model). */
#define GVD_ATT_INPUT_BOTH 0
#define GVD_ATT_INPUT_FEATMAP 1
#define GVD_ATT_INPUT_DUAL_REGION 2
#define GVD_ATT_INPUT_REGION 3
GVD_API int gvd_model_create_mode(const gvd_dims_t* dims, int att_input_mode, gvd_model_t** out);   /* region_attn_mode 'mix' */
/* opt.region_attn_mode (opts.py:63-64, AttModel.py:56-108): how the region attention Attention2 (and attention2_dual in DUAL_REGION)
 * scores proposal r against the query q = h2att(h_att).  The temporal attention is additive in every mode; the grounding is unchanged.
 *   MIX     (0) z_r = w . tanh(p_r + q) + b   (the default);
 *   MIX_MUL (1) z_r = w . tanh(p_r * q) + b   (element-wise product; same parameters as MIX);
 *   DP      (2) z_r = p_r . q                 (no tanh, weight or bias: the parameter list has no core.attention2.alpha_net.* nor, in
 *               DUAL_REGION, core.attention2_dual.alpha_net.*).
 * 'add' (a model-level alpha_net the grounding applies to 2048-wide vectors, model.py:55-56,256-261) and 'cat' (Attention2.forward reads an
 * undefined `xt`, AttModel.py:87) cannot run in the reference and are rejected. */
#define GVD_REGION_ATTN_MIX 0
#define GVD_REGION_ATTN_MIX_MUL 1
#define GVD_REGION_ATTN_DP 2
GVD_API int gvd_model_create_modes(const gvd_dims_t* dims, int att_input_mode, int region_attn_mode, gvd_model_t** out);
/* opt.transfer_mode (opts.py:62, model.py:84-85,180-215): how the class side of the region-class similarity comes from the detector.
 *   CLS  (0) vis_embed and the model-level vis_classifiers_bias [D+1] start from the detector's classifier (the default);
 *   NONE (1) the "no knowledge transfer" ablation: the module has no vis_classifiers_bias, so the similarity (model.py:326-336,524-533,
 *            652-661) and the teacher-forced grounding logits (model.py:472-476) carry no class bias, and the parameter list is one entry
 *            shorter (the first one).  Everything else is that of CLS.
 * 'glove' and 'both' cannot run in the reference and are rejected: 'glove' sizes the fc7 layer ctx2pool_grd [300, 2048] and fails copying
 * the detector's [2048, 2048] fc7 weights into it (model.py:88-89,158,177); 'both' makes fc7 2348 wide, so the region features reach
 * pool_embed 300 columns wider than it was built for: the reference fails reshaping them to pool_feat_size (model.py:86-87,70,370). */
#define GVD_TRANSFER_CLS 0
#define GVD_TRANSFER_NONE 1
/* butd = opt.enable_BUTD (opts.py:66, model.py:65-69,357-364,537-547): the bottom-up baseline.  The region features are the fc7 output
 * alone: no location embedding, no label features, no LayerNorms, so pool_embed.0.weight is [rnn_size, att_feat_size = 2048] (loc_fc.* stays
 * in the parameter list: the reference builds it, unused).  It needs att_input_mode GVD_ATT_INPUT_REGION (the reference asserts the pair,
 * model.py:66), and REGION needs butd = 1; any other pairing is rejected.  The prologue then skips the region-embedding row kernel, runs the
 * similarity stage only when sim_mat_out is given, and (with pack fusion) fc7 stores only the operand image its readers stream, so the
 * workspace's "g_pool" is not written.  Such a model serves the transformer captioner (gvd_prologue_fwd + pool_feats into gvd_tfm_*);
 * the top-down decode, beam, teacher-forced, single-step and host-buffer entry points reject it. */
GVD_API int gvd_model_create_opts(const gvd_dims_t* dims, int att_input_mode, int region_attn_mode, int transfer_mode, int butd,
                                  gvd_model_t** out);
GVD_API void gvd_model_destroy(gvd_model_t* m);
/* Copy one state_dict entry (by its reference key, e.g. "core.att_lstm.weight_ih") from a
 * DEVICE fp32 buffer of `numel` elements into the model's packed weight arena. */
GVD_API int gvd_model_set_param(gvd_model_t* m, const char* key, const float* dev_ptr, size_t numel, void* stream);
/* Number of keys / i-th key the model expects (the reference state_dict contract, SURVEY.md 8b). */
GVD_API int gvd_model_num_params(const gvd_model_t* m);
GVD_API const char* gvd_model_param_key(const gvd_model_t* m, int i, size_t* numel);
/* Derive packed / fused operands after all params are set (concats, ReLU(vis_embed), BN affine). */
GVD_API int gvd_model_finalize(gvd_model_t* m, void* stream);

/* ---- workspace (activations of one batch); caller-owned device memory */
GVD_API size_t gvd_workspace_bytes(const gvd_model_t* m, int B, int T);
GVD_API size_t gvd_workspace_bytes_beam(const gvd_model_t* m, int B, int T, int beam_size);   /* for gvd_beam_decode */
/* Address of a named activation inside a workspace laid out for (B,T): "fc_feats" [B,H],
 * "g_pool" [B,R,2048], "pool_embed"/"pool_feats" [B,R,H], "p_pool_feats" [B,R,A],
 * "conv_feats" [B,T,H], "p_conv_feats" [B,T,A] ([V,T,H] / [V,T,A], unmasked, after gvd_prologue_fwd_video).  NULL if unknown. */
GVD_API float* gvd_workspace_tensor(const gvd_model_t* m, void* workspace, int B, int T, const char* name);

/* ---- P1-P7: everything _sample computes before the loop (misc/model.py:504-568) */
GVD_API int gvd_prologue_fwd(gvd_model_t* m, int B, int T,
                     const float* segs_feat,        /* [B,T,fc_feat_size]          */
                     const float* ppls,             /* [B,R,7]                     */
                     const int64_t* num,            /* [B,7] int64 (main.py:572)   */
                     const float* ppls_feat,        /* [B,R,att_feat_size]         */
                     const int64_t* sample_idx,     /* [B,2]                       */
                     const uint8_t* pnt_mask,       /* [B,R+1], leading 0 column   */
                     void* workspace, size_t workspace_bytes,
                     float* sim_mat_out,            /* [B,D+1,R] or NULL           */
                     void* stream);

/* ---- video-indexed batch: B events (clips) of V videos, the frame features passed once per video.  The result equals gvd_prologue_fwd
 * on segs_feat[video_idx] (and every decode entry point after it equals the per-clip decode), with less traffic and work:
 *   - the frame mean and the frame branch (att_embed, BatchNorm, bi-GRU, ctx2att) run on the V videos, UNMASKED: the workspace holds
 *     conv_feats [V,T,H] / p_conv_feats [V,T,A] instead of B masked copies; clip b's clip vector reads video video_idx[b]'s mean;
 *   - the region stages are per clip as in gvd_prologue_fwd;
 *   - the decode attention of clip b reads only the rows of video video_idx[b] inside its window sample_idx[b] = [lo, hi) ∩ [0,T) and adds
 *     the closed form of the T - n_in rows outside it (in the per-clip path: zero features, p_conv = ctx2att.bias, one shared score).
 * Workspace: gvd_workspace_bytes_video(B, V, T, beam_size, nbox) (beam_size 1 / nbox 0 for the greedy and sampling loops).  The prologue
 * copies video_idx and sample_idx into it and records the workspace as video-indexed: gvd_decode_greedy / _sample / gvd_beam_decode /
 * gvd_teacher_fwd / gvd_decode_step_fwd / gvd_workspace_tensor with the same (B,T) then use that layout, until gvd_prologue_fwd runs on
 * the same workspace.  video_idx must lie in [0,V) (not checked on the device). */
GVD_API size_t gvd_workspace_bytes_video(const gvd_model_t* m, int B, int V, int T, int beam_size, int nbox);
GVD_API int gvd_prologue_fwd_video(gvd_model_t* m, int B, int V, int T,
                     const float* segs_feat,        /* [V,T,fc_feat_size]          */
                     const float* ppls,             /* [B,R,7]                     */
                     const int64_t* num,            /* [B,7]                       */
                     const float* ppls_feat,        /* [B,R,att_feat_size]         */
                     const int64_t* sample_idx,     /* [B,2] each clip's window    */
                     const int64_t* video_idx,      /* [B] in [0,V)                */
                     const uint8_t* pnt_mask,       /* [B,R+1]                     */
                     void* workspace, size_t workspace_bytes,
                     float* sim_mat_out,            /* [B,D+1,R] or NULL           */
                     void* stream);

/* ---- S1-S5: the 20-step greedy loop (misc/model.py:579-624); needs gvd_prologue_fwd's workspace */
GVD_API int gvd_decode_greedy(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes,
                      const uint8_t* pnt_mask,      /* [B,R+1]                     */
                      int64_t* seq_out,             /* [B,L]                       */
                      float* logprobs_out,          /* [B,L] or NULL               */
                      float* att2_logits_out,       /* [B,L,R] masked logits (Q8)  */
                      void* stream);

/* ---- the same loop with multinomial sampling (sample_max = 0, misc/model.py:595-603): same shapes and outputs as gvd_decode_greedy.
 * Word i of batch row b at step t (0 .. L-1) is drawn with the Gumbel-max trick: it = argmax_i (logit_i / temperature + g_i), ties to the
 * lower index, g_i = -log(-log(u_i)), u_i = ((w >> 9) + 0.5) * 2^-23 with w = word (i & 3) of Philox4x32-10(counter = (i >> 2, b, t, 0),
 * key = seed) — the token follows softmax(logit / temperature), the distribution torch.multinomial draws from.  logprobs_out holds the
 * UNTEMPERED log-softmax of the drawn word (model.py:602); there is no UNK rule.  The 23-bit uniforms bound g to [-2.82, 16.64]: a word
 * whose key is more than ~19.5 below the best is never drawn (probability < 1e-8).  b is the row's index in this call, so splitting a batch
 * changes the draws.  A row whose keys are all -inf or all NaN yields token 0.  temperature: finite and > 0.
 * The seed and temperature travel in a workspace-resident parameter block, so the captured loop is replayed, not re-captured, for new ones. */
GVD_API int gvd_decode_sample(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes,
                      const uint8_t* pnt_mask,      /* [B,R+1]                     */
                      uint64_t seed, float temperature,
                      int64_t* seq_out,             /* [B,L]                       */
                      float* logprobs_out,          /* [B,L] or NULL               */
                      float* att2_logits_out,       /* [B,L,R] masked logits (Q8)  */
                      void* stream);

/* ---- n sampled captions per clip from one prologue (sample_max = 0, several candidates per clip).
 * Rows: caption j of clip b is row b*n + j of seq_out / logprobs_out / att2_logits_out.  Equality: every output equals gvd_decode_sample on
 * the batch whose clips are repeated n times in place (torch.repeat_interleave(n, 0) of every prologue input) with the same seed and
 * temperature, bit for bit, given the same prologue outputs: the Philox counter takes the row index b*n + j, and the decode step runs the
 * same kernels at B*n rows.  The prologue runs once per clip; the n rows of a clip attend over its one copy of the features (feat_div = n,
 * as the beam rows do).  A prologue on the repeated batch runs its GEMMs with n times the rows, which can change their last bits.
 * Workspace: gvd_workspace_bytes_sample_n(B, V, T, n) bytes (V = 0 after gvd_prologue_fwd, V > 0 after gvd_prologue_fwd_video): the
 * prologue's outputs for B clips and decode state for B*n rows; gvd_prologue_fwd / _video must have filled it for the same (B, T).  The loop
 * is captured as its own graph per (B, T, n); seed and temperature travel in the parameter block as for gvd_decode_sample.  n = 1 is
 * gvd_decode_sample.  Vocabularies above 6144 words take the sliced tail as there.  Limits: n >= 1, B * n < 2^31. */
GVD_API size_t gvd_workspace_bytes_sample_n(const gvd_model_t* m, int B, int V, int T, int n);
GVD_API int gvd_decode_sample_n(gvd_model_t* m, int B, int T, int n, void* workspace, size_t workspace_bytes,
                      const uint8_t* pnt_mask,      /* [B,R+1] per clip            */
                      uint64_t seed, float temperature,
                      int64_t* seq_out,             /* [B*n,L]                     */
                      float* logprobs_out,          /* [B*n,L] or NULL             */
                      float* att2_logits_out,       /* [B*n,L,R] masked logits     */
                      void* stream);

/* ---- S2-S4 one teacher-forced / externally driven step (misc/AttModel.py:134-164).
 * state layout in the workspace; `step` selects the ping-pong parity and must count from 0. */
GVD_API int gvd_decode_step_fwd(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, int step,
                        const int64_t* tokens,      /* [B] input word ids          */
                        const uint8_t* att_mask,    /* [B,R+1] softmax mask        */
                        const uint8_t* out_mask,    /* [B,R+1] extra mask on the returned logits */
                        float* att2_logits_out, int64_t att2_stride_b, /* z[b*stride + r] */
                        float* h_lang_out,          /* [B,H] language-LSTM output or NULL */
                        void* stream);
GVD_API int gvd_decode_reset_state(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, void* stream);

/* ---- B1/B2: beam search of all clips at once, bookkeeping on the device (misc/model.py:627-742,
 * misc/CaptionModelBU.py:24-185 with the documented minimal repair; as-run aliasing reproduced).
 * Needs a workspace of gvd_workspace_bytes_beam() bytes that gvd_prologue_fwd filled for the same (B,T).
 * NaN rules of the bookkeeping: a row of logits that is all NaN ranks words 0 .. beam_size-1 (as a stable torch.sort(descending=True) does),
 * an all-NaN row of region scores gives region 0 (torch.argmax); see gvd_op_beam_topk / gvd_op_row_argmax. */
GVD_API int gvd_beam_decode(gvd_model_t* m, int B, int T, int beam_size, void* workspace, size_t workspace_bytes,
                    const uint8_t* pnt_mask,      /* [B,R+1]                              */
                    int64_t* seq_out,             /* [B,L]                                */
                    float* logprobs_out,          /* [B,L]                                */
                    int64_t* att2_idx_out,        /* [B,L] argmax region index per word   */
                    void* stream);

/* ---- the same beam search, grounded: additionally the region-attention logits of the returned caption (the second output of
 * forward(..., 'sample') with eval_opt['att2_weights']).  Row t of att2_logits_out is the masked logit row [R] (as gvd_decode_greedy
 * returns them) that the caption's own beam used to pick word t: row 0 is the <bos> step, row t that of the beam's ancestor at step t,
 * found by following the parent pointers back from the slot and step at which the caption finished.  Rows after the caption's last word
 * are 0.  seq_out / logprobs_out / att2_idx_out equal gvd_beam_decode's bit for bit.
 * Workspace: gvd_workspace_bytes_beam_att2(B, V, T, beam_size) (V = 0: the layout of gvd_prologue_fwd, V > 0: gvd_prologue_fwd_video's):
 * gvd_workspace_bytes_beam / _video plus a logit history [L][B*beam][R] fp32, the parents of every step and the finishing steps, laid out
 * after every other slot.  0 for beam_size < 2. */
GVD_API size_t gvd_workspace_bytes_beam_att2(const gvd_model_t* m, int B, int V, int T, int beam_size);
GVD_API int gvd_beam_decode_att2(gvd_model_t* m, int B, int T, int beam_size, void* workspace, size_t workspace_bytes,
                    const uint8_t* pnt_mask,      /* [B,R+1]                              */
                    int64_t* seq_out,             /* [B,L]                                */
                    float* logprobs_out,          /* [B,L]                                */
                    int64_t* att2_idx_out,        /* [B,L] as gvd_beam_decode             */
                    float* att2_logits_out,       /* [B,L,R] the caption's logit rows     */
                    void* stream);

/* ---- T1-T6 / G1: teacher-forced forward (misc/model.py:283-489) after gvd_prologue_fwd on the same batch,
 * eval-mode arithmetic (no dropout, BatchNorm running statistics).  Workspace: gvd_workspace_bytes_teacher().
 *   mode 0 'MLE': losses_out[4] = lm, att2, ground, cls (utils.py:122-152, model.py:345-350)
 *   mode 1 'GRD': att_idx_out / grd_idx_out [B,S,num_sampled_frm] = argmax over each frame's proposals
 *                 (model.py:486-489); sim_target_out [B,nbox,R] int32 and cls_pred_out [B,R] int32 give
 *                 the (target, predicted class) pairs of model.py:353-355 (compacted by the caller).
 * seq [B,L+1] = [0, gt_seq]; input_cls [B,L+1] = input_seq[:,0,:,0]; S = number of executed steps
 * (first i >= 1 with an all-zero token column, else L: model.py:425). */
GVD_API size_t gvd_workspace_bytes_teacher(const gvd_model_t* m, int B, int T, int nbox);
GVD_API int gvd_teacher_fwd(gvd_model_t* m, int B, int T, int nbox, int S, int mode, void* workspace, size_t workspace_bytes,
                    const int64_t* seq, const int64_t* input_cls, const float* ppls, const float* gt_boxes /* [B,nbox,6] */,
                    const uint8_t* mask_boxes /* [B,nbox,L+1] */, const uint8_t* frm_mask /* [B,R,nbox] */, const uint8_t* pnt_mask,
                    float* losses_out, int64_t* att_idx_out, int64_t* grd_idx_out, int32_t* sim_target_out, int32_t* cls_pred_out,
                    void* stream);

/* ---- end-to-end convenience with HOST buffers (pinned or pageable): H2D, prologue, loop, D2H.
 * This is what bench.py's `e2e` times. `workspace` is device memory. */
GVD_API int gvd_sample_greedy_host(gvd_model_t* m, int B, int T,
                           const float* h_segs_feat, const float* h_ppls, const int64_t* h_num,
                           const float* h_ppls_feat, const int64_t* h_sample_idx, const uint8_t* h_pnt_mask,
                           void* workspace, size_t workspace_bytes,
                           int64_t* h_seq_out, float* h_logprobs_out, float* h_att2_out, float* h_sim_mat_out,
                           void* stream);
/* the same for a video-indexed batch (see gvd_prologue_fwd_video): h_segs_feat [V,T,F], so V videos' frames cross PCIe instead of B
 * copies; h_video_idx [B] is checked on the host.  Workspace: gvd_workspace_bytes_video(B, V, T, 1, 0). */
GVD_API int gvd_sample_greedy_host_video(gvd_model_t* m, int B, int V, int T,
                           const float* h_segs_feat, const float* h_ppls, const int64_t* h_num,
                           const float* h_ppls_feat, const int64_t* h_sample_idx, const int64_t* h_video_idx, const uint8_t* h_pnt_mask,
                           void* workspace, size_t workspace_bytes,
                           int64_t* h_seq_out, float* h_logprobs_out, float* h_att2_out, float* h_sim_mat_out,
                           void* stream);

/* ---- single-op entry points (parity tests drive the kernels through the same ABI) */
GVD_API int gvd_op_linear(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc,
                  int M, int N, int K, int act, void* stream);
GVD_API int gvd_op_tanh(const float* x, float* y, int n, void* stream);
/* Post-decode grounding extraction (main.py:364-370; SURVEY 8(f) rank 2): att2 [B,L,F*P] region-attention logits of 'sample',
   ppls [B,F*P,7] -> idx_out [B,L,F] int64 = argmax over the P proposals of each frame (ties: lowest index),
   boxes_out [B,L,F,7] = the selected proposal rows (NULL to skip).  Replaces torch.max + permute + gather on the host side. */
GVD_API int gvd_grounding_extract(const float* att2, const float* ppls, int B, int L, int num_frames, int num_prop, int64_t* idx_out,
                  float* boxes_out, void* stream);
/* Grounding-evaluator hit test, batched over words (tools/anet_entities/scripts/eval_grd_anet_entities.py:95-102 with
   scripts/utils.py:75-128; SURVEY 8(f) rank 3): pred [N,F,5] = (x1,y1,x2,y2,frame) of the box chosen in every frame,
   ref [N,K,5] annotated boxes (first nref[n] rows valid) -> max_iou_out [N] (IoU with the +1 convention, 0 across frames,
   0 for zero-area annotations, -1 for zero-area predictions) and hit_out [N] = max > iou_thresh; bit-exact vs the fp32 CPU code. */
GVD_API int gvd_grounding_eval(const float* pred, const float* ref, const int* nref, int N, int F, int K, float iou_thresh,
                  float* max_iou_out, unsigned char* hit_out, void* stream);
/* host-side planning helper of the split-K decode products (backend bit 3): number of K splits used for a product
   with `weight_rows` x `k_total` weights and `batch_rows` activations rows, 0 if the shape falls back to the regular path */
GVD_API int gvd_plan_skinny_splits(int weight_rows, int k_total, int batch_rows);
/* host-side planning helper of gvd_sample_greedy_host: the clip chunks in which the fc6 region features cross PCIe (main.py:344-350 copies the
   whole batch in one piece).  `unit` = clips per self-attention sub-batch; writes at most `cap` chunk sizes to `chunks_out`, returns their number
   (the sizes sum to batch_clips), or -1 with gvd_last_error() set.  The entry point itself uses this schedule. */
GVD_API int gvd_plan_h2d_chunks(int batch_clips, int unit, int* chunks_out, int cap);
/* the same contraction on the wgmma tensor cores (3xTF32, fp32-faithful) */
GVD_API int gvd_op_linear_tc(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc,
                  int M, int N, int K, int act, void* stream);
/* batched short-K (hs <= 192) product C[b,h] = A[b][:, h*hs:(h+1)*hs] . W[b][:, h*hs:(h+1)*hs]^T — the self-attention
   score shape of transformer.py:111 — through the tensor-core score product; A [nb,M,ld], W [nb,N,ld], C [nb,nh,M,N] */
GVD_API int gvd_op_scores_tc(const float* A, const float* W, float* C, int nb, int nh, int M, int N, int hs, int64_t ld, void* stream);
/* self-attention core of one region-encoder layer (transformer.py:84-118) on a packed projection buffer qkv [nb, R, 3*HP]
   (Q | K | V; head h = columns [h*hs, (h+1)*hs)): out[nb, R, HP] = concat_h softmax(Q_h K_h^T * scale) V_h through the fused
   wgmma pair.  stages bit 0: A-stationary scores with the softmax-numerator epilogue -> numer [nb,nh,R,R] and per-(row,
   32-key group) factors factor [nb,nh,ceil(R/32),R] (softmax = numer * factor); bit 1: the row-scaled P.V -> out */
GVD_API int gvd_op_self_attention_tc(const float* qkv, float* out, int nb, int nh, int R, int hs, int HP, float scale,
                  float* numer, float* factor, int stages, void* stream);
/* the same self-attention core through the fused kernel (scores, softmax and P.V in one launch, the scores never leave the SM): the key
   and V^T operand images are built inside the call.  img == NULL: out[nb, R, HP] fp32 (columns [h*hs, (h+1)*hs) of every head);
   else the fp16x3 operand image of the output, [nb*R, img_ld] 32-bit words (scale 4, columns [nh*hs, img_ld) zeros), and out is unused */
GVD_API int gvd_op_self_attention_fused(const float* qkv, float* out, int nb, int nh, int R, int hs, int HP, float scale, float* img,
                  int64_t img_ld, void* stream);
/* the conversion-free prologue GEMM on its own (operands packed into fp16x3 images inside the call); img_out: optional fp16x3 image of
   the output, [M, rup32(N)] 32-bit words (what the next GEMM would stream), C may then be NULL.  nh > 0: the region encoder's Q|K|V
   projection (N = 3 * nh * hs, M a multiple of R, no bias / activation, img_out NULL): Q to C columns [0, nh * hs), K to the per-head
   image k_img [M, nh, rup32(hs)] words, V to the V^T image vt_img [M / R, nh * hs, rup32(R)] words; qkv_ref != 0 builds the same images
   from the fp32 product (all N columns of C) with the separate pack passes.  nh == 0: k_img, vt_img and qkv_ref are ignored */
GVD_API int gvd_op_linear_f16ss(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc,
                  float* img_out, int M, int N, int K, int act, int nh, int hs, int R, float* k_img, float* vt_img, int qkv_ref,
                  void* stream);
/* one LSTMCell step (AttModel.py:139,160) from up to two dense input segments; backend 0 = CUDA cores, 1 = wgmma */
GVD_API int gvd_op_lstm_step(int B, int H, const float* x0, int K0, const float* w0, int64_t ldw0, const float* x1, int K1,
                  const float* w1, int64_t ldw1, const float* bias1, const float* bias2, const float* c_prev,
                  float* h_out, float* c_out, int backend, void* stream);
/* ---- the decode step's default path op by op (tests/test_gpu_decode_ops.py): operand-swapped split-K product, its three reductions,
 * the three greedy samplers and one bidirectional GRU layer.
 * Partial planes: part[s][b][n], row pitch ldp >= Nw (ldp % 4 == 0), plane stride B * ldp; columns [Nw, ldp) are never written.
 * f16_images 0: operands split in the kernel (3xTF32, or fp16x3 with backend bit 4); 1: both operands packed into fp16x3 images first
 * (the conversion-free product of the default backend).  S = 0: the plan of gvd_plan_skinny_splits.  fp16x3 holds |x| <= 16376 and
 * |w| <= 255; larger values overflow to inf. */
GVD_API int gvd_op_skinny_partials(const float* W, int Nw, int K, const float* X, int64_t ldx, int B, int S, int f16_images, float* part,
                  int ldp, void* stream);
/* sum of the S planes (ascending s) + pre + biases -> LSTMCell; h to up to three fp32 destinations and two fp16x3 images (H % 32 == 0) */
GVD_API int gvd_op_reduce_lstm(const float* part, int S, int ldp, const float* pre, int pre_div, const float* bias1, const float* bias2,
                  const float* c_prev, float* c_out, float* h0, int64_t ldh0, float* h1, int64_t ldh1, float* h2, int64_t ldh2, int B, int H,
                  float* pk1, int64_t ldpk1, float* pk2, int64_t ldpk2, void* stream);
GVD_API int gvd_op_reduce_bias(const float* part, int S, int Nw, int ldp, const float* bias, float* out, int64_t ld_out, int B, void* stream);
/* Samplers (model.py:590-615): top-2 with ties to the lower index, the runner-up if the winner is unk_idx, log-prob of the token taken;
 * it_out [B]; seq_out / logp_out element b at [b * out_stride] (NULL to skip); xt [B, ld_xt] = ReLU(embed[token]) (NULL to skip), xt_pk
 * its fp16x3 image.  A row without any finite comparison (all NaN) yields token 0.  reduce_pick: 2 <= V <= 6144. */
GVD_API int gvd_op_reduce_pick(const float* part, int S, int ldp, const float* bias, int B, int V, int unk_idx, int64_t* it_out,
                  int64_t* seq_out, float* logp_out, int64_t out_stride, const float* embed, float* xt, int64_t ld_xt, int E,
                  float* logits_out, int64_t ld_logits, float* xt_pk, int64_t ld_xt_pk, void* stream);
GVD_API int gvd_op_greedy_pick(const float* logits, int64_t ld, int B, int V, int unk_idx, int64_t* it_out, int64_t* seq_out, float* logp_out,
                  int64_t out_stride, const float* embed, float* xt, int64_t ld_xt, int E, void* stream);
/* the multinomial sampler of gvd_decode_sample on S partial planes (+ bias or NULL) at decode step `step`, same destinations as reduce_pick */
GVD_API int gvd_op_reduce_sample(const float* part, int S, int ldp, const float* bias, int B, int V, float temperature, uint64_t seed, int step,
                  int64_t* it_out, int64_t* seq_out, float* logp_out, int64_t out_stride, const float* embed, float* xt, int64_t ld_xt, int E,
                  float* xt_pk, int64_t ld_xt_pk, void* stream);
/* the vocabulary tail for any V (2 <= V <= 65535 * 1024), the one the decode loops run above 6144 words: one CTA per (row, 1024 words) writes
 * a record of its slice, the last CTA of the row merges the records in a fixed order.  mode GVD_VOCAB_GREEDY: top-2 + UNK rule as
 * reduce_pick; GVD_VOCAB_SAMPLE: the draw of reduce_sample at (temperature, seed, step); GVD_VOCAB_ARGMAX: the first maximum (transformer
 * head).  ldp % 4 == 0, part 16-byte aligned; logits_out (or NULL) receives the summed logits at pitch ld_logits. */
#define GVD_VOCAB_GREEDY 0
#define GVD_VOCAB_SAMPLE 1
#define GVD_VOCAB_ARGMAX 2
GVD_API int gvd_op_reduce_pick_split(const float* part, int S, int ldp, const float* bias, int B, int V, int mode, int unk_idx, float temperature,
                  uint64_t seed, int step, int64_t* it_out, int64_t* seq_out, float* logp_out, int64_t out_stride, const float* embed, float* xt,
                  int64_t ld_xt, int E, float* logits_out, int64_t ld_logits, float* xt_pk, int64_t ld_xt_pk, void* stream);
/* vocabulary head h [B,K] . W [V,K]^T + bias with the sampler in the GEMM epilogue; B <= 128, E % 4 == 0, xt [B,E] */
GVD_API int gvd_op_logit_pick_tc(const float* h, int64_t ldh, const float* W, int64_t ldw, const float* bias, int B, int V, int K, int unk_idx,
                  const float* embed, int E, int64_t* it_out, int64_t* seq_out, float* logp_out, int64_t out_stride, float* xt, void* stream);
/* one bidirectional GRU layer (model.py:150-154) from its input projections gi [B,T,6G] (b_ih included): Whh [2,3G,G], bhh [2,3G],
 * sample_idx [B,2] or NULL (output rows t outside [lo, hi) are 0), out [B,T,2G].  path 0: GEMM + pointwise kernel per step (the GEMM
 * follows the backend switch); path 1: tensor-core layer kernel (B <= 128, G % 32 == 0). */
GVD_API int gvd_op_gru_layer(int path, const float* gi, const float* Whh, const float* bhh, const int64_t* sample_idx, int B, int T, int G,
                  float* out, void* stream);
/* ---- the decode attention and the beam-search bookkeeping op by op (tests/test_gpu_attn_beam_ops.py).
 * gvd_op_attention: Attention + Attention2 (AttModel.py:33-53, :71-108) of B query rows; row b attends over clip b / feat_div.
 *   p_pool [B/feat_div,R,A], pool [.,R,H], p_conv [.,T,A], conv [.,T,H]; the query [B,2A] (temporal | region) is either q or the sum
 *   q_bias + q_part[0..q_S) over split-K planes [q_S][B][2A] (then q == NULL).  w1,b1 / w2,b2: the two alpha_net layers ([A], [1]).
 *   Masks [B/feat_div, R+1] uint8 with the legacy leading column (ignored); out_mask rows at pitch out_mask_stride (0 = R+1).
 *   z_out[b * z_stride_b + r] = region logit, MIN_VALUE where att_mask or out_mask is set.  x_out[b * x_ld + h] (x_ld 0 = H) = att + att2;
 *   x_pk: optional fp16x3 image of it (scale 4, pitch x_pk_ld words).  RC / TC rows per region / temporal chunk (1 .. 128); partial
 *   [B, ceil(R/RC) + ceil(T/TC), H+4] chunk records (max, sum of exp, 2 unused words, unnormalised weighted sum), region chunks first.
 *   ticket [B] zeroed ints: the last chunk CTA of a row merges (and resets its ticket to 0); NULL: a separate combine kernel merges
 *   (x_ld must then be 0 or H, no x_pk).  A, H multiples of 4, A and H <= 1024. */
GVD_API int gvd_op_attention(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q, const float* q_part,
                  int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2, const float* b2, const uint8_t* att_mask,
                  const uint8_t* out_mask, int64_t out_mask_stride, float* z_out, int64_t z_stride_b, float* partial, int* ticket, float* x_out,
                  int64_t x_ld, float* x_pk, int64_t x_pk_ld, int B, int R, int T, int A, int H, int RC, int TC, int feat_div, void* stream);
/* gvd_op_attention_mode: the same with att_input_mode GVD_ATT_INPUT_* (gvd_op_attention = BOTH).  FEATMAP: x_out = att; the region
 *   chunks write z_out and their (max, sum) words only (their weighted-sum words are not written), and `pool` may be NULL.
 *   DUAL_REGION: q = [attention2_dual query | attention2 query], w1 / b1 = attention2_dual.alpha_net, w2 / b2 = attention2.alpha_net;
 *   p_conv / conv unused (may be NULL); partial [B, 2 ceil(R/RC), H+4] (attention2 chunks, then attention2_dual chunks); ticket required;
 *   x_out = g att2 + (1 - g) att2_dual with g = sigmoid(gate_w . gate_h[b * gate_ld ..] + gate_b[0]) (dual_pointer, [H] and [1]). */
GVD_API int gvd_op_attention_mode(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                  const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2, const float* b2,
                  const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out, int64_t z_stride_b, float* partial,
                  int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld, int B, int R, int T, int A, int H, int RC, int TC,
                  int feat_div, int att_input_mode, const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld,
                  void* stream);
/* gvd_op_attention_form: gvd_op_attention_mode with the region score form GVD_REGION_ATTN_* (gvd_op_attention_mode = MIX).  In DP the region
 *   alpha_net pointers (w2 / b2, and w1 / b1 in DUAL_REGION) are not read and may be NULL. */
GVD_API int gvd_op_attention_form(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                  const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2, const float* b2,
                  const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out, int64_t z_stride_b, float* partial,
                  int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld, int B, int R, int T, int A, int H, int RC, int TC,
                  int feat_div, int att_input_mode, const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld,
                  int region_attn_mode, void* stream);
/* gvd_op_attention_video: gvd_op_attention_form over video-level frame features: p_conv / conv [V,T,A|H] unmasked, video_idx [B / feat_div]
 *   int64 in [0,V), sample_idx [B / feat_div, 2] the windows, ctx_bias [A] (ctx2att.bias, 16-byte aligned): the temporal attention of row b
 *   equals gvd_op_attention_form on conv[video] with the rows outside the window zeroed and p_conv there = ctx_bias. */
GVD_API int gvd_op_attention_video(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                  const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2, const float* b2,
                  const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out, int64_t z_stride_b, float* partial,
                  int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld, int B, int R, int T, int A, int H, int RC, int TC,
                  int feat_div, int att_input_mode, const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld,
                  int region_attn_mode, const int64_t* video_idx, const int64_t* sample_idx, const float* ctx_bias, void* stream);
/* gvd_op_attention_path: gvd_op_attention_video's arguments (video_idx / sample_idx / ctx_bias NULL: per-clip frame features) and the
 *   kernel: path 0 = one CTA per (row, chunk), what every decode entry point runs; path 1 = one CTA per (clip, group of up to 8 of its
 *   feat_div rows, chunk), which streams the chunk's features once for the group.  Both give the same bits per row. */
GVD_API int gvd_op_attention_path(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                  const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2, const float* b2,
                  const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out, int64_t z_stride_b, float* partial,
                  int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld, int B, int R, int T, int A, int H, int RC, int TC,
                  int feat_div, int att_input_mode, const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld,
                  int region_attn_mode, const int64_t* video_idx, const int64_t* sample_idx, const float* ctx_bias, int path, void* stream);
/* beam_topk: per row of logits [rows, V] (pitch ld) the K <= 8 (K <= V) best words, value descending, ties to the lower index:
 *   topv [rows, K] = their log_softmax, topi [rows, K].  NaN words are skipped; a pick that finds only NaN left takes the lowest untaken
 *   index, so an all-NaN row gives 0 .. K-1 (as a stable torch.sort(descending=True) does).  Rows only partly NaN differ from torch,
 *   which ranks NaN first.
 * row_argmax: idx [rows] int32 = first index of the row maximum of z [rows, R] (pitch ld); an all -inf or all-NaN row gives 0 like
 *   torch.argmax (NaN entries are skipped: a row only partly NaN differs, torch returns its first NaN). */
GVD_API int gvd_op_beam_topk(const float* logits, int64_t ld, int rows, int V, int K, float* topv, int* topi, void* stream);
GVD_API int gvd_op_row_argmax(const float* z, int64_t ld, int rows, int R, int* idx, void* stream);
/* gvd_beam_decode's bookkeeping with the model replaced by a script (K <= 8, L <= 64): logits [L][B*K][V] (step t's vocabulary logits),
 * z [L+1][B*K][R] (region scores of core step t; t = 0 is the <bos> step), probe [B*K][H] (H % 4 == 0): a stand-in for the recurrent
 * state, reordered to the surviving beams after every step but the last, in place.  seq_out / logp_out / att2_idx_out [B, L] as
 * gvd_beam_decode returns them; parents_out [L][B*K] int32: every step's parent beam of each new beam (index within the clip). */
GVD_API int gvd_op_beam_search_scripted(const float* logits, const float* z, float* probe, int B, int K, int L, int V, int R, int H,
                  int64_t* seq_out, float* logp_out, int64_t* att2_idx_out, int* parents_out, void* stream);
/* ... the same, plus att2_out [B, L, R]: the rows of z the returned caption used, gathered as gvd_beam_decode_att2 gathers them. */
GVD_API int gvd_op_beam_att2_scripted(const float* logits, const float* z, float* probe, int B, int K, int L, int V, int R, int H,
                  int64_t* seq_out, float* logp_out, int64_t* att2_idx_out, int* parents_out, float* att2_out, void* stream);
/* arithmetic backend switches: bit 0 wgmma tensor cores for every GEMM-shaped stage (0 = fp32 CUDA cores); bit 1 fused self-attention pair;
   bit 2 (4) inert; bit 3 (8) operand-swapped split-K decode products with fused
   reduce + sampler; bit 4 (16) fp16x3 instead of 3xTF32 in the forward GEMMs, pre-split weights, conversion-free decode step, tensor-core GRU;
   bit 5 (32) inert; bit 6 (64) programmatic dependent launch in the decode loop (off); bit 7 (128)
   conversion-free prologue GEMMs; bit 8 (256) fp16x3 key / value images in the self-attention pair; bit 9 (512) pack fusion
   (producers store the operand image of the next GEMM); bit 10 (1024) inert.  The inert bits 2, 5 and 10 are accepted so that stored flag
   values keep working; nothing reads them.  Default 923 = 1 + 2 + 8 + 16 + 128 + 256 + 512.  Every combination in
   tests/test_gpu_tcgen05.py meets the same parity bar. */
GVD_API int gvd_set_backend(int flags);
GVD_API int gvd_get_backend(void);
GVD_API int gvd_op_kernel_launches(void);   /* kernels launched by this process through the library so far */

/* ---- optional per-stage CUDA-event timing on the launching stream (bench.py's per-kernel roofline).
 * Enable, run, synchronise the stream, then read (name, total ms, launches) entries. */
GVD_API int gvd_profile_enable(int on);
GVD_API int gvd_profile_reset(void);
GVD_API int gvd_profile_count(void);
GVD_API const char* gvd_profile_entry(int i, double* total_ms, long long* count);


/* ---------------------------------------------------------------------------------------------------------------------------
 * Training-step primitives (main.py:235-266: teacher-forced forward in train mode, explicit backward, clip, Adam) — the
 * element-wise / row-wise / reduction kernels the host orchestration in gvd_b200/train.py is written over; dense products go
 * through gvd_op_linear and gvd_tr_gemm_nt_batched.  Definitions of
 * every primitive: tests/ops_ref.py.  All tensors fp32 and contiguous unless noted; masks uint8; indices int64.
 * ------------------------------------------------------------------------------------------------------------------------- */
/* op: 0 a+b, 1 a*b, 2 a*s, 3 relu(a), 4 relu backward (a = dy, b = y), 5 mask ? s : a */
GVD_API int gvd_tr_ew(int op, const float* a, const float* b, const unsigned char* mask, float s, float* out, long long n, void* stream);
GVD_API int gvd_tr_outer_rows(const float* a, const float* v, float* out, int B, int N, int H, void* stream);          /* out[b,n,h] = a[b,n] v[b,h] */
GVD_API int gvd_tr_colsum(const float* x, float* out, int batch, long long M, int N, void* stream);                   /* out[z,n] = sum_m x[z,m,n] */
GVD_API int gvd_tr_rowsum(const float* x, float* out, long long M, int N, void* stream);
GVD_API int gvd_tr_sum_all(const float* x, float* out, long long n, void* stream);
GVD_API int gvd_tr_mean_dim1(const float* x, float* out, int B, int T, int F, void* stream);
GVD_API int gvd_tr_ln_fwd(const float* x, float* y, long long rows, int n, void* stream);                              /* F.layer_norm, no affine */
GVD_API int gvd_tr_ln_bwd(const float* dy, const float* y, const float* x, float* dx, long long rows, int n, void* stream);
GVD_API int gvd_tr_ln_star_fwd(const float* x, const float* gamma, const float* beta, float* y, long long rows, int n, void* stream);   /* transformer.py:74-77 */
GVD_API int gvd_tr_ln_star_bwd(const float* dy, const float* x, const float* gamma, float* dx, float* dy_xhat, long long rows, int n, void* stream);
GVD_API int gvd_tr_softmax_fwd(const float* x, float scale, float* p, long long rows, int n, void* stream);
GVD_API int gvd_tr_softmax_bwd(const float* dp, const float* p, float scale, float* dx, long long rows, int n, void* stream);
GVD_API int gvd_tr_lm_nll(const float* logits, const int64_t* target, const unsigned char* mask, const float* inv_n /* device scalar: gvd_tr_count_inv */, float* rowloss, float* dlogits,
                  long long rows, int n, void* stream);                                                                /* utils.py:126-136 */
GVD_API int gvd_tr_pos_nll(const float* x, const unsigned char* pos, const float* inv_n /* device scalar: gvd_tr_count_inv */, float* rowloss, float* dx, long long rows, int n, void* stream);   /* utils.py:139,142 */
GVD_API int gvd_tr_cls_nll(const float* simT, const int* target, const float* inv_n /* device scalar: gvd_tr_count_inv */, float* part, float* dsimT, int B, int R, int NB, int C, void* stream);  /* model.py:345-350 */
GVD_API int gvd_tr_targets(const float* ppls, const float* gt_boxes, const unsigned char* frm_mask, const unsigned char* pnt_mask,
                  const unsigned char* mask_boxes, int B, int R, int NB, int S, int L1, float* overlaps, int* cls_target,
                  unsigned char* labels, unsigned char* frame_masks, void* stream);                                    /* utils.py:293-328, model.py:436-440 */
GVD_API int gvd_tr_lstm_cell_fwd(const float* gates, const float* c, float* h2, float* c2, float* act, int B, int H, void* stream);
GVD_API int gvd_tr_lstm_cell_bwd(const float* dh2, const float* dc2, const float* act, const float* c, const float* c2, float* dgates, float* dc,
                  int B, int H, void* stream);
GVD_API int gvd_tr_gru_cell_fwd(const float* gi, const float* gh, const float* h, float* h2, float* r, float* z, float* n, int B, int G, void* stream);
GVD_API int gvd_tr_gru_cell_bwd(const float* dh, const float* r, const float* z, const float* n, const float* h, const float* ghn, float* dgi,
                  float* dgh, float* dh_keep, int B, int G, void* stream);
GVD_API int gvd_tr_att_scores_fwd(const float* p, const float* q, const float* w, const float* bias, float* s, int B, int N, int A, void* stream);
GVD_API int gvd_tr_att_scores_bwd(const float* ds, const float* p, const float* q, const float* w, float* dpre, float* ds_t, int B, int N, int A, void* stream);
/* multiplicative scores (region_attn_mode 'mix_mul'): s[b,n] = w . tanh(p[b,n,:] * q[b,:]) + bias; the backward writes, per [b,n,a] with
 * t = tanh(p q) and dpre = ds[b,n] w[a] (1 - t^2):  dp = dpre q[b,a],  dq_t = dpre p[b,n,a] (dq = its sum over n),  ds_t = ds[b,n] t (dw = its
 * sum over b, n) */
GVD_API int gvd_tr_att_scores_mul_fwd(const float* p, const float* q, const float* w, const float* bias, float* s, int B, int N, int A, void* stream);
GVD_API int gvd_tr_att_scores_mul_bwd(const float* ds, const float* p, const float* q, const float* w, float* dp, float* dq_t, float* ds_t, int B,
                  int N, int A, void* stream);
GVD_API int gvd_tr_gather_rows(const float* table, const int64_t* idx, float* out, long long M, int D, void* stream);
GVD_API int gvd_tr_index_add_rows(const int64_t* idx, const float* rows, float* out, int n_rows, int M, int D, void* stream);
GVD_API int gvd_tr_bn_normalize(const float* e, const float* mu, const float* var, float* out, long long M, int N, void* stream);
GVD_API int gvd_tr_bn_bwd(const float* dxh, const float* e_hat, const float* var, const float* s1, const float* s2, float* de, long long M, int N, void* stream);
GVD_API int gvd_tr_adam_first_step(const float* w, const float* g, float coef, float lr, float b1, float b2, float eps, float* out, long long n, void* stream);
GVD_API int gvd_tr_gemm_nt_batched(const float* A, long long lda, long long sA, const float* W, long long ldw, long long sW, float* C, long long ldc,
                  long long sC, int M, int N, int K, int batch, void* stream);                                         /* C[z] = A[z] W[z]^T */
/* flat-buffer optimiser: global gradient norm + clip coefficient on the device (clip_grad_norm_, main.py:265) and one torch.optim.Adam step
   with a per-tensor learning-rate table (one param group per tensor, main.py:660-677); the single NCCL all-reduce of D1 runs on the same flat
   gradient buffer between the backward and these two calls. */
/* train-mode dropout (nn.Dropout sites of misc/model.py:75-119,153, AttModel.py:161, transformer.py:84-88,100): counter-based Philox4x32-10
   mask keyed by (seed, site, step) — the same call on the upstream gradient is the backward; nothing is stored. */
GVD_API int gvd_tr_dropout(const float* x, float* y, long long n, float p, long long seed, int site, long long step, void* stream);
GVD_API size_t gvd_tr_sumsq_scratch_bytes(void);
GVD_API int gvd_tr_grad_norm(const float* g, long long n, float max_norm, void* scratch, float* norm_out /* [2]: norm, clip coef */, void* stream);
GVD_API int gvd_tr_adam_flat(float* w, float* g, float* m, float* v, long long n, const int64_t* seg_end, const float* seg_lr, int nseg,
                             const float* norm, float b1, float b2, float eps, float weight_decay, int t, void* stream);
/* The other two optimisers main.py:671-677 builds (--optim sgd | adamax), on the same flat layout as gvd_tr_adam_flat: segment s covers
   [seg_end[s-1], seg_end[s]) with learning rate seg_lr[s] (lr <= 0: the tensor got no gradient and is left bit-identical, state included), g
   is scaled in place by the clip coefficient norm[1] (null: 1).  torch keeps optimiser state per parameter, so seg_step[s] (int32, device) is
   the number of steps segment s has taken; each call advances it for the segments with lr > 0, after the update.
   gvd_tr_sgd_flat:    torch.optim.SGD(momentum, dampening=0, nesterov=False, weight_decay):  d = g coef + wd w;  buf = d on the segment's
                       first step, else buf = momentum buf + d;  w -= lr buf.  (main.py:673 builds it with momentum = 0.9.)
   gvd_tr_adamax_flat: torch.optim.Adamax(betas=(b1, b2), eps, weight_decay):  d = g coef + wd w;  m = b1 m + (1 - b1) d;
                       u = max(b2 u, |d| + eps);  w -= lr / (1 - b1^t) m / u,  t = seg_step[s] + 1.  (main.py:677, betas = optim_alpha /
                       optim_beta of main.py:666-669.) */
GVD_API int gvd_tr_sgd_flat(float* w, float* g, float* buf, long long n, const int64_t* seg_end, const float* seg_lr, int* seg_step, int nseg,
                            const float* norm, float momentum, float weight_decay, void* stream);
GVD_API int gvd_tr_adamax_flat(float* w, float* g, float* m, float* u, long long n, const int64_t* seg_end, const float* seg_lr, int* seg_step,
                               int nseg, const float* norm, float b1, float b2, float eps, float weight_decay, void* stream);
GVD_API int gvd_tr_count_inv(const void* data, long long n, int elem_bytes /* 1: bytes != 0, 4: int32 > 0 */, float* inv_out, void* stream);   /* 1 / count on the device */
GVD_API int gvd_tr_scalar_mul(const float* a, const float* b, float* out, void* stream);
GVD_API int gvd_tr_outer_rows_acc(const float* a, const float* v, float* acc, int B, int N, int H, void* stream);   /* acc[b,n,:] += a[b,n] v[b,:] */
GVD_API int gvd_tr_transpose(const float* in, float* out, int batch, int R, int C, void* stream);                      /* out[z,c,r] = in[z,r,c] */
/* multi-head attention of the transformer captioner's decoder in train mode (misc/transformer.py:92-123; csrc/gvd_tfm_train.cu): q [B, Lq, H],
   k / v [B, N, H] already projected, heads = the torch.chunk(6, -1) column ranges read in place, scores q.k * scale, causal: row t sees keys
   r <= t.  o [B, Lq, H] (heads concatenated), lse [B, n_heads, Lq] = the softmax's log-sum-exp for the backward.  p > 0: each head's
   probabilities are dropped with the mask gvd_tr_dropout draws on that head's contiguous [B, Lq, N] tensor at site site_base + head.
   Lq <= 64, N <= 1000, head width <= 192; anything else is refused with status 1. */
GVD_API int gvd_tr_mha_fwd(const float* q, const float* k, const float* v, float* o, float* lse, int B, int Lq, int N, int H, int causal, float scale,
                           float p, long long seed, int site_base, long long step, void* stream);
GVD_API int gvd_tr_mha_bwd(const float* q, const float* k, const float* v, const float* o, const float* d_o, const float* lse, float* dq, float* dk,
                           float* dv, int B, int Lq, int N, int H, int causal, float scale, float p, long long seed, int site_base, long long step,
                           void* stream);

/* ---- transformer captioner (att_model = 'transformer'): Decoder.greedy of misc/transformer.py:214-241 behind
 * TransformerDecoder.forward(infer=True) (:271-274), called by misc/model.py:570-578 after the prologue.  The weights are the
 * cap_model.decoder.* entries of the state_dict (device fp32, nn.Linear layout [out, in]); the binding owns them (they are not part of
 * gvd_model_t: the prologue P1-P7 is shared with the top-down captioner, the decoder is not). */
typedef struct {
    const float *self_wq, *self_wk, *self_wv, *self_wo, *self_gamma, *self_beta;    /* layers.l.selfattn.{layer.w*.weight, layernorm.*}   */
    const float *att_wq, *att_wk, *att_wv, *att_wo, *att_gamma, *att_beta;          /* layers.l.attention.{...}                           */
    const float *ff_w1, *ff_b1, *ff_w2, *ff_b2, *ff_gamma, *ff_beta;                /* layers.l.feedforward.{layer.linear{1,2}.*, layernorm.*} */
} gvd_tfm_layer_t;
typedef struct {
    int d_model;             /* rnn_size (model.py:142)                                  */
    int d_hidden;            /* rnn_size / 2                                             */
    int vocab_size;          /* rows of decoder.out                                      */
    int n_heads;             /* 6 (model.py:139): torch.chunk head split of d_model      */
    gvd_tfm_layer_t layer[2];
    const float *out_w, *out_b;   /* decoder.out: vocabulary head AND (times sqrt(d_model)) the token embedding (transformer.py:207,222) */
} gvd_tfm_weights_t;
GVD_API size_t gvd_tfm_workspace_bytes(const gvd_tfm_weights_t* w, int B, int L, int n0, int n1);
/* enc0 [B,n0,d_model] / enc1 [B,n1,d_model]: the encoder outputs of decoder layers 0 / 1 (att_input_mode 'both': conv_feats, pool_feats of
 * the prologue workspace; 'featmap': conv_feats twice; 'region': pool_feats twice).  pe [L,d_model]: positional_encodings_like
 * (transformer.py:30-49), computed by the binding.  seq_out [B,L] int64: the prediction; logits_out [B,L,vocab] or NULL: the vocabulary-head
 * output of every step (tests).  L <= 64, d_model <= 1024. */
GVD_API int gvd_tfm_decode_greedy(const gvd_tfm_weights_t* w, int B, int L, const float* enc0, int n0, const float* enc1, int n1,
                     const float* pe, void* workspace, size_t workspace_bytes, int64_t* seq_out, float* logits_out, void* stream);
/* Teacher-forced pass + loss of the captioner (Decoder.forward, mask(), F.cross_entropy: transformer.py:207-212,51-54,276-280; model.py:411-419),
 * eval mode.  seq [B,S+1] int64 = [0, gt_seq]: position t is fed seq[:,t] and scored against seq[:,t+1] where that is != 0; loss_out [1]. */
GVD_API int gvd_tfm_teacher_fwd(const gvd_tfm_weights_t* w, int B, int S, const float* enc0, int n0, const float* enc1, int n1,
                     const float* pe, void* workspace, size_t workspace_bytes, const int64_t* seq, float* loss_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GVD_B200_H */
