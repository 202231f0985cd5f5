// gvd-b200: C-ABI (include/gvd_b200.h) — model/weight arena, workspace layout, prologue and
// decode orchestration.  Host code only launches kernels; there is no CPU compute path.
#include <atomic>
#include <mutex>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/gvd_b200.h"
#include "gvd_kernels.cuh"

// ------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};
void gvd_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void gvd_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long gvd_launch_count() { return g_launches.load(); }
void gvd_launch_count_add(long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" GVD_API const char* gvd_last_error(void) { return g_err; }
extern "C" GVD_API const char* gvd_version(void) { return "gvd-b200 0.1.0 (sm_90a)"; }
extern "C" GVD_API int gvd_op_kernel_launches(void) { return (int)g_launches.load(); }
// backend switches (gvd_set_backend): bit 0 wgmma tensor cores for every GEMM-shaped stage (0 = fp32 CUDA cores); bit 1 fused self-attention
// pair; bit 2 (4) inert (it selected 256-column tiles of a kernel that needed tensor memory); bit 3 (8) operand-swapped split-K decode products
// with fused reduce + sampler; bit 4 (16) fp16x3 instead of 3xTF32 in the forward GEMMs (pre-split constant weights); bit 5 (32) inert (it
// selected a cooperative GRU layer kernel); bit 6 (64) programmatic dependent launch in the decode loop (off); bit 7 (128) conversion-free
// GEMMs for the prologue (activations packed into the fp16x3 image, both operands straight from TMA); bit 8 (256)
// fp16x3 images instead of tf32 planes in the fused self-attention pair; bit 9 (512) pack fusion: the producer of a prologue activation (GEMM
// epilogue / row kernel) stores the fp16x3 operand image the next GEMM streams, instead of a separate pack pass; bit 10 (1024) inert (it
// selected CTA pairs).  Bits 2, 5 and 10 are accepted so that stored flag values keep working; nothing reads them.  Names: GvdBackendBit
// (gvd_common.cuh).  Default 923 = 1 + 2 + 8 + 16 + 128 + 256 + 512.
static std::atomic<int> g_backend{923};
int gvd_backend() { return g_backend.load(std::memory_order_relaxed); }
// registry of pre-split constant weights (fp16x3 variant): fp32 weight pointer -> packed image
namespace {
struct PackedW { const float* packed; long long ld; int N, K; long long ldw; };
std::mutex g_pw_mu;
std::unordered_map<const float*, PackedW> g_pw;
}  // namespace
bool gvd_packed_lookup(const float* W, long long ldw, int N, int K, const float** packed, long long* ld_packed) {
    std::lock_guard<std::mutex> lk(g_pw_mu);
    auto it = g_pw.find(W);
    if (it == g_pw.end() || it->second.ldw != ldw || it->second.N != N || it->second.K != K) return false;
    *packed = it->second.packed;
    *ld_packed = it->second.ld;
    return true;
}
bool gvd_pdl() { return gvd_backend_on(BK_PDL); }
static thread_local int g_f16_depth = 0;
void gvd_f16_scope(int delta) { g_f16_depth += delta; }
bool gvd_gemm_f16() { return g_f16_depth > 0 && gvd_backend_on(BK_F16X3); }
extern "C" GVD_API int gvd_set_backend(int flags) { g_backend.store(flags); return 0; }
extern "C" GVD_API int gvd_get_backend(void) { return g_backend.load(); }

// ------------------------------------------------------------------------------------ stage profiler
// Optional CUDA-event timing of each stage / kernel family ON THE LAUNCHING STREAM (bench.py uses it
// for the per-kernel roofline; off by default: zero events recorded).
#include <mutex>
namespace {
struct ProfRec { const char* name; cudaEvent_t a, b; };
std::atomic<int> g_prof_on{0};
std::mutex g_prof_mu;
std::vector<ProfRec> g_prof_recs;
std::vector<cudaEvent_t> g_prof_pool;
struct ProfAgg { double ms; long long n; };
std::unordered_map<std::string, ProfAgg> g_prof_agg;
cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
struct ProfScope {
    const char* name; cudaStream_t st; cudaEvent_t a{}, b{}; bool on;
    ProfScope(const char* n, cudaStream_t s) : name(n), st(s), on(g_prof_on.load(std::memory_order_relaxed) != 0) {
        if (!on) return;
        std::lock_guard<std::mutex> lk(g_prof_mu);
        a = prof_event(); b = prof_event();
        cudaEventRecord(a, st);
    }
    ~ProfScope() {
        if (!on) return;
        cudaEventRecord(b, st);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof_recs.push_back({name, a, b});
    }
};
void prof_collect() {      // caller has synchronised the stream(s)
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto& r : g_prof_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { auto& g = g_prof_agg[r.name]; g.ms += ms; g.n += 1; }
        g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
    }
    g_prof_recs.clear();
}
}  // namespace
extern "C" GVD_API int gvd_profile_enable(int on) {
    g_prof_on.store(on ? 1 : 0);
    return 0;
}
extern "C" GVD_API int gvd_profile_reset(void) {
    prof_collect();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_agg.clear();
    return 0;
}
extern "C" GVD_API int gvd_profile_count(void) {
    prof_collect();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    return (int)g_prof_agg.size();
}
extern "C" GVD_API const char* gvd_profile_entry(int i, double* total_ms, long long* count) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    int k = 0;
    for (auto& kv : g_prof_agg) {
        if (k++ == i) { if (total_ms) *total_ms = kv.second.ms; if (count) *count = kv.second.n; return kv.first.c_str(); }
    }
    return nullptr;
}
#define GVD_STAGE(name, expr) do { ProfScope _ps(name, st); GVD_TRY(expr); } while (0)

static inline size_t rup(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int rup4(int x) { return (x + 3) / 4 * 4; }

// ------------------------------------------------------------------------------------ small pack kernels
namespace {
__global__ void relu_copy_kernel(const float* x, float* y, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = fmaxf(x[i], 0.f);
}
__global__ void add2_kernel(const float* a, const float* b, float* y, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = a[i] + b[i];
}
// dst[r, c] = (rmap[r] >= 0 && cmap[c] >= 0) ? src[rmap[r], cmap[c]] : 0 ; identity map when nullptr
__global__ void pack_kernel(float* dst, long long ld_dst, const float* src, long long ld_src, const int* rmap, const int* cmap,
                            int nrows, int ncols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= ncols || r >= nrows) return;
    const int sr = rmap ? rmap[r] : r, sc = cmap ? cmap[c] : c;
    dst[(long long)r * ld_dst + c] = (sr >= 0 && sc >= 0) ? src[(long long)sr * ld_src + sc] : 0.f;
}
// xt = ReLU(embed[token]) (model.py:79-82,605): materialised once per step for the tensor-core LSTM path
__global__ void embed_relu_kernel(const float* table, const long long* tokens, float* out, long long ld_out, int B, int E, int V, float* pk,
                                  long long ld_pk) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * E) return;                       // B * E is a multiple of 32 whenever pk is given (E % 32 == 0)
    const int b = i / E, e = i % E;
    const long long tok = tokens[b];
    // ids outside the table read as NaN instead of out of bounds (nn.Embedding raises; the Python shim validates host-visible ids)
    const float v = (tok >= 0 && tok < V) ? fmaxf(table[tok * E + e], 0.f) : __int_as_float(0x7fc00000);
    out[(long long)b * ld_out + e] = v;
    if (pk) {                                     // fp16x3 operand image (E even: lanes e, e + 1 sit in one warp)
        const float vn = __shfl_down_sync(0xffffffffu, v, 1);
        if (!(e & 1)) {
            uint32_t hi, lo;
            f16x3_split_pair(v, vn, GVD_F16_SA, hi, lo);
            uint32_t* dst = reinterpret_cast<uint32_t*>(pk) + (long long)b * ld_pk + f16x3_word(e);
            dst[0] = hi; dst[16] = lo;
        }
    }
}
__global__ void bn_affine_kernel(const float* w, const float* b, const float* mean, const float* var, float* scale, float* shift,
                                 int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float s = w[i] / sqrtf(var[i] + 1e-5f);      // BatchNorm1d eval, eps 1e-5 (model.py:114)
    scale[i] = s;
    shift[i] = b[i] - mean[i] * s;
}
}  // namespace

// ------------------------------------------------------------------------------------ model
struct Param { std::string key; size_t numel; size_t off; bool set; };
struct LoopKey { int B, T, backend; void* ws; size_t ws_bytes; int V, div; };   // what a captured decode loop depends on
// a workspace whose prologue ran on a video-indexed batch (gvd_prologue_fwd_video): the decode entries lay it out for V videos
struct VideoWs { void* ws; int B, T, V; };

struct gvd_model {
    gvd_dims_t d;
    int att_mode = GVD_ATT_INPUT_BOTH;   // opt.att_input_mode (GVD_ATT_INPUT_*): what the language LSTM reads, AttModel.py:144-156
    int region_form = GVD_REGION_ATTN_MIX;   // opt.region_attn_mode (GVD_REGION_ATTN_*): the region attentions' score, AttModel.py:79-96
    bool butd = false;                       // opt.enable_BUTD: the region features are fc7 alone (model.py:65-69,357-364)
    int R, G, NC, FCX, FCXp, PIN, PINp, NCp, Vp, HS, HP, nheads, rgb, motion;
    std::vector<int> head_off, head_size;
    std::vector<Param> params;
    std::unordered_map<std::string, int> index;
    float* arena = nullptr;      // raw state_dict entries
    float* packed = nullptr;     // derived operands
    size_t arena_floats = 0, packed_floats = 0;
    bool finalized = false;
    // packed operands
    float *fc_embed_w, *pool_embed_w, *vis_relu, *h2att_w, *h2att_b, *att_bias_sum, *bn_scale, *bn_shift;
    float *w_att_cat, *w_lang_cat;      // [4H, E+H] = [W_ih[:, H:] | W_hh] and [4H, 3H] = [W_ih | W_hh]: one K axis per LSTM (split-K path)
    float *wqk[2], *wv[2], *wo[2];
    float *gru_wih[2], *gru_bih[2], *gru_whh[2], *gru_bhh[2];
    int* maps = nullptr;
    float* packed16 = nullptr;   // fp16x3 images of the constant GEMM weights (gvd_pack_f16x3), registered in g_pw
    std::vector<const float*> pw_keys;
    // host-buffer entry point: second stream + events for the chunked H2D / compute pipeline
    cudaStream_t copy_stream = nullptr;
    std::vector<cudaEvent_t> events;
    // frame branch (P1 + P7) on its own stream, concurrent with the region stages (P2-P6): the bi-GRU is a chain of short
    // launches on 32 SMs that the big GEMMs would otherwise wait behind
    cudaStream_t frame_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // greedy loop captured once per (batch, frames, workspace, backend) as a CUDA graph: 20 steps x 6 launches replayed with one
    // cudaGraphLaunch (no per-launch host cost, back-to-back scheduling on the device)
    cudaStream_t capture_stream = nullptr;
    cudaGraphExec_t greedy_exec = nullptr;
    LoopKey greedy_key{0, 0, 0, nullptr, 0, 0, 0};
    long long greedy_nodes = 0;      // kernel launches inside one replay (counted while capturing)
    // the multinomial-sampling loop has a graph of its own (alternating greedy and sampling calls re-capture neither); its seed and
    // temperature are read from the workspace, so a new draw replays the same graph
    cudaGraphExec_t sample_exec = nullptr;
    LoopKey sample_key{0, 0, 0, nullptr, 0, 0, 0};
    long long sample_nodes = 0;
    // ... and the loop over n sampled rows per clip (gvd_decode_sample_n), one more graph keyed by (B, T, n)
    cudaGraphExec_t sample_n_exec = nullptr;
    LoopKey sample_n_key{0, 0, 0, nullptr, 0, 0, 0};
    long long sample_n_nodes = 0;
    std::vector<VideoWs> video_ws;   // set by the video prologues, cleared by a per-clip prologue on the same workspace

    float* P(const std::string& k) const {
        auto it = index.find(k);
        return it == index.end() ? nullptr : arena + params[it->second].off;
    }
};

static void add_param(gvd_model* m, const std::string& key, size_t numel) {
    Param p{key, numel, m->arena_floats, false};
    m->arena_floats += rup(numel, 64);
    m->index[key] = (int)m->params.size();
    m->params.push_back(p);
}

extern "C" GVD_API int gvd_model_create(const gvd_dims_t* dims, gvd_model_t** out) {
    return gvd_model_create_mode(dims, GVD_ATT_INPUT_BOTH, out);
}

extern "C" GVD_API int gvd_model_create_mode(const gvd_dims_t* dims, int att_input_mode, gvd_model_t** out) {
    return gvd_model_create_modes(dims, att_input_mode, GVD_REGION_ATTN_MIX, out);
}

extern "C" GVD_API int gvd_model_create_modes(const gvd_dims_t* dims, int att_input_mode, int region_attn_mode, gvd_model_t** out) {
    return gvd_model_create_opts(dims, att_input_mode, region_attn_mode, GVD_TRANSFER_CLS, 0, out);
}

extern "C" GVD_API int gvd_model_create_opts(const gvd_dims_t* dims, int att_input_mode, int region_attn_mode, int transfer_mode, int butd,
                                             gvd_model_t** out) {
    GVD_REQUIRE(dims && out, "model_create: null argument");
    GVD_REQUIRE(transfer_mode == GVD_TRANSFER_CLS || transfer_mode == GVD_TRANSFER_NONE,
                "model_create: transfer_mode %d is not implemented (0 = 'cls', 1 = 'none'; 'glove' and 'both' fail in the reference)", transfer_mode);
    GVD_REQUIRE(butd == 0 || butd == 1, "model_create: butd must be 0 or 1 (got %d)", butd);
    // BUTD and 'region' come together: the reference asserts the pair (model.py:66), and 'region' is only the transformer captioner's encoder
    GVD_REQUIRE((att_input_mode == GVD_ATT_INPUT_REGION) == (butd == 1),
                "model_create: enable_BUTD needs att_input_mode 'region' (model.py:66), and 'region' is only built with enable_BUTD (att_input_mode %d, "
                "butd %d)", att_input_mode, butd);
    if (butd) att_input_mode = GVD_ATT_INPUT_BOTH;   // checked above; the modes below are the top-down decode's

    GVD_REQUIRE(region_attn_mode == GVD_REGION_ATTN_MIX || region_attn_mode == GVD_REGION_ATTN_MIX_MUL || region_attn_mode == GVD_REGION_ATTN_DP,
                "model_create: region_attn_mode %d is not implemented (0 = 'mix', 1 = 'mix_mul', 2 = 'dp')", region_attn_mode);
    GVD_REQUIRE(att_input_mode == GVD_ATT_INPUT_BOTH || att_input_mode == GVD_ATT_INPUT_FEATMAP || att_input_mode == GVD_ATT_INPUT_DUAL_REGION,
                "model_create: att_input_mode %d is not implemented (0 = 'both', 1 = 'featmap', 2 = 'dual_region')", att_input_mode);
    const gvd_dims_t& d = *dims;
    GVD_REQUIRE(d.rnn_size % 4 == 0 && d.rnn_size >= 8 && d.rnn_size <= 1024, "rnn_size must be a multiple of 4 in [8,1024] (got %d)",
                d.rnn_size);
    GVD_REQUIRE(d.rnn_size % 2 == 0 && (d.rnn_size / 2) % 4 == 0, "rnn_size/2 must be a multiple of 4");
    GVD_REQUIRE(d.att_hid_size % 4 == 0 && d.att_hid_size > 0, "att_hid_size must be a multiple of 4");
    GVD_REQUIRE(d.input_encoding_size % 4 == 0 && d.input_encoding_size > 0, "input_encoding_size must be a multiple of 4");
    GVD_REQUIRE(d.att_feat_size == 2048, "att_feat_size must be 2048 (fc7 transfer, misc/model.py:158-178)");
    GVD_REQUIRE(d.fc_feat_size > 2048 && (d.fc_feat_size - 2048) % 4 == 0, "fc_feat_size must be 2048 + motion width");
    GVD_REQUIRE(d.vocab_size >= 2 && d.detect_size >= 1 && d.seq_length >= 1, "bad vocab/detect/seq sizes");
    GVD_REQUIRE(d.num_sampled_frm >= 1 && d.num_prop_per_frm >= 1, "bad proposal grid");
    GVD_REQUIRE(d.unk_idx >= 0 && d.unk_idx < d.vocab_size, "unk_idx out of range");
    gvd_model* m = new gvd_model();
    m->d = d;
    m->att_mode = att_input_mode;
    m->region_form = region_attn_mode;
    m->butd = butd == 1;
    const int H = d.rnn_size, A = d.att_hid_size, E = d.input_encoding_size, V = d.vocab_size, D = d.detect_size;
    m->R = d.num_sampled_frm * d.num_prop_per_frm;
    GVD_REQUIRE(!d.obj_interact || m->R % 4 == 0, "obj_interact needs R %% 4 == 0 (R=%d)", m->R);
    m->G = H / 2;
    m->NC = D + 1;
    m->NCp = rup4(m->NC);
    m->FCX = d.fc_feat_size + 50;
    m->FCXp = rup4(m->FCX);
    m->PIN = butd ? d.att_feat_size : d.att_feat_size + 300 + D + 1;      // BUTD: pool_embed reads fc7 alone (model.py:65-69)
    m->PINp = rup4(m->PIN);
    m->Vp = rup4(V);
    m->rgb = 2048;
    m->motion = d.fc_feat_size - 2048;
    // torch.chunk(6, -1) head split (transformer.py:121): ceil(H/6) each, remainder last
    const int c = (H + 5) / 6;
    for (int o = 0; o < H; o += c) { m->head_off.push_back(o); m->head_size.push_back(std::min(c, H - o)); }
    m->nheads = (int)m->head_off.size();
    m->HS = rup4(c);
    m->HP = m->HS * m->nheads;
    const int G = m->G;
    // the reference state_dict (SURVEY.md 8b), float entries only
    if (transfer_mode == GVD_TRANSFER_CLS) add_param(m, "vis_classifiers_bias", D + 1);   // 'none' has no class bias (model.py:196-203)
    add_param(m, "loc_fc.0.weight", 300 * 5); add_param(m, "loc_fc.0.bias", 300);
    add_param(m, "embed.0.weight", (size_t)V * E);
    add_param(m, "vis_embed.0.weight", (size_t)(D + 1) * 2048);
    add_param(m, "fc_embed.0.weight", (size_t)H * m->FCX); add_param(m, "fc_embed.0.bias", H);
    add_param(m, "seg_info_embed.0.weight", 50 * 4); add_param(m, "seg_info_embed.0.bias", 50);
    add_param(m, "att_embed.0.0.weight", (size_t)(H / 2) * 2048); add_param(m, "att_embed.0.0.bias", H / 2);
    add_param(m, "att_embed.1.0.weight", (size_t)(H / 2) * m->motion); add_param(m, "att_embed.1.0.bias", H / 2);
    add_param(m, "att_embed_aux.0.weight", H); add_param(m, "att_embed_aux.0.bias", H);
    add_param(m, "att_embed_aux.0.running_mean", H); add_param(m, "att_embed_aux.0.running_var", H);
    add_param(m, "pool_embed.0.weight", (size_t)H * m->PIN); add_param(m, "pool_embed.0.bias", H);
    add_param(m, "ctx2att.weight", (size_t)A * H); add_param(m, "ctx2att.bias", A);
    add_param(m, "ctx2pool.weight", (size_t)A * H); add_param(m, "ctx2pool.bias", A);
    add_param(m, "logit.weight", (size_t)V * H); add_param(m, "logit.bias", V);
    if (d.obj_interact) {
        for (int l = 0; l < 2; ++l) {
            const std::string p = "obj_interact.encoder.layers." + std::to_string(l) + ".";
            for (const char* w : {"wq", "wk", "wv", "wo"}) add_param(m, p + "selfattn.layer." + w + ".weight", (size_t)H * H);
            add_param(m, p + "selfattn.layernorm.gamma", H); add_param(m, p + "selfattn.layernorm.beta", H);
            add_param(m, p + "feedforward.layer.linear1.weight", (size_t)(H / 2) * H); add_param(m, p + "feedforward.layer.linear1.bias", H / 2);
            add_param(m, p + "feedforward.layer.linear2.weight", (size_t)H * (H / 2)); add_param(m, p + "feedforward.layer.linear2.bias", H);
            add_param(m, p + "feedforward.layernorm.gamma", H); add_param(m, p + "feedforward.layernorm.beta", H);
        }
    }
    for (int l = 0; l < 2; ++l)
        for (const char* sfx : {"", "_reverse"}) {
            const std::string s = "_l" + std::to_string(l) + sfx;
            add_param(m, "context_enc.weight_ih" + s, (size_t)3 * G * (l == 0 ? H : 2 * G));
            add_param(m, "context_enc.weight_hh" + s, (size_t)3 * G * G);
            add_param(m, "context_enc.bias_ih" + s, 3 * G);
            add_param(m, "context_enc.bias_hh" + s, 3 * G);
        }
    add_param(m, "ctx2pool_grd.0.weight", (size_t)2048 * d.att_feat_size); add_param(m, "ctx2pool_grd.0.bias", 2048);
    add_param(m, "core.att_lstm.weight_ih", (size_t)4 * H * (E + H)); add_param(m, "core.att_lstm.weight_hh", (size_t)4 * H * H);
    add_param(m, "core.att_lstm.bias_ih", 4 * H); add_param(m, "core.att_lstm.bias_hh", 4 * H);
    add_param(m, "core.lang_lstm.weight_ih", (size_t)4 * H * 2 * H); add_param(m, "core.lang_lstm.weight_hh", (size_t)4 * H * H);
    add_param(m, "core.lang_lstm.bias_ih", 4 * H); add_param(m, "core.lang_lstm.bias_hh", 4 * H);
    const bool region_alpha = region_attn_mode != GVD_REGION_ATTN_DP;   // 'dp' builds Attention2 without alpha_net (AttModel.py:62-65)
    for (const char* a : {"attention", "attention2"}) {
        add_param(m, std::string("core.") + a + ".h2att.weight", (size_t)A * H); add_param(m, std::string("core.") + a + ".h2att.bias", A);
        if (std::string(a) == "attention" || region_alpha) {
            add_param(m, std::string("core.") + a + ".alpha_net.weight", A); add_param(m, std::string("core.") + a + ".alpha_net.bias", 1);
        }
    }
    if (att_input_mode == GVD_ATT_INPUT_DUAL_REGION) {   // AttModel.py:126-128
        add_param(m, "core.attention2_dual.h2att.weight", (size_t)A * H); add_param(m, "core.attention2_dual.h2att.bias", A);
        if (region_alpha) { add_param(m, "core.attention2_dual.alpha_net.weight", A); add_param(m, "core.attention2_dual.alpha_net.bias", 1); }
        add_param(m, "core.dual_pointer.0.weight", H); add_param(m, "core.dual_pointer.0.bias", 1);
    }
    // present in the checkpoint but never used by the forward pass (AttModel.py:130-131, quirk Q10)
    add_param(m, "core.i2h_2.weight", (size_t)H * 2 * H); add_param(m, "core.i2h_2.bias", H);
    add_param(m, "core.h2h_2.weight", (size_t)H * H); add_param(m, "core.h2h_2.bias", H);

    // packed operand arena
    size_t pf = 0;
    auto take = [&](size_t n) { size_t o = pf; pf += rup(n, 64); return o; };
    std::vector<std::pair<float**, size_t>> slots;
    auto slot = [&](float** p, size_t n) { slots.push_back({p, take(n)}); };
    slot(&m->fc_embed_w, (size_t)H * m->FCXp);
    slot(&m->pool_embed_w, (size_t)H * m->PINp);
    slot(&m->vis_relu, (size_t)m->NC * 2048);
    slot(&m->h2att_w, (size_t)2 * A * H);
    slot(&m->h2att_b, 2 * A);
    slot(&m->att_bias_sum, 4 * H);
    slot(&m->w_att_cat, (size_t)4 * H * (d.input_encoding_size + H));
    slot(&m->w_lang_cat, (size_t)4 * H * 3 * H);
    slot(&m->bn_scale, H);
    slot(&m->bn_shift, H);
    for (int l = 0; l < 2; ++l) {
        if (d.obj_interact) {
            slot(&m->wqk[l], (size_t)3 * m->HP * H);       // [Wq; Wk; Wv] head-padded, one projection GEMM
            slot(&m->wo[l], (size_t)H * m->HP);
        }
        slot(&m->gru_wih[l], (size_t)6 * G * (l == 0 ? H : 2 * G));
        slot(&m->gru_bih[l], 6 * G);
        slot(&m->gru_whh[l], (size_t)6 * G * G);
        slot(&m->gru_bhh[l], 6 * G);
    }
    m->packed_floats = pf;
    if (cudaMalloc(&m->arena, m->arena_floats * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&m->packed, m->packed_floats * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&m->maps, (size_t)(m->HP + 16) * sizeof(int)) != cudaSuccess) {
        gvd_set_error("model_create: cudaMalloc failed (%s)", cudaGetErrorString(cudaGetLastError()));
        gvd_model_destroy(m);
        return 2;
    }
    for (auto& s : slots) *s.first = m->packed + s.second;
    if (d.obj_interact)
        for (int l = 0; l < 2; ++l) m->wv[l] = m->wqk[l] + (size_t)2 * m->HP * H;
    *out = m;
    return 0;
}

extern "C" GVD_API void gvd_model_destroy(gvd_model_t* m) {
    if (!m) return;
    if (m->arena) cudaFree(m->arena);
    if (m->packed) cudaFree(m->packed);
    if (m->maps) cudaFree(m->maps);
    {
        std::lock_guard<std::mutex> lk(g_pw_mu);
        for (const float* k : m->pw_keys) g_pw.erase(k);
    }
    if (m->packed16) cudaFree(m->packed16);
    for (cudaEvent_t e : m->events) cudaEventDestroy(e);
    if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
    if (m->frame_stream) cudaStreamDestroy(m->frame_stream);
    if (m->ev_fork) cudaEventDestroy(m->ev_fork);
    if (m->ev_join) cudaEventDestroy(m->ev_join);
    if (m->greedy_exec) cudaGraphExecDestroy(m->greedy_exec);
    if (m->sample_exec) cudaGraphExecDestroy(m->sample_exec);
    if (m->sample_n_exec) cudaGraphExecDestroy(m->sample_n_exec);
    if (m->capture_stream) cudaStreamDestroy(m->capture_stream);
    delete m;
}

extern "C" GVD_API int gvd_model_num_params(const gvd_model_t* m) { return m ? (int)m->params.size() : 0; }
extern "C" GVD_API const char* gvd_model_param_key(const gvd_model_t* m, int i, size_t* numel) {
    if (!m || i < 0 || i >= (int)m->params.size()) return nullptr;
    if (numel) *numel = m->params[i].numel;
    return m->params[i].key.c_str();
}

extern "C" GVD_API int gvd_model_set_param(gvd_model_t* m, const char* key, const float* dev_ptr, size_t numel, void* stream) {
    GVD_REQUIRE(m && key && dev_ptr, "set_param: null argument");
    auto it = m->index.find(key);
    GVD_REQUIRE(it != m->index.end(), "set_param: unexpected key '%s' (not in the reference state_dict for these dims)", key);
    Param& p = m->params[it->second];
    GVD_REQUIRE(p.numel == numel, "set_param: size mismatch for '%s': expected %zu elements, got %zu", key, p.numel, numel);
    GVD_CHECK_CUDA(cudaMemcpyAsync(m->arena + p.off, dev_ptr, numel * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    p.set = true;
    m->finalized = false;
    return 0;
}

static int pack2d(float* dst, long long ld_dst, const float* src, long long ld_src, const int* rmap, const int* cmap, int nrows,
                  int ncols, cudaStream_t st) {
    dim3 grid(gvd_cdiv(ncols, 256), nrows);
    pack_kernel<<<grid, 256, 0, st>>>(dst, ld_dst, src, ld_src, rmap, cmap, nrows, ncols);
    GVD_CHECK_LAUNCH();
    return 0;
}

extern "C" GVD_API int gvd_model_finalize(gvd_model_t* m, void* stream) {
    GVD_REQUIRE(m, "finalize: null model");
    cudaStream_t st = (cudaStream_t)stream;
    for (auto& p : m->params)
        GVD_REQUIRE(p.set || p.key.rfind("core.i2h_2", 0) == 0 || p.key.rfind("core.h2h_2", 0) == 0,
                    "finalize: parameter '%s' was never set (strict load, main.py:638)", p.key.c_str());
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, G = m->G;
    // padded-K copies (16-byte row alignment for the 128-bit operand loads)
    GVD_CHECK_CUDA(cudaMemsetAsync(m->fc_embed_w, 0, (size_t)H * m->FCXp * sizeof(float), st));
    GVD_TRY(pack2d(m->fc_embed_w, m->FCXp, m->P("fc_embed.0.weight"), m->FCX, nullptr, nullptr, H, m->FCX, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(m->pool_embed_w, 0, (size_t)H * m->PINp * sizeof(float), st));
    GVD_TRY(pack2d(m->pool_embed_w, m->PINp, m->P("pool_embed.0.weight"), m->PIN, nullptr, nullptr, H, m->PIN, st));
    {   // vis_embed = Embedding + ReLU (model.py:93-97): the class "classifiers" are ReLU(weight)
        const size_t n = (size_t)m->NC * 2048;
        relu_copy_kernel<<<gvd_cdiv(n, 256), 256, 0, st>>>(m->P("vis_embed.0.weight"), m->vis_relu, n);
        GVD_CHECK_LAUNCH();
    }
    // the query GEMM's first slot: the temporal query, or in dual_region (no temporal attention) attention2_dual's
    const std::string q0 = m->att_mode == GVD_ATT_INPUT_DUAL_REGION ? "core.attention2_dual" : "core.attention";
    GVD_CHECK_CUDA(cudaMemcpyAsync(m->h2att_w, m->P(q0 + ".h2att.weight"), (size_t)A * H * 4, cudaMemcpyDeviceToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(m->h2att_w + (size_t)A * H, m->P("core.attention2.h2att.weight"), (size_t)A * H * 4, cudaMemcpyDeviceToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(m->h2att_b, m->P(q0 + ".h2att.bias"), A * 4, cudaMemcpyDeviceToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(m->h2att_b + A, m->P("core.attention2.h2att.bias"), A * 4, cudaMemcpyDeviceToDevice, st));
    add2_kernel<<<gvd_cdiv(4 * H, 256), 256, 0, st>>>(m->P("core.att_lstm.bias_ih"), m->P("core.att_lstm.bias_hh"), m->att_bias_sum, 4 * H);
    GVD_CHECK_LAUNCH();
    {   // one K axis per LSTM for the split-K path: [W_ih (token part) | W_hh] and [W_ih | W_hh]
        const int E = d.input_encoding_size;
        GVD_TRY(pack2d(m->w_att_cat, E + H, m->P("core.att_lstm.weight_ih") + H, H + E, nullptr, nullptr, 4 * H, E, st));
        GVD_TRY(pack2d(m->w_att_cat + E, E + H, m->P("core.att_lstm.weight_hh"), H, nullptr, nullptr, 4 * H, H, st));
        GVD_TRY(pack2d(m->w_lang_cat, 3 * H, m->P("core.lang_lstm.weight_ih"), 2 * H, nullptr, nullptr, 4 * H, 2 * H, st));
        GVD_TRY(pack2d(m->w_lang_cat + 2 * H, 3 * H, m->P("core.lang_lstm.weight_hh"), H, nullptr, nullptr, 4 * H, H, st));
    }
    bn_affine_kernel<<<gvd_cdiv(H, 256), 256, 0, st>>>(m->P("att_embed_aux.0.weight"), m->P("att_embed_aux.0.bias"),
                                                        m->P("att_embed_aux.0.running_mean"), m->P("att_embed_aux.0.running_var"),
                                                        m->bn_scale, m->bn_shift, H);
    GVD_CHECK_LAUNCH();
    if (d.obj_interact) {
        // head-padded projections: head h occupies columns [h*HS, h*HS+size_h) (zeros beyond), so every
        // per-head operand starts 16-byte aligned although torch.chunk gives 171/169-wide heads
        std::vector<int> map(m->HP, -1);
        for (int h = 0; h < m->nheads; ++h)
            for (int i = 0; i < m->head_size[h]; ++i) map[h * m->HS + i] = m->head_off[h] + i;
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->maps, map.data(), m->HP * sizeof(int), cudaMemcpyHostToDevice, st));
        GVD_CHECK_CUDA(cudaStreamSynchronize(st));   // `map` is a stack-lifetime host buffer
        for (int l = 0; l < 2; ++l) {
            const std::string p = "obj_interact.encoder.layers." + std::to_string(l) + ".selfattn.layer.";
            GVD_TRY(pack2d(m->wqk[l], H, m->P(p + "wq.weight"), H, m->maps, nullptr, m->HP, H, st));
            GVD_TRY(pack2d(m->wqk[l] + (size_t)m->HP * H, H, m->P(p + "wk.weight"), H, m->maps, nullptr, m->HP, H, st));
            GVD_TRY(pack2d(m->wv[l], H, m->P(p + "wv.weight"), H, m->maps, nullptr, m->HP, H, st));
            GVD_TRY(pack2d(m->wo[l], m->HP, m->P(p + "wo.weight"), H, nullptr, m->maps, H, m->HP, st));
        }
    }
    for (int l = 0; l < 2; ++l) {
        const int in = l == 0 ? H : 2 * G;
        const std::string s = "_l" + std::to_string(l);
        const size_t wsz = (size_t)3 * G * in, hsz = (size_t)3 * G * G;
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_wih[l], m->P("context_enc.weight_ih" + s), wsz * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_wih[l] + wsz, m->P("context_enc.weight_ih" + s + "_reverse"), wsz * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_bih[l], m->P("context_enc.bias_ih" + s), 3 * G * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_bih[l] + 3 * G, m->P("context_enc.bias_ih" + s + "_reverse"), 3 * G * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_whh[l], m->P("context_enc.weight_hh" + s), hsz * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_whh[l] + hsz, m->P("context_enc.weight_hh" + s + "_reverse"), hsz * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_bhh[l], m->P("context_enc.bias_hh" + s), 3 * G * 4, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(m->gru_bhh[l] + 3 * G, m->P("context_enc.bias_hh" + s + "_reverse"), 3 * G * 4, cudaMemcpyDeviceToDevice, st));
    }
    {   // fp16x3 images of every constant weight that is the W operand of a forward GEMM (used when backend bit 4 is set)
        struct Ent { const float* W; long long ldw; int N, K; };
        std::vector<Ent> ents;
        const int E = d.input_encoding_size, V = d.vocab_size;
        ents.push_back({m->P("ctx2pool_grd.0.weight"), d.att_feat_size, 2048, d.att_feat_size});
        ents.push_back({m->vis_relu, 2048, m->NC, 2048});
        ents.push_back({m->pool_embed_w, m->PINp, H, m->PINp});
        ents.push_back({m->fc_embed_w, m->FCXp, H, m->FCXp});
        ents.push_back({m->P("ctx2pool.weight"), H, A, H});
        ents.push_back({m->P("ctx2att.weight"), H, A, H});
        ents.push_back({m->P("att_embed.0.0.weight"), m->rgb, H / 2, m->rgb});
        ents.push_back({m->P("att_embed.1.0.weight"), m->motion, H / 2, m->motion});
        ents.push_back({m->P("core.att_lstm.weight_ih"), H + E, 4 * H, H});                 // pre_att: the fc_feats columns
        ents.push_back({m->P("logit.weight"), H, V, H});
        ents.push_back({m->h2att_w, H, 2 * A, H});
        ents.push_back({m->w_att_cat, H + E, 4 * H, H + E});       // A operands of the conversion-free decode products (skinny_f16_kernel)
        ents.push_back({m->w_lang_cat, 3 * H, 4 * H, 3 * H});
        for (int l = 0; l < 2; ++l) {
            ents.push_back({m->gru_wih[l], l == 0 ? H : 2 * G, 6 * G, l == 0 ? H : 2 * G});
            ents.push_back({m->gru_whh[l], G, 6 * G, G});          // [2 directions][3G][G]: B operand of the tensor-core GRU step
            if (d.obj_interact) {
                const std::string p = "obj_interact.encoder.layers." + std::to_string(l) + ".";
                ents.push_back({m->wqk[l], H, 3 * m->HP, H});
                ents.push_back({m->wo[l], m->HP, H, m->HP});
                ents.push_back({m->P(p + "feedforward.layer.linear1.weight"), H, H / 2, H});
                ents.push_back({m->P(p + "feedforward.layer.linear2.weight"), H / 2, H, H / 2});
            }
        }
        size_t total = 0;
        for (auto& e : ents) total += rup((size_t)e.N * (size_t)((e.K + 31) / 32 * 32), 64);
        if (!m->packed16) GVD_CHECK_CUDA(cudaMalloc(&m->packed16, total * sizeof(float)));
        size_t off = 0;
        std::lock_guard<std::mutex> lk(g_pw_mu);
        for (const float* k : m->pw_keys) g_pw.erase(k);
        m->pw_keys.clear();
        for (auto& e : ents) {
            const long long Kp = (e.K + 31) / 32 * 32;
            GVD_TRY(gvd_pack_f16x3(e.W, e.ldw, e.N, e.K, m->packed16 + off, Kp, st));
            g_pw[e.W] = PackedW{m->packed16 + off, Kp, e.N, e.K, e.ldw};
            m->pw_keys.push_back(e.W);
            off += rup((size_t)e.N * (size_t)Kp, 64);
        }
    }
    m->finalized = true;
    return 0;
}

// ------------------------------------------------------------------------------------ workspace
struct WS {
    // inputs staged for the host-buffer entry point
    float *in_segs, *in_ppls, *in_feat, *out_att2, *out_sim, *out_logp;
    long long *in_num, *in_sidx, *out_seq;
    unsigned char* in_mask;
    // prologue
    float *fc_mean, *xcat, *fc_feats, *g_pool, *simT, *pool_in, *pool_embed, *pool_feats, *tmp_a, *qk, *vT, *vTl, *khi, *klo, *smxF, *S, *att_o, *ffn_h,
        *p_pool, *e, *gi, *gru_out0, *conv, *p_conv, *gh, *hstate;
    // decode
    float *pre_att, *h_att, *c_att, *h_lang, *c_lang, *q, *partial, *x_lang, *logits, *xt;
    float *xcat_att, *xcat_lang, *sk_part;   // split-K path: concatenated LSTM inputs, transposed partial sums [S][B][Nw]
    float *xp_att, *xp_lang;                 // the same concatenated inputs as fp16x3 operand images (conversion-free products, bit 4)
    float* q_part;                           // [4][B][2A] split-K partials of the query projection (summed inside the attention kernel)
    float *k_img, *vt_img;                   // fp16x3 images of the keys (per head) and of V^T for the fused self-attention (bit 8)
    float* a_pk_frame;                       // ... and the frame branch's own (P7 runs on a second stream next to P2-P6)
    float* a_pk;                             // fp16x3 image of the activation operand of the current prologue GEMM (bit 7)
    float *img_h, *img_ffn, *img_g;          // operand images written by the PRODUCER of an activation (GEMM epilogue / row kernel) instead of
                                             // a pack pass: [BR, H] (region embedding / encoder state), [BR, H/2] (FFN hidden), [BR, 2048] (fc7)
    int sk_ldp;
    long long* it;
    float* h_img;                      // [2 parity][2 dir][B][G] words: fp16x3 images of the GRU state (tensor-core step kernel)
    int* ticket;                       // [rows] last-CTA tickets of the fused attention combine
    float* pk_part; int* pk_ticket;    // fused vocabulary head + greedy pick: per-CTA partials, one ticket
    GvdSampleParams* sample_par;       // seed + temperature of the multinomial sampler, copied in before each decode
    float* vt_rec; int* vt_ticket;     // vocabularies above 6144 words: per-(row, slice) records and per-row tickets of gvd_vocab_tail
    // beam search (rows = B * beam)
    BeamBufs bb;
    int* bos_att;
    float *z_rows, *gather_tmp;
    float* att2_hist;                  // gvd_beam_decode_att2 only: [L][B*K][R] (with bb.parent_hist / bb.done_step)
    // teacher-forced path (MLE / GRD)
    float *ov, *outs, *z_all, *emb, *G, *logits_all, *part_sum;
    unsigned char *labels, *fm;
    int *target, *pred_cls, *cls_idx, *part_cnt;
    long long* tok_col;
    int RC, TC, nch_r, nch_t, clip_chunk, beam, nbox;
    int V;                             // > 0: video-indexed batch, the frame tensors hold V videos' rows (V = 0: one copy per clip)
    bool rows_n;                       // gvd_decode_sample_n: `beam` sampled rows per clip, no beam bookkeeping, row-sized loop outputs
    long long* in_vid;                 // [B] video of each clip (V > 0); the windows stay in in_sidx
    size_t bytes;
};

static void attn_chunking(int B, int R, int T, int* RC, int* TC) {
    const int target = std::max(1, gvd_cdiv(592, B));          // ~4 work items per SM
    auto pick = [&](int n) {
        int c = gvd_cdiv(n, target);
        c = (c + 7) / 8 * 8;
        return std::min(128, std::max(16, c));
    };
    *RC = pick(R);
    *TC = pick(T);
}

// att2_hist (beam > 1): also the beam's logit history for gvd_beam_decode_att2, after every other slot so that the layout without it is
// unchanged
// rows_n (beam > 1): the layout of gvd_decode_sample_n, `beam` sampled rows per clip; the loop's workspace-resident outputs then have one row
// per sampled caption and move to the end, so the prologue's slots stay where a per-clip layout has them (the per-clip out_seq / out_logp /
// out_att2 slots stay allocated and unused in this layout)
static WS ws_layout(const gvd_model* m, int B, int T, void* base, int beam = 1, int nbox = 0, int V = 0, bool att2_hist = false,
                    bool rows_n = false) {
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, R = m->R, G = m->G;
    WS w{};
    size_t off = 0;
    char* b0 = (char*)base;
    auto take = [&](size_t bytes) { size_t o = off; off += rup(bytes, 256); return (void*)(b0 ? b0 + o : (char*)0 + o); };
    const size_t NV = V > 0 ? V : B;          // rows of the frame branch: the clips, or the videos of a video-indexed batch
    const size_t BR = (size_t)B * R, BT = NV * T;
    const size_t BD = (size_t)B * beam;       // decode rows (beam rows of one clip share its features)
    w.beam = beam;
    w.V = V;
    w.rows_n = rows_n && beam > 1;
    attn_chunking((int)BD, R, T, &w.RC, &w.TC);
    gvd_attn_chunks(R, T, w.RC, w.TC, &w.nch_r, &w.nch_t);
    w.clip_chunk = std::max(1, std::min(B, (int)(100000000ll / ((long long)m->nheads * R * R * 4 + 1))));   // S chunk ~<= 100 MB (L2)
    // the attention kernels run one CTA per (clip, head, 128 query rows) and one CTA per SM: a chunk that is one full wave
    // (132 SMs -> 2 clips x 6 heads x 8 row blocks = 96 CTAs at R = 1000) has no partial second wave
    w.clip_chunk = std::max(1, std::min(w.clip_chunk, 132 / std::max(1, m->nheads * ((R + 127) / 128))));
    w.in_segs = (float*)take(BT * d.fc_feat_size * 4);
    w.in_ppls = (float*)take(BR * 7 * 4);
    w.in_feat = (float*)take(BR * d.att_feat_size * 4);
    w.in_num = (long long*)take((size_t)B * 7 * 8);
    w.in_sidx = (long long*)take((size_t)B * 2 * 8);
    // (ahead of every slot sized by beam / nbox: the prologue lays the workspace out for one row per clip, the beam and teacher-forced
    // decodes for theirs, and both must find the video indices at the same place)
    w.in_vid = V > 0 ? (long long*)take((size_t)B * 8) : nullptr;
    w.in_mask = (unsigned char*)take((size_t)B * (R + 1));
    w.out_seq = (long long*)take((size_t)B * d.seq_length * 8);
    w.out_logp = (float*)take((size_t)B * d.seq_length * 4);
    w.out_att2 = (float*)take((size_t)B * d.seq_length * R * 4);
    w.out_sim = (float*)take((size_t)B * m->NC * R * 4);
    w.fc_mean = (float*)take(NV * d.fc_feat_size * 4);
    w.xcat = (float*)take((size_t)B * m->FCXp * 4);
    w.fc_feats = (float*)take((size_t)B * H * 4);
    w.g_pool = (float*)take(BR * 2048 * 4);
    w.simT = (float*)take(BR * m->NCp * 4);
    w.pool_in = (float*)take(BR * m->PINp * 4);
    w.pool_embed = (float*)take(BR * H * 4);
    if (d.obj_interact) {
        w.pool_feats = (float*)take(BR * H * 4);
        w.tmp_a = (float*)take(BR * H * 4);
        w.qk = (float*)take(BR * 3 * m->HP * 4);
        w.vT = (float*)take((size_t)B * m->HP * R * 4);
        w.vTl = (float*)take((size_t)B * m->HP * R * 4);          // tf32 lo plane of V^T (vT then holds the hi plane)
        w.khi = (float*)take(BR * m->HP * 4);                     // tf32 hi / lo planes of the key projections
        w.klo = (float*)take(BR * m->HP * 4);
        w.smxF = (float*)take((size_t)w.clip_chunk * m->nheads * ((R + 31) / 32) * R * 4);   // softmax group factors of one chunk
        w.S = (float*)take((size_t)w.clip_chunk * m->nheads * R * R * 4);
        w.att_o = (float*)take(BR * m->HP * 4);
        w.k_img = (float*)take(BR * (size_t)m->nheads * ((m->HS + 31) / 32 * 32) * 4);
        w.vt_img = (float*)take((size_t)B * m->HP * ((R + 31) / 32 * 32) * 4);
        w.ffn_h = (float*)take(BR * (H / 2) * 4);
    } else {
        w.pool_feats = w.pool_embed;
    }
    w.p_pool = (float*)take(BR * A * 4);
    w.a_pk = (float*)take(BR * (size_t)std::max(std::max(m->PINp + 32, 2048 + 32), m->HP + 32) * 4);
    w.img_h = (float*)take(BR * (size_t)((m->d.rnn_size + 31) / 32 * 32) * 4);
    w.img_ffn = (float*)take(BR * (size_t)((m->d.rnn_size / 2 + 31) / 32 * 32) * 4);
    w.img_g = (float*)take(BR * (size_t)2048 * 4);
    w.e = (float*)take(BT * H * 4);
    w.gi = (float*)take(BT * 6 * G * 4);
    w.gru_out0 = (float*)take(BT * 2 * G * 4);
    w.conv = (float*)take(BT * H * 4);
    w.p_conv = (float*)take(BT * A * 4);
    w.gh = (float*)take((size_t)2 * NV * 3 * G * 4);
    w.hstate = (float*)take((size_t)2 * 2 * NV * G * 4);
    w.h_img = (float*)take((size_t)2 * 2 * NV * G * 4);
    w.a_pk_frame = (float*)take(BT * (size_t)((std::max(H, 2 * G) + 31) / 32 * 32 + 32) * 4);   // the frame branch's own pack buffer (it runs concurrently with the region stages)
    w.pre_att = (float*)take((size_t)B * 4 * H * 4);
    w.h_att = (float*)take(2 * BD * H * 4);
    w.c_att = (float*)take(BD * H * 4);
    w.h_lang = (float*)take(2 * BD * H * 4);
    w.c_lang = (float*)take(BD * H * 4);
    w.q = (float*)take(BD * 2 * A * 4);
    w.partial = (float*)take(BD * std::max(w.nch_r + w.nch_t, m->att_mode == GVD_ATT_INPUT_DUAL_REGION ? 2 * w.nch_r : 0) * (H + 4) * 4);
    w.x_lang = (float*)take(BD * H * 4);
    w.logits = (float*)take(BD * m->Vp * 4);
    w.it = (long long*)take(BD * 8);
    w.xt = (float*)take(BD * d.input_encoding_size * 4);
    w.sk_ldp = (int)rup(BD, 4);
    w.xcat_att = w.xcat_lang = w.sk_part = w.xp_att = w.xp_lang = nullptr;
    if (BD <= 128) {    // operand-swapped split-K path (BK_SPLITK): at most 132 (weight-row tile, K split) pairs per product
        w.xcat_att = (float*)take(BD * (size_t)(d.input_encoding_size + H) * 4);
        w.xcat_lang = (float*)take(BD * (size_t)3 * H * 4);
        w.sk_part = (float*)take((size_t)132 * 128 * w.sk_ldp * 4 + (size_t)BD * 64);      // [S][B][ldp], S * ceil(Nw/128) <= 132, ldp <= Nw + 3
        w.xp_att = (float*)take(BD * (size_t)(d.input_encoding_size + H) * 4);
        w.xp_lang = (float*)take(BD * (size_t)3 * H * 4);
        w.q_part = (float*)take((size_t)4 * BD * 2 * A * 4);
    }
    w.ticket = (int*)take(BD * 4);
    w.pk_part = (float*)take((size_t)gvd_cdiv(d.vocab_size, 32) * 128 * 8 * 4);
    w.pk_ticket = (int*)take(256);
    // the sampler's parameter block shares the ticket's slot: the workspace keeps the size and layout it has without sampling
    w.sample_par = (GvdSampleParams*)((char*)w.pk_ticket + 128);
    w.vt_rec = nullptr; w.vt_ticket = nullptr;
    if (d.vocab_size > 6144) {
        w.vt_rec = (float*)take(gvd_vocab_rec_floats((int)BD, d.vocab_size) * 4);
        w.vt_ticket = (int*)take(BD * 4);
    }
    if (beam > 1 && !w.rows_n) {
        const size_t L = d.seq_length, K = beam;
        w.bb.seq = (int*)take((size_t)B * L * K * 4);
        w.bb.att = (int*)take((size_t)B * L * K * 4);
        w.bb.lp = (float*)take((size_t)B * L * K * 4);
        w.bb.sums = (float*)take((size_t)B * K * 4);
        w.bb.parent = (int*)take(BD * 4);
        w.bb.att_ind = (int*)take(BD * 4);
        w.bb.done_flag = (int*)take((size_t)B * 4);
        w.bb.done_slot = (int*)take((size_t)B * 4);
        w.bb.done_seq = (int*)take((size_t)B * L * 4);
        w.bb.done_lp = (float*)take((size_t)B * L * 4);
        w.bb.topv = (float*)take(BD * K * 4);
        w.bb.topi = (int*)take(BD * K * 4);
        w.bb.tokens = (long long*)take(BD * 8);
        w.bos_att = (int*)take(BD * 4);
        w.z_rows = (float*)take(BD * R * 4);
        w.gather_tmp = (float*)take(BD * H * 4);
    }
    w.nbox = nbox;
    if (nbox > 0) {
        const size_t L = d.seq_length, NB = nbox;
        w.ov = (float*)take(BR * NB * 4);
        w.target = (int*)take((size_t)B * NB * R * 4);
        w.pred_cls = (int*)take(BR * 4);
        w.labels = (unsigned char*)take((size_t)B * L * R);
        w.fm = (unsigned char*)take((size_t)B * L * (R + 1));
        w.outs = (float*)take((size_t)B * L * H * 4);
        w.z_all = (float*)take((size_t)B * L * R * 4);
        w.emb = (float*)take((size_t)B * L * 2048 * 4);
        w.cls_idx = (int*)take((size_t)B * L * 4);
        w.G = (float*)take((size_t)B * L * R * 4);
        w.logits_all = (float*)take((size_t)B * L * m->Vp * 4);
        w.part_sum = (float*)take(std::max((size_t)B * L, (size_t)B * NB) * 4);
        w.part_cnt = (int*)take(std::max((size_t)B * L, (size_t)B * NB) * 4);
        w.tok_col = (long long*)take((size_t)B * 8);
    }
    if (w.rows_n) {
        w.out_seq = (long long*)take(BD * d.seq_length * 8);
        w.out_logp = (float*)take(BD * d.seq_length * 4);
        w.out_att2 = (float*)take(BD * d.seq_length * R * 4);
    }
    if (beam > 1 && att2_hist && !w.rows_n) {
        const size_t L = d.seq_length;
        w.att2_hist = (float*)take(L * BD * R * 4);       // step t's region-attention logits of every beam row, [L][B*K][R]
        w.bb.parent_hist = (int*)take(L * BD * 4);
        w.bb.done_step = (int*)take((size_t)B * 4);
    }
    w.bytes = off;
    return w;
}

extern "C" GVD_API size_t gvd_workspace_bytes(const gvd_model_t* m, int B, int T) {
    if (!m || B < 1 || T < 1) return 0;
    return ws_layout(m, B, T, nullptr).bytes;
}
extern "C" GVD_API size_t gvd_workspace_bytes_teacher(const gvd_model_t* m, int B, int T, int nbox) {
    if (!m || B < 1 || T < 1 || nbox < 1) return 0;
    return ws_layout(m, B, T, nullptr, 1, nbox).bytes;
}
extern "C" GVD_API size_t gvd_workspace_bytes_beam(const gvd_model_t* m, int B, int T, int beam_size) {
    if (!m || B < 1 || T < 1 || beam_size < 1) return 0;
    return ws_layout(m, B, T, nullptr, beam_size).bytes;
}

extern "C" GVD_API size_t gvd_workspace_bytes_beam_att2(const gvd_model_t* m, int B, int V, int T, int beam_size) {
    if (!m || B < 1 || V < 0 || T < 1 || beam_size < 2) return 0;
    return ws_layout(m, B, T, nullptr, beam_size, 0, V, true).bytes;
}

extern "C" GVD_API size_t gvd_workspace_bytes_sample_n(const gvd_model_t* m, int B, int V, int T, int n) {
    if (!m || B < 1 || V < 0 || T < 1 || n < 1) return 0;
    return ws_layout(m, B, T, nullptr, n, 0, V, false, true).bytes;
}

extern "C" GVD_API size_t gvd_workspace_bytes_video(const gvd_model_t* m, int B, int V, int T, int beam_size, int nbox) {
    if (!m || B < 1 || V < 1 || T < 1 || beam_size < 1 || nbox < 0) return 0;
    return ws_layout(m, B, T, nullptr, beam_size, nbox, V).bytes;
}

// V of the video prologue whose outputs sit in `workspace` for (B, T), 0 if a per-clip prologue (or none) filled it
static int video_of(const gvd_model* m, const void* workspace, int B, int T) {
    for (const VideoWs& v : m->video_ws)
        if (v.ws == workspace) return v.B == B && v.T == T ? v.V : 0;
    return 0;
}
static void set_video(gvd_model* m, void* workspace, int B, int T, int V) {
    auto& vs = m->video_ws;
    for (size_t i = 0; i < vs.size(); ++i)
        if (vs[i].ws == workspace) { vs.erase(vs.begin() + i); break; }
    if (V > 0) vs.push_back(VideoWs{workspace, B, T, V});
}

extern "C" GVD_API float* gvd_workspace_tensor(const gvd_model_t* m, void* workspace, int B, int T, const char* name) {
    if (!m || !workspace || !name) return nullptr;
    WS w = ws_layout(m, B, T, workspace, 1, 0, video_of(m, workspace, B, T));
    const std::string n(name);
    if (n == "fc_feats") return w.fc_feats;
    if (n == "g_pool") return w.g_pool;
    if (n == "pool_embed") return w.pool_embed;
    if (n == "pool_feats") return w.pool_feats;
    if (n == "p_pool_feats") return w.p_pool;
    if (n == "conv_feats") return w.conv;
    if (n == "p_conv_feats") return w.p_conv;
    if (n == "simT") return w.simT;
    if (n == "h_att") return w.h_att;
    if (n == "h_lang") return w.h_lang;
    if (n == "logits") return w.logits;
    return nullptr;
}

// V < 0: the layout the last prologue on this workspace left (video_of); V >= 0: that layout explicitly (a prologue about to run)
// the top-down captioner's decode and teacher-forced entry points: a BUTD model ('region') only feeds the transformer captioner
static int require_topdown(const gvd_model* m, const char* who) {
    GVD_REQUIRE(m, "%s: null model", who);
    GVD_REQUIRE(!m->butd, "%s: this model was built with enable_BUTD (att_input_mode 'region'), which only the transformer captioner runs; "
                "the top-down captioner does not take 'region'", who);
    return 0;
}

static int check_ws(const gvd_model* m, int B, int T, void* workspace, size_t bytes, WS* w, int beam = 1, int nbox = 0, int V = -1,
                    bool att2_hist = false, bool rows_n = false) {
    GVD_REQUIRE(m && m->finalized, "model not finalized (call gvd_model_finalize after setting every parameter)");
    GVD_REQUIRE(B >= 1 && T >= 1, "bad batch/frames B=%d T=%d", B, T);
    GVD_REQUIRE(workspace && ((uintptr_t)workspace & 255) == 0, "workspace must be a 256-byte aligned device pointer");
    *w = ws_layout(m, B, T, workspace, beam, nbox, V < 0 ? video_of(m, workspace, B, T) : V, att2_hist, rows_n);
    GVD_REQUIRE(bytes >= w->bytes, "workspace too small: %zu < %zu bytes", bytes, w->bytes);
    return 0;
}

// ------------------------------------------------------------------------------------ prologue
// C = act(A W^T + bias) for a constant, registered weight W.  Backend bit 7: pack the activation operand into the fp16x3 image (one
// element-wise pass: 4 B read + 4 B written per element) and run the conversion-free kernel (ss_gemm_kernel: TMA -> wgmma on two operand images);
// otherwise the conversion kernel (tc2_gemm_kernel) on the fp32 operand.
// Pack fusion: the producer of an activation can store its operand image directly (A_img: the image of A, pitch rup32(K), already
// written by whoever produced A; C_img: have THIS GEMM's epilogue store the image of its output, pitch rup32(N)) — the pack pass and
// its 8 B / element of traffic disappear.  C may be null when only the image is consumed.
static bool linear_w_f16ss(const WS& w, const float* W, long long ldw, int M, int N, int K, const float** Wp = nullptr, long long* ldwp = nullptr) {
    const float* p = nullptr;
    long long l = 0;
    const bool ok = gvd_backend_on(BK_SS_GEMM) && gvd_gemm_f16() && M >= 1024 && w.a_pk && gvd_packed_lookup(W, ldw, N, K, &p, &l);
    if (Wp) *Wp = p;
    if (ldwp) *ldwp = l;
    return ok;
}
static bool pack_fusion() { return gvd_backend_on(BK_PACK_FUSION); }
static int linear_w(const WS& w, const float* A, long long lda, const float* W, long long ldw, const float* bias, float* C, long long ldc, int M, int N,
                    int K, int act, cudaStream_t st, const float* scale2 = nullptr, const float* shift2 = nullptr, const float* A_img = nullptr,
                    float* C_img = nullptr) {
    const float* Wp = nullptr;
    long long ldwp = 0;
    const long long Kp = (K + 31) / 32 * 32, Np = (N + 31) / 32 * 32;
    if (linear_w_f16ss(w, W, ldw, M, N, K, &Wp, &ldwp)) {
        if (!A_img) {
            GVD_REQUIRE(A, "linear_w: no operand");
            GVD_STAGE("kernel.pack_f16x3", gvd_pack_f16x3(A, lda, M, K, w.a_pk, Kp, st, GVD_F16_SA));
            A_img = w.a_pk;
        }
        GVD_STAGE("kernel.f16ss_gemm", gvd_gemm_f16ss(A_img, Kp, Wp, ldwp, bias, scale2, shift2, act, C, ldc, M, N, K, st, C_img, C_img ? Np : 0));
        return 0;
    }
    GVD_REQUIRE(A && C, "linear_w: the conversion kernel needs the fp32 operand and output");
    GemmArgs g{};
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.C = C; g.ldc = ldc; g.bias = bias; g.scale2 = scale2; g.shift2 = shift2;
    g.M = M; g.N = N; g.K = K; g.nh = 1; g.act = act; g.alpha = 1.f;
    GVD_TRY(gvd_gemm_nt(g, 1, st));
    if (C_img) GVD_TRY(gvd_pack_f16x3(C, ldc, M, N, C_img, Np, st, GVD_F16_SA));
    return 0;
}

// clips [c0, c0 + B) of the batch the workspace was laid out for (every region buffer is clip-major, so a clip range is a row range)
static int obj_interact_fwd(const gvd_model* m, const WS& w0, int c0, int B, cudaStream_t st, bool fuse) {
    GvdF16Scope f16;
    const int H = m->d.rnn_size, R = m->R, HP = m->HP, HS = m->HS, nh = m->nheads;
    const long long BR = (long long)B * R, r0 = (long long)c0 * R;
    WS w = w0;
    w.pool_embed += r0 * H; w.pool_feats += r0 * H; w.tmp_a += r0 * H; w.qk += r0 * 3 * HP; w.vT += (long long)c0 * HP * R; w.vTl += (long long)c0 * HP * R; w.khi += r0 * HP; w.klo += r0 * HP;
    if (w.k_img) { w.k_img += r0 * nh * ((HS + 31) / 32 * 32); w.vt_img += (long long)c0 * HP * ((R + 31) / 32 * 32); }
    w.att_o += r0 * HP; w.ffn_h += r0 * (H / 2);
    const float* x = w.pool_embed;
    // pack fusion (decided by the caller): w.img_h holds the operand image of x on entry (written by the region-embedding GEMM) and of the
    // encoder state after every add & norm (on exit: of the output); the FFN hidden layer exists only as an image
    for (int l = 0; l < 2; ++l) {
        const std::string p = "obj_interact.encoder.layers." + std::to_string(l) + ".";
        // Q|K|V projections for every region in one GEMM (bias-free, transformer.py:111-114,119)
        const bool fused = gvd_backend_on(BK_TC | BK_FUSED_ATTN) && HS <= 192;
        const bool att16 = fused && gvd_backend_on(BK_ATT_F16) && w.k_img != nullptr;      // fp16x3 images instead of tf32 planes
        const int KH = (HS + 31) / 32 * 32, Rp = (R + 31) / 32 * 32;
        // pack fusion of the attention operands: the projection's epilogue stores Q as fp32, K as the per-head image and V as the image of V^T
        const float* Wp = nullptr;
        long long ldwp = 0;
        const bool qkv_img = fuse && att16 && R % 2 == 0 && HS % 4 == 0 && linear_w_f16ss(w, m->wqk[l], H, (int)BR, 3 * HP, H, &Wp, &ldwp);
        if (qkv_img) {
            GvdQkvImages qi{HP, HS, KH, nh, R, Rp, w.k_img, w.vt_img, GVD_ATT_SK, GVD_ATT_SV};
            ProfScope _pk("kernel.f16ss_gemm", st);
            GVD_STAGE("interact.qkv_proj", gvd_gemm_f16ss(w.img_h, (H + 31) / 32 * 32, Wp, ldwp, nullptr, nullptr, nullptr, GVD_ACT_NONE, w.qk, 3 * HP, (int)BR, 3 * HP, H,
                                                          st, nullptr, 0, &qi));
        } else
        GVD_STAGE("interact.qkv_proj", linear_w(w, x, H, m->wqk[l], H, nullptr, w.qk, 3 * HP, (int)BR, 3 * HP, H, GVD_ACT_NONE, st, nullptr, nullptr,
                                                fuse ? w.img_h : nullptr));
        if (qkv_img) {
        } else if (att16) {
            GVD_STAGE("interact.k_split", gvd_pack_heads_f16x3(w.qk + HP, 3 * HP, BR, nh, HS, HS, KH, GVD_ATT_SK, w.k_img, st));
            GVD_STAGE("interact.v_transpose", gvd_transpose_pack_f16x3(w.qk + 2 * HP, w.vt_img, B, R, HP, 3 * HP, Rp, GVD_ATT_SV, st));
        } else if (fused) {
            // tf32 hi / lo planes of K and V^T, made once per layer: the two attention kernels then stream them without converting
            GVD_STAGE("interact.k_split", gvd_split_hilo(w.qk + HP, 3 * HP, w.khi, w.klo, HP, BR, HP, st));
            GVD_STAGE("interact.v_transpose", gvd_transpose_split(w.qk + 2 * HP, w.vT, w.vTl, B, R, HP, 3 * HP, st));
        } else {
            // V^T per clip (the P.V product is then again an NT GEMM with K = R contiguous)
            GVD_STAGE("interact.v_transpose", gvd_transpose(w.qk + 2 * HP, w.vT, B, R, HP, 3 * HP, st));
        }
        // With pack fusion the attention stores the operand image of the output projection's input (no fp32 att_o, no pack pass).
        const long long HPi = (HP + 31) / 32 * 32;
        const bool o_img = fuse && att16 && HS % 4 == 0 && linear_w_f16ss(w, m->wo[l], HP, (int)BR, H, HP);
        if (att16) {
            // softmax(Q K^T / sqrt(d_model)) V of every clip and head in one launch, the scores never leave the SM
            // (the scale is sqrt(1024)=32, not sqrt(d_head): transformer.py:94,111; quirk Q1)
            GVD_STAGE("interact.attn", gvd_self_attn_fused(w.qk, 3 * HP, w.k_img, w.vt_img, B, R, nh, HS, HP, 1.f / sqrtf((float)H), w.att_o, HP,
                                                           o_img ? w.a_pk : nullptr, HPi, st));
        } else
        for (int b0 = 0; b0 < B; b0 += w.clip_chunk) {
            const int cb = std::min(w.clip_chunk, B - b0);
            {   // S[b,h] = Q_h K_h^T  (heads are zero-padded to HS columns)
                GemmArgs g{};
                g.A = w.qk + (long long)b0 * R * 3 * HP; g.lda = 3 * HP; g.sAb = (long long)R * 3 * HP; g.sAh = HS;
                g.W = g.A + HP; g.ldw = 3 * HP; g.sWb = g.sAb; g.sWh = HS;
                g.C = w.S; g.ldc = R; g.sCb = (long long)nh * R * R; g.sCh = (long long)R * R;
                g.M = R; g.N = R; g.K = HS; g.nh = nh; g.alpha = 1.f;
                if (fused) {
                    // scores + softmax numerator in one sweep: E = exp((s - mu_group)/sqrt(d_model)), group factors -> smxF
                    // (the scale is sqrt(1024)=32, not sqrt(d_head): transformer.py:94,111; quirk Q1)
                    g.W = w.khi + (long long)b0 * R * HP; g.ldw = HP; g.sWb = (long long)R * HP;
                    GVD_STAGE("interact.scores", gvd_attn_scores_tc(g, w.klo + (long long)b0 * R * HP, w.smxF, 1.f / sqrtf((float)H), cb * nh, st));
                } else {
                    GVD_STAGE("interact.scores", gvd_gemm_nt(g, cb * nh, st));
                }
            }
            // softmax(S / sqrt(d_model)) — the scale is sqrt(1024)=32, not sqrt(d_head) (transformer.py:94,111; quirk Q1)
            if (!fused) GVD_STAGE("interact.softmax", gvd_scaled_softmax_rows(w.S, (long long)cb * nh * R, R, R, 1.f / sqrtf((float)H), st));
            {   // O_h = P V_h
                GemmArgs g{};
                g.A = w.S; g.lda = R; g.sAb = (long long)nh * R * R; g.sAh = (long long)R * R;
                g.W = w.vT + (long long)b0 * HP * R; g.ldw = R; g.sWb = (long long)HP * R; g.sWh = (long long)HS * R;
                g.C = w.att_o + (long long)b0 * R * HP; g.ldc = HP; g.sCb = (long long)R * HP; g.sCh = HS;
                g.M = R; g.N = HS; g.K = R; g.nh = nh; g.alpha = 1.f;
                if (fused) GVD_STAGE("interact.pv", gvd_attn_pv_tc(g, w.vTl + (long long)b0 * HP * R, w.smxF, cb * nh, st));
                else GVD_STAGE("interact.pv", gvd_gemm_nt(g, cb * nh, st));
            }
        }
        GVD_STAGE("interact.wo", linear_w(w, w.att_o, HP, m->wo[l], HP, nullptr, w.tmp_a, H, (int)BR, H, HP, GVD_ACT_NONE, st, nullptr, nullptr, o_img ? w.a_pk : nullptr));
        GVD_STAGE("interact.add_ln", gvd_add_ln_star(x, w.tmp_a, m->P(p + "selfattn.layernorm.gamma"), m->P(p + "selfattn.layernorm.beta"), w.pool_feats, BR, H, st,
                                                     fuse ? w.img_h : nullptr));
        const float* w1 = m->P(p + "feedforward.layer.linear1.weight");
        const float* w2 = m->P(p + "feedforward.layer.linear2.weight");
        const bool hid_img = fuse && linear_w_f16ss(w, w1, H, (int)BR, H / 2, H) && linear_w_f16ss(w, w2, H / 2, (int)BR, H, H / 2);
        GVD_STAGE("interact.ffn1", linear_w(w, w.pool_feats, H, w1, H, m->P(p + "feedforward.layer.linear1.bias"), hid_img ? nullptr : w.ffn_h, H / 2, (int)BR,
                                            H / 2, H, GVD_ACT_RELU, st, nullptr, nullptr, fuse ? w.img_h : nullptr, hid_img ? w.img_ffn : nullptr));
        GVD_STAGE("interact.ffn2", linear_w(w, w.ffn_h, H / 2, w2, H / 2, m->P(p + "feedforward.layer.linear2.bias"), w.tmp_a, H, (int)BR, H, H / 2, GVD_ACT_NONE,
                                            st, nullptr, nullptr, hid_img ? w.img_ffn : nullptr));
        GVD_STAGE("interact.add_ln", gvd_add_ln_star(w.pool_feats, w.tmp_a, m->P(p + "feedforward.layernorm.gamma"), m->P(p + "feedforward.layernorm.beta"),
                                w.pool_feats, BR, H, st, fuse ? w.img_h : nullptr));
        x = w.pool_feats;
    }
    return 0;
}

// One bidirectional GRU layer step by step: gh = W_hh h(t-1) + b_hh of both directions in one batched GEMM, then the pointwise cell.
// hstate [2 parity][2 dir][B][G] zeroed by the caller, gh [2 dir][B][3G] scratch, whh [2][3G][G], bhh [2][3G].
static int gru_layer_steps(const float* gi, const float* whh, const float* bhh, float* hstate, float* gh, float* out,
                           const long long* sample_idx, int B, int T, int G, cudaStream_t st) {
    for (int s = 0; s < T; ++s) {
        float* h_prev = hstate + (size_t)(s & 1) * 2 * B * G;
        float* h_new = hstate + (size_t)((s + 1) & 1) * 2 * B * G;
        GemmArgs g{};
        g.A = h_prev; g.lda = G; g.sAb = (long long)B * G;
        g.W = whh; g.ldw = G; g.sWb = (long long)3 * G * G;
        g.bias = bhh; g.sBb = 3 * G;
        g.C = gh; g.ldc = 3 * G; g.sCb = (long long)B * 3 * G;
        g.M = B; g.N = 3 * G; g.K = G; g.nh = 1; g.alpha = 1.f;
        GVD_STAGE("frame.gru_hh", gvd_gemm_nt(g, 2, st));
        GVD_STAGE("frame.gru_pointwise", gvd_gru_pointwise(gi, gh, h_prev, h_new, out, sample_idx, B, T, G, s, st));
    }
    return 0;
}

static int frame_branch_fwd(const gvd_model* m, const WS& w0, int B, int T, const float* segs, const long long* sample_idx,
                            cudaStream_t st) {
    GvdF16Scope f16;
    WS w = w0;
    w.a_pk = w0.a_pk_frame;                 // (the region stages may be packing into a_pk on another stream)
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, G = m->G, FC = d.fc_feat_size;
    const long long BT = (long long)B * T;
    // att_embed (rgb | motion) -> BatchNorm1d(eval) -> ReLU fused into the GEMM epilogue (model.py:556-560)
    {
        GemmArgs g{};
        g.A = segs; g.lda = FC; g.W = m->P("att_embed.0.0.weight"); g.ldw = m->rgb; g.bias = m->P("att_embed.0.0.bias");
        g.C = w.e; g.ldc = H; g.M = (int)BT; g.N = H / 2; g.K = m->rgb; g.nh = 1; g.alpha = 1.f;
        g.act = GVD_ACT_RELU_AFFINE_RELU; g.scale2 = m->bn_scale; g.shift2 = m->bn_shift;
        GVD_STAGE("frame.att_embed", gvd_gemm_nt(g, 1, st));
        g.A = segs + m->rgb; g.W = m->P("att_embed.1.0.weight"); g.ldw = m->motion; g.bias = m->P("att_embed.1.0.bias");
        g.C = w.e + H / 2; g.K = m->motion; g.scale2 = m->bn_scale + H / 2; g.shift2 = m->bn_shift + H / 2;
        GVD_STAGE("frame.att_embed", gvd_gemm_nt(g, 1, st));
    }
    // 2-layer bidirectional GRU, hidden G per direction (model.py:150-154,562)
    for (int l = 0; l < 2; ++l) {
        const float* xin = l == 0 ? w.e : w.gru_out0;
        const int in = l == 0 ? H : 2 * G;
        float* out = l == 0 ? w.gru_out0 : w.conv;
        GVD_STAGE("frame.gru_in", linear_w(w, xin, in, m->gru_wih[l], in, m->gru_bih[l], w.gi, 6 * G, (int)BT, 6 * G, in, GVD_ACT_NONE, st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.hstate, 0, (size_t)2 * 2 * B * G * sizeof(float), st));
        {
            // tensor-core step kernel (bit 4): gh = W_hh h on wgmma from two pre-split operands with the gate math in the epilogue — one
            // launch per time step instead of a CUDA-core GEMM + a pointwise kernel
            const float* Wimg = nullptr;
            long long ldw = 0;
            if (gvd_gemm_f16() && B <= 128 && G % 32 == 0 && gvd_packed_lookup(m->gru_whh[l], G, 6 * G, G, &Wimg, &ldw)) {
                GVD_STAGE("frame.gru_layer_tc", gvd_gru_layer_f16(w.gi, Wimg, m->gru_bhh[l], w.hstate, w.h_img, out, l == 1 ? sample_idx : nullptr, B, T, G, st));
                continue;
            }
        }
        GVD_TRY(gru_layer_steps(w.gi, m->gru_whh[l], m->gru_bhh[l], w.hstate, w.gh, out, l == 1 ? sample_idx : nullptr, B, T, G, st));
    }
    GVD_STAGE("frame.ctx2att", gvd_linear(w.conv, H, m->P("ctx2att.weight"), H, m->P("ctx2att.bias"), w.p_conv, A, (int)BT, A, H, GVD_ACT_NONE, st));
    return 0;
}

// P2-P6 for clips [c0, c0 + cb): per-clip independent, so the host-buffer entry point can run it chunk by chunk
// while the next chunk's fc6 features are still crossing PCIe.  Input pointers are already offset to clip c0.
static int region_prologue(const gvd_model* m, const WS& w0, int c0, int cb, const float* ppls, const float* ppls_feat,
                           const uint8_t* pnt_mask, float* sim_mat_out, cudaStream_t st) {
    GvdF16Scope f16;
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, R = m->R;
    const int B = cb;
    const long long BR = (long long)cb * R, r0 = (long long)c0 * R;
    WS w = w0;
    w.g_pool += r0 * 2048; w.simT += r0 * m->NCp; w.pool_in += r0 * m->PINp; w.pool_embed += r0 * H; w.p_pool += r0 * A;
    if (d.obj_interact) w.pool_feats += r0 * H; else w.pool_feats = w.pool_embed;
    // P2 fc7 on every RoI (model.py:512-514)
    // pack fusion (see linear_w): fc7's epilogue also stores the image the similarity GEMM streams; the region-embedding row kernel writes the
    // image of its 2784-wide row and nothing else; the embedding GEMM stores the image the encoder's first projection / ctx2pool stream
    const bool fuse = pack_fusion() && H % 64 == 0 && linear_w_f16ss(w, m->P("ctx2pool.weight"), H, (int)BR, A, H) &&
                      linear_w_f16ss(w, m->pool_embed_w, m->PINp, (int)BR, H, m->PINp) && linear_w_f16ss(w, m->vis_relu, 2048, (int)BR, m->NC, 2048) &&
                      (!d.obj_interact || linear_w_f16ss(w, m->wqk[0], H, (int)BR, 3 * m->HP, H));
    // BUTD with pack fusion: every reader of fc7 (pool_embed, the similarity) streams its operand image, so the epilogue stores the image alone
    GVD_STAGE("region.fc7", linear_w(w, ppls_feat, d.att_feat_size, m->P("ctx2pool_grd.0.weight"), d.att_feat_size, m->P("ctx2pool_grd.0.bias"),
                                     m->butd && fuse ? nullptr : w.g_pool, 2048, (int)BR, 2048, d.att_feat_size, GVD_ACT_RELU, st, nullptr, nullptr, nullptr,
                                     fuse ? w.img_g : nullptr));
    // P3 region-class similarity, stored region-major: simT[(b,r), c] (model.py:519-535); transfer_mode 'none' has no class bias (P() is NULL).
    // BUTD: the region features do not read it (model.py:357-364), so it runs only for the caller's sim_mat_out
    if (!m->butd || sim_mat_out) {
        GVD_STAGE("region.sim_gemm", linear_w(w, w.g_pool, 2048, m->vis_relu, 2048, m->P("vis_classifiers_bias"), w.simT, m->NCp, (int)BR, m->NC, 2048, GVD_ACT_NONE,
                                              st, nullptr, nullptr, fuse ? w.img_g : nullptr));
        GVD_STAGE("region.sim_softmax", gvd_sim_softmax(w.simT, pnt_mask, B, R, m->NC, m->NCp, st));
    }
    if (sim_mat_out) GVD_STAGE("region.sim_transpose", gvd_transpose(w.simT, sim_mat_out, B, R, m->NC, m->NCp, st));
    // P4 region embedding (model.py:537-547); BUTD: pool_embed on fc7 alone, K = 2048 (model.py:65-69,384)
    if (m->butd) {
        GVD_STAGE("region.pool_embed", linear_w(w, w.g_pool, 2048, m->pool_embed_w, m->PINp, m->P("pool_embed.0.bias"), w.pool_embed, H, (int)BR, H, 2048,
                                                GVD_ACT_RELU, st, nullptr, nullptr, fuse ? w.img_g : nullptr, fuse ? w.img_h : nullptr));
    } else {
        const int PINi = (m->PINp + 31) / 32 * 32;
        GVD_STAGE("region.pool_in", gvd_pool_in(w.g_pool, ppls, w.simT, m->P("loc_fc.0.weight"), m->P("loc_fc.0.bias"), fuse ? nullptr : w.pool_in, BR, 2048, 300,
                                                m->NC, m->NCp, m->PINp, d.num_sampled_frm, st, fuse ? w.a_pk : nullptr, PINi));
        GVD_STAGE("region.pool_embed", linear_w(w, w.pool_in, m->PINp, m->pool_embed_w, m->PINp, m->P("pool_embed.0.bias"), w.pool_embed, H, (int)BR, H, m->PINp,
                                                GVD_ACT_RELU, st, nullptr, nullptr, fuse ? w.a_pk : nullptr, fuse ? w.img_h : nullptr));
    }
    // P5 object interaction (model.py:550-551)
    if (d.obj_interact) GVD_TRY(obj_interact_fwd(m, w0, c0, cb, st, fuse));
    // P6 (model.py:554)
    GVD_STAGE("region.ctx2pool", linear_w(w, w.pool_feats, H, m->P("ctx2pool.weight"), H, m->P("ctx2pool.bias"), w.p_pool, A, (int)BR, A, H, GVD_ACT_NONE, st,
                                          nullptr, nullptr, fuse ? w.img_h : nullptr));
    return 0;
}

// P1 + P7 + the constant part of the attention-LSTM gates: everything that only needs the frame features.
// Video-indexed batch (w.V > 0, vid = the workspace's copy of video_idx): segs_feat holds V videos; the frame mean and the frame branch run
// once per video, the latter unmasked (the decode attention applies each clip's window), and clip b's vector reads video vid[b]'s mean.
static int frame_stages(const gvd_model* m, const WS& w, int B, int T, const float* segs_feat, const long long* num, const long long* sample_idx,
                        cudaStream_t st, const long long* vid = nullptr) {
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, E = d.input_encoding_size, FC = d.fc_feat_size;
    const int NV = vid ? w.V : B;
    // P1 clip vector (model.py:508-510,548)
    GVD_STAGE("clip.frame_mean", gvd_frame_mean(segs_feat, w.fc_mean, NV, T, FC, st));
    GVD_STAGE("clip.vector", gvd_clip_vector(w.fc_mean, num, m->P("seg_info_embed.0.weight"), m->P("seg_info_embed.0.bias"), w.xcat, B, FC, 50, m->FCXp, st,
                                             vid));
    GVD_STAGE("clip.fc_embed", gvd_linear(w.xcat, m->FCXp, m->fc_embed_w, m->FCXp, m->P("fc_embed.0.bias"), w.fc_feats, H, B, H, m->FCXp, GVD_ACT_RELU, st));
    // P7 frame branch (model.py:556-565); dual_region reads no frame features (model.py:393: dummies)
    if (m->att_mode != GVD_ATT_INPUT_DUAL_REGION) GVD_TRY(frame_branch_fwd(m, w, NV, T, segs_feat, vid ? nullptr : sample_idx, st));
    // constant part of the attention-LSTM gates: W_ih[:, :H] fc_feats + b_ih + b_hh (fc_feats is the same at every step)
    GVD_STAGE("decode.pre_att", gvd_linear(w.fc_feats, H, m->P("core.att_lstm.weight_ih"), H + E, m->att_bias_sum, w.pre_att, 4 * H, B, 4 * H, H, GVD_ACT_NONE, st));
    return 0;
}

// The frame stages next to the region stages (P2-P6) instead of behind them: the bi-GRU is 2 * 2 * T dependent launches of a few CTAs
// that nothing else in the prologue depends on.  They run on a second stream; no GEMM here is persistent, so the chain's CTAs find SMs as
// the region kernels' CTAs retire.  Off under the stage profiler (its per-stage times are meant to be serial).
static bool frame_overlap_on() { return g_prof_on.load(std::memory_order_relaxed) == 0; }
static int frame_fork(gvd_model* m, cudaStream_t st) {
    if (!m->frame_stream) {
        int lo = 0, hi = 0;
        GVD_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        // lowest priority: at the highest one the GRU chain can hold back every region kernel until it ends
        GVD_CHECK_CUDA(cudaStreamCreateWithPriority(&m->frame_stream, cudaStreamNonBlocking, lo));
        GVD_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_fork, cudaEventDisableTiming));
        GVD_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_join, cudaEventDisableTiming));
    }
    GVD_CHECK_CUDA(cudaEventRecord(m->ev_fork, st));              // the workspace may still be in use by earlier work on `st`
    GVD_CHECK_CUDA(cudaStreamWaitEvent(m->frame_stream, m->ev_fork, 0));
    return 0;
}
static int frame_join(gvd_model* m, cudaStream_t st) {
    GVD_CHECK_CUDA(cudaEventRecord(m->ev_join, m->frame_stream));
    GVD_CHECK_CUDA(cudaStreamWaitEvent(st, m->ev_join, 0));
    return 0;
}
// V = 0: per-clip batch; V > 0: video-indexed batch (segs_feat [V,T,F], video_idx [B])
static int prologue_run(gvd_model_t* m, int B, int V, int T, const float* segs_feat, const float* ppls, const int64_t* num,
                        const float* ppls_feat, const int64_t* sample_idx, const int64_t* video_idx, const uint8_t* pnt_mask, void* workspace,
                        size_t workspace_bytes, float* sim_mat_out, void* stream) {
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w, 1, 0, V));
    GVD_REQUIRE(segs_feat && ppls && num && ppls_feat && sample_idx && pnt_mask && (V == 0 || video_idx), "prologue: null input");
    cudaStream_t st = (cudaStream_t)stream;
    set_video(m, workspace, B, T, V);
    if (V > 0) {       // the decode entries read each clip's video and window from the workspace
        GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_vid, video_idx, (size_t)B * 8, cudaMemcpyDeviceToDevice, st));
        GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_sidx, sample_idx, (size_t)B * 2 * 8, cudaMemcpyDeviceToDevice, st));
    }
    const bool overlap = frame_overlap_on();
    cudaStream_t fst = st;
    if (overlap) { GVD_TRY(frame_fork(m, st)); fst = m->frame_stream; }
    const int rc_frame = frame_stages(m, w, B, T, segs_feat, (const long long*)num, (const long long*)sample_idx, fst, V > 0 ? w.in_vid : nullptr);
    if (overlap && rc_frame != 0) frame_join(m, st);            // never leave the second stream dangling behind an error return
    if (rc_frame != 0) return rc_frame;
    const int rc = region_prologue(m, w, 0, B, ppls, ppls_feat, pnt_mask, sim_mat_out, st);          // P2-P6
    if (overlap) GVD_TRY(frame_join(m, st));
    return rc;
}
extern "C" GVD_API int gvd_prologue_fwd(gvd_model_t* m, int B, int T, const float* segs_feat, const float* ppls, const int64_t* num,
                                const float* ppls_feat, const int64_t* sample_idx, const uint8_t* pnt_mask, void* workspace,
                                size_t workspace_bytes, float* sim_mat_out, void* stream) {
    return prologue_run(m, B, 0, T, segs_feat, ppls, num, ppls_feat, sample_idx, nullptr, pnt_mask, workspace, workspace_bytes, sim_mat_out, stream);
}
extern "C" GVD_API int gvd_prologue_fwd_video(gvd_model_t* m, int B, int V, int T, const float* segs_feat, const float* ppls, const int64_t* num,
                                              const float* ppls_feat, const int64_t* sample_idx, const int64_t* video_idx, const uint8_t* pnt_mask,
                                              void* workspace, size_t workspace_bytes, float* sim_mat_out, void* stream) {
    GVD_REQUIRE(V >= 1, "prologue_video: V=%d must be >= 1", V);
    return prologue_run(m, B, V, T, segs_feat, ppls, num, ppls_feat, sample_idx, video_idx, pnt_mask, workspace, workspace_bytes, sim_mat_out, stream);
}

// ------------------------------------------------------------------------------------ decode
// zero recurrent state and tickets of the layout's B * beam decode rows
static int reset_state(const gvd_model* m, const WS& w, int B, cudaStream_t st) {
    const size_t n = (size_t)B * w.beam * m->d.rnn_size * sizeof(float);
    GVD_CHECK_CUDA(cudaMemsetAsync(w.h_att, 0, 2 * n, st));     // init_hidden: zeros (model.py:237-240)
    GVD_CHECK_CUDA(cudaMemsetAsync(w.c_att, 0, n, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(w.h_lang, 0, 2 * n, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(w.c_lang, 0, n, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(w.ticket, 0, (size_t)B * w.beam * sizeof(int), st));
    GVD_CHECK_CUDA(cudaMemsetAsync(w.pk_ticket, 0, sizeof(int), st));
    if (w.vt_ticket) GVD_CHECK_CUDA(cudaMemsetAsync(w.vt_ticket, 0, (size_t)B * w.beam * sizeof(int), st));
    if (w.xcat_att) {      // split-K path: the recurrent states also live inside the concatenated LSTM inputs
        GVD_CHECK_CUDA(cudaMemsetAsync(w.xcat_att, 0, (size_t)B * w.beam * (m->d.input_encoding_size + m->d.rnn_size) * sizeof(float), st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.xcat_lang, 0, (size_t)B * w.beam * 3 * m->d.rnn_size * sizeof(float), st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.xp_att, 0, (size_t)B * w.beam * (m->d.input_encoding_size + m->d.rnn_size) * sizeof(float), st));   // +0 halves
        GVD_CHECK_CUDA(cudaMemsetAsync(w.xp_lang, 0, (size_t)B * w.beam * 3 * m->d.rnn_size * sizeof(float), st));
    }
    return 0;
}

extern "C" GVD_API int gvd_decode_reset_state(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, void* stream) {
    GVD_TRY(require_topdown(m, "decode_reset_state"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w));
    return reset_state(m, w, B, (cudaStream_t)stream);
}

// does the core step run its three products operand-swapped + split along K (gvd_skinny.cu)?  Then xt / h_att / h_lang live inside the
// concatenated LSTM inputs xcat_att = [xt | h_att] and xcat_lang = [att + att2 | h_att | h_lang].
static bool core_skinny(const gvd_model* m, const WS& w, int B, int div) {
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, E = d.input_encoding_size;
    return gvd_backend_on(BK_TC | BK_SPLITK) && H % 8 == 0 && (div == 1 || w.rows_n) && w.sk_part != nullptr && E % 4 == 0 &&
           gvd_skinny_splits(4 * H, E + H, B) > 0 && gvd_skinny_splits(2 * A, H, B) > 0 && gvd_skinny_splits(4 * H, 3 * H, B) > 0;
}

// ... and with backend bit 4 through the conversion-free kernel: weights AND activations in the fp16x3 operand image (needs 32-column
// granularity of every concatenated segment)
static bool core_skinny_f16(const gvd_model* m) {
    const gvd_dims_t& d = m->d;
    return gvd_backend_on(BK_F16X3) && d.rnn_size % 32 == 0 && d.input_encoding_size % 32 == 0 && d.att_hid_size % 16 == 0;
}

// B = decode rows (clips x beam or sampled rows); rows [k*div, (k+1)*div) attend over clip k's features / masks.  The split-K products take
// any div in the sampled-rows layout (no beam reorder of the recurrent rows, which would have to reach into the concatenated inputs)
static int core_step(const gvd_model* m, const WS& w, int B, int T, int step, const long long* tokens, const unsigned char* att_mask,
                     const unsigned char* out_mask, float* z_out, long long z_stride_b, cudaStream_t st, int div = 1, long long out_mask_stride = 0,
                     bool xt_ready = false) {
    GvdF16Scope f16;
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, A = d.att_hid_size, E = d.input_encoding_size, R = m->R;
    const size_t BH = (size_t)B * H;
    float* h_att_cur = w.h_att + (size_t)(step & 1) * BH;
    float* h_att_nxt = w.h_att + (size_t)((step + 1) & 1) * BH;
    float* h_lang_cur = w.h_lang + (size_t)(step & 1) * BH;
    float* h_lang_nxt = w.h_lang + (size_t)((step + 1) & 1) * BH;
    const bool tc = gvd_backend_on(BK_TC) && H % 8 == 0;
    // operand-swapped split-K products (gvd_skinny.cu, BK_SPLITK); one `pre` row per batch row only
    const bool skinny = core_skinny(m, w, B, div);
    const bool sk16 = skinny && core_skinny_f16(m);     // both operands pre-split: conversion-free products (skinny_f16_kernel)
    {   // attention LSTM: input cat(fc_feats, xt), xt = ReLU(embed[token]) (AttModel.py:138-139)
        LstmArgs a{};
        a.nseg = 2;
        a.seg[0] = LstmSeg{m->P("embed.0.weight"), E, tokens, 1, m->P("core.att_lstm.weight_ih") + H, H + E, E};
        a.seg[1] = LstmSeg{h_att_cur, H, nullptr, 0, m->P("core.att_lstm.weight_hh"), H, H};
        a.pre = w.pre_att; a.pre_div = div;
        a.c_prev = w.c_att; a.c_out = w.c_att; a.h_out = h_att_nxt; a.B = B; a.H = H;
        if (tc) {
            // split-K path: the input [xt | h_att(t-1)] is ONE matrix (xcat_att): the sampler / this embedding write xt into its first E
            // columns, the previous step's reduction wrote h_att into the rest; no concat launch
            if (!xt_ready) {
                embed_relu_kernel<<<gvd_cdiv((long long)B * E, 256), 256, 0, st>>>(m->P("embed.0.weight"), tokens, skinny ? w.xcat_att : w.xt, skinny ? E + H : E, B,
                                                                                 E, d.vocab_size, sk16 ? w.xp_att : nullptr, E + H);
                GVD_CHECK_LAUNCH();
            }
            a.seg[0] = LstmSeg{w.xt, E, nullptr, 0, m->P("core.att_lstm.weight_ih") + H, H + E, E};
            if (skinny) {
                const int S = gvd_skinny_splits(4 * H, E + H, B);
                const float* Wp; long long ldwp;
                if (sk16 && gvd_packed_lookup(m->w_att_cat, E + H, 4 * H, E + H, &Wp, &ldwp)) {
                    GVD_STAGE("decode.lstm_att", gvd_skinny_f16(Wp, ldwp, 4 * H, w.xp_att, E + H, B, E + H, S, w.sk_part, 4 * H, st));
                } else {
                    GVD_REQUIRE(!sk16, "core_step: packed attention-LSTM weights missing");
                    GVD_STAGE("decode.lstm_att", gvd_skinny_splitk(m->w_att_cat, 4 * H, E + H, w.xcat_att, E + H, B, S, w.sk_part, 4 * H, st));
                }
                GVD_STAGE("decode.lstm_att_reduce", gvd_reduce_lstm(w.sk_part, S, 4 * H, a.pre, a.pre_div, nullptr, nullptr, a.c_prev, a.c_out, a.h_out, H,
                                                                    w.xcat_att + E, E + H, w.xcat_lang + H, 3 * H, B, H, st,
                                                                    sk16 ? w.xp_att + E : nullptr, E + H, sk16 ? w.xp_lang + H : nullptr, 3 * H));
            } else {
                GVD_STAGE("decode.lstm_att", gvd_lstm_step_tc(a, st));
            }
        } else {
            GVD_STAGE("decode.lstm_att", gvd_lstm_step(a, st));
        }
    }
    // both attention queries in one GEMM: q = [h2att(h_a) | h2att2(h_a)]
    int q_S = 0;          // > 0: the queries stay as q_S split-K partials in w.q_part, summed by the attention kernel
    {
        if (skinny) {
            const int S = gvd_skinny_splits(2 * A, H, B);
            const float* Wp; long long ldwp;
            if (sk16 && gvd_packed_lookup(m->h2att_w, H, 2 * A, H, &Wp, &ldwp)) {
                // 4 splits only: the attention kernel sums the partials itself while it loads its query (no reduction launch)
                q_S = std::min(S, 4);
                while (H % (32 * q_S) != 0) --q_S;
                GVD_STAGE("decode.h2att", gvd_skinny_f16(Wp, ldwp, 2 * A, w.xp_lang + H, 3 * H, B, H, q_S, w.q_part, 2 * A, st));       // X = h_att(t) inside xp_lang
            } else {
                GVD_REQUIRE(!sk16, "core_step: packed query weights missing");
                GVD_STAGE("decode.h2att", gvd_skinny_splitk(m->h2att_w, 2 * A, H, h_att_nxt, H, B, S, w.sk_part, 2 * A, st));
            }
            if (!q_S) GVD_STAGE("decode.h2att_reduce", gvd_reduce_bias(w.sk_part, S, 2 * A, 2 * A, m->h2att_b, w.q, 2 * A, B, st));
        } else {
            GVD_STAGE("decode.h2att", gvd_linear(h_att_nxt, H, m->h2att_w, H, m->h2att_b, w.q, 2 * A, B, 2 * A, H, GVD_ACT_NONE, st));
        }
    }
    {
        AttnArgs a{};
        a.p_pool = w.p_pool; a.pool = w.pool_feats; a.p_conv = w.p_conv; a.conv = w.conv; a.q = w.q;
        if (q_S) { a.q = nullptr; a.q_part = w.q_part; a.q_S = q_S; a.q_plane = (long long)B * 2 * A; a.q_bias = m->h2att_b; }
        a.w1 = m->P("core.attention.alpha_net.weight"); a.b1 = m->P("core.attention.alpha_net.bias");
        if (m->att_mode == GVD_ATT_INPUT_DUAL_REGION) {
            a.w1 = m->P("core.attention2_dual.alpha_net.weight"); a.b1 = m->P("core.attention2_dual.alpha_net.bias");
            a.gate_w = m->P("core.dual_pointer.0.weight"); a.gate_b = m->P("core.dual_pointer.0.bias"); a.gate_h = h_att_nxt; a.gate_ld = H;
        }
        a.w2 = m->P("core.attention2.alpha_net.weight"); a.b2 = m->P("core.attention2.alpha_net.bias");
        a.att_mask = att_mask; a.out_mask = out_mask; a.z_out = z_out; a.z_stride_b = z_stride_b;
        a.partial = w.partial; a.B = B; a.R = R; a.T = T; a.A = A; a.H = H; a.RC = w.RC; a.TC = w.TC; a.feat_div = div;
        a.out_mask_stride = out_mask_stride; a.mode = m->att_mode; a.form = m->region_form;   // (dp: P() of the absent alpha_net keys is NULL)
        if (w.V > 0) { a.vid = w.in_vid; a.win = w.in_sidx; a.ctx_bias = m->P("ctx2att.bias"); }   // video-level p_conv / conv
        a.ticket = w.ticket; a.x_out = w.x_lang;         // chunk partials are merged by the last CTA of each row (no combine launch)
        if (skinny) { a.x_out = w.xcat_lang; a.x_ld = 3 * H; }   // ... straight into the language LSTM's concatenated input
        if (sk16) { a.x_pk = w.xp_lang; a.x_pk_ld = 3 * H; }
        GVD_STAGE("decode.attn_partial", gvd_attn_partial(a, st));
    }
    {   // language LSTM: input cat(att + att2, h_att), featmap cat(att, h_att) (AttModel.py:144-160): x_lang as the attention kernel merged it
        LstmArgs a{};
        a.nseg = 3;
        a.seg[0] = LstmSeg{w.x_lang, H, nullptr, 0, m->P("core.lang_lstm.weight_ih"), 2 * H, H};
        a.seg[1] = LstmSeg{h_att_nxt, H, nullptr, 0, m->P("core.lang_lstm.weight_ih") + H, 2 * H, H};
        a.seg[2] = LstmSeg{h_lang_cur, H, nullptr, 0, m->P("core.lang_lstm.weight_hh"), H, H};
        a.bias1 = m->P("core.lang_lstm.bias_ih"); a.bias2 = m->P("core.lang_lstm.bias_hh");
        a.c_prev = w.c_lang; a.c_out = w.c_lang; a.h_out = h_lang_nxt; a.B = B; a.H = H;
        if (skinny) {
            const int S = gvd_skinny_splits(4 * H, 3 * H, B);
            const float* Wp; long long ldwp;
            if (sk16 && gvd_packed_lookup(m->w_lang_cat, 3 * H, 4 * H, 3 * H, &Wp, &ldwp)) {
                GVD_STAGE("decode.lstm_lang", gvd_skinny_f16(Wp, ldwp, 4 * H, w.xp_lang, 3 * H, B, 3 * H, S, w.sk_part, 4 * H, st));
            } else {
                GVD_REQUIRE(!sk16, "core_step: packed language-LSTM weights missing");
                GVD_STAGE("decode.lstm_lang", gvd_skinny_splitk(m->w_lang_cat, 4 * H, 3 * H, w.xcat_lang, 3 * H, B, S, w.sk_part, 4 * H, st));
            }
            GVD_STAGE("decode.lstm_lang_reduce", gvd_reduce_lstm(w.sk_part, S, 4 * H, nullptr, 0, a.bias1, a.bias2, a.c_prev, a.c_out, a.h_out, H,
                                                                 w.xcat_lang + 2 * H, 3 * H, nullptr, 0, B, H, st, sk16 ? w.xp_lang + 2 * H : nullptr, 3 * H,
                                                                 nullptr, 0));
        } else if (tc) GVD_STAGE("decode.lstm_lang", gvd_lstm_step_tc(a, st));
        else GVD_STAGE("decode.lstm_lang", gvd_lstm_step(a, st));
    }
    return 0;
}

extern "C" GVD_API int gvd_decode_step_fwd(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, int step,
                                   const int64_t* tokens, const uint8_t* att_mask, const uint8_t* out_mask, float* att2_logits_out,
                                   int64_t att2_stride_b, float* h_lang_out, void* stream) {
    GVD_TRY(require_topdown(m, "decode_step"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w));
    GVD_REQUIRE(tokens && att_mask && out_mask && att2_logits_out && step >= 0, "decode_step: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    GVD_TRY(core_step(m, w, B, T, step, (const long long*)tokens, att_mask, out_mask, att2_logits_out, att2_stride_b, st));
    if (h_lang_out) {
        const size_t BH = (size_t)B * m->d.rnn_size;
        GVD_CHECK_CUDA(cudaMemcpyAsync(h_lang_out, w.h_lang + (size_t)((step + 1) & 1) * BH, BH * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

// S1: the 21-iteration decode loop (model.py:579-624) enqueued on `st`; every pointer is fixed for a given workspace, so the
// whole enqueue is capturable as a CUDA graph.  sample == nullptr: greedy (top-2 + UNK rule, sample_max = 1); otherwise multinomial
// sampling (sample_max = 0) with the seed and temperature the kernels read from the parameter block `sample`.
// div > 1 (gvd_decode_sample_n): B = clips x div decode rows in the sampled-rows layout, rows [k*div, (k+1)*div) of clip k.
static int decode_greedy_enqueue(gvd_model_t* m, const WS& w, int B, int T, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                                 int64_t* seq_out, float* logprobs_out, float* att2_logits_out, cudaStream_t st,
                                 const GvdSampleParams* sample = nullptr, int div = 1) {
    GvdF16Scope f16;
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, V = d.vocab_size, L = d.seq_length, R = m->R;
    if (div > 1) GVD_TRY(reset_state(m, w, B / div, st));
    else GVD_TRY(gvd_decode_reset_state(m, B, T, workspace, workspace_bytes, (void*)st));
    GVD_CHECK_CUDA(cudaMemsetAsync(w.it, 0, (size_t)B * sizeof(long long), st));            // <bos> = 0 (model.py:587-588)
    // The pick kernel also writes the next step's xt = ReLU(embed[token]) (no separate embedding launch).  Folding the whole
    // sampler into the vocabulary-head GEMM epilogue (MODE_PICK of wg_gemm_kernel, last-CTA merge of the per-CTA partials) is
    // implemented and compared with the two other samplers and an fp64 reference in tests/test_gpu_decode_ops.py (through
    // gvd_op_logit_pick_tc); its merge is a serial chain on one CTA, so the loop only uses it when GVD_FUSED_PICK is set.
    const bool tc = gvd_backend_on(BK_TC) && H % 8 == 0;
    static const bool fused_pick = getenv("GVD_FUSED_PICK") != nullptr;
    const bool fused = tc && fused_pick && B <= 128 && !sample;     // the fused head has no multinomial sampler: sampling takes the split-K path
    for (int t = 0; t < L; ++t) {
        GVD_TRY(core_step(m, w, B, T, t, w.it, pnt_mask, pnt_mask, att2_logits_out + (size_t)t * R, (long long)L * R, st, div, 0, tc && t > 0));
        const float* h = w.h_lang + (size_t)((t + 1) & 1) * B * H;
        if (fused) {
            GVD_STAGE("decode.logit_pick", gvd_logit_pick_tc(h, H, m->P("logit.weight"), H, m->P("logit.bias"), B, V, H, d.unk_idx, w.pk_part,
                                                             w.pk_ticket, w.it, (long long*)seq_out + t, logprobs_out ? logprobs_out + t : nullptr, L,
                                                             m->P("embed.0.weight"), w.xt, d.input_encoding_size, st));
        } else {
            const int E = d.input_encoding_size;
            const int S = (tc && gvd_backend_on(BK_SPLITK) && w.sk_part) ? gvd_skinny_splits(V, H, B) : 0;
            const bool sk_core = core_skinny(m, w, B, div);                     // then xt goes into the core step's concatenated input
            const bool sk16 = sk_core && core_skinny_f16(m);                    // ... and its fp16x3 image into xp_att
            // above 6144 words (reduce_pick / reduce_sample hold a row in one CTA's registers): the sliced tail, one CTA per (row, 1024 words)
            auto vocab_tail = [&](const float* part, int nplanes, const float* bias, float* xt, float* xt_pk) {
                VocabTailArgs a{};
                a.part = part; a.S = nplanes; a.plane = (long long)B * m->Vp; a.ldp = m->Vp; a.bias = bias; a.B = B; a.V = V;
                a.mode = sample ? VOCAB_SAMPLE : VOCAB_GREEDY; a.unk_idx = d.unk_idx; a.par = sample; a.step = t;
                a.it_out = w.it; a.seq_out = (long long*)seq_out + t; a.logp_out = logprobs_out ? logprobs_out + t : nullptr; a.out_stride = L;
                a.embed = xt ? m->P("embed.0.weight") : nullptr; a.xt = xt; a.ld_xt = sk_core ? E + H : E; a.E = E; a.xt_pk = xt_pk; a.ld_xt_pk = E + H;
                a.rec = w.vt_rec; a.ticket = w.vt_ticket;
                return gvd_vocab_tail(a, st);
            };
            if (S > 0) {
                // vocabulary head: split-K partials, then ONE kernel sums them, adds the bias and samples (no [B,V] logits round trip)
                const float* Wp; long long ldwp;
                if (sk16 && gvd_packed_lookup(m->P("logit.weight"), H, V, H, &Wp, &ldwp)) {
                    GVD_STAGE("decode.logit", gvd_skinny_f16(Wp, ldwp, V, w.xp_lang + 2 * H, 3 * H, B, H, S, w.sk_part, m->Vp, st));     // X = h_lang(t) inside xp_lang
                } else {
                    GVD_REQUIRE(!sk16, "decode: packed vocabulary-head weights missing");
                    GVD_STAGE("decode.logit", gvd_skinny_splitk(m->P("logit.weight"), V, H, h, H, B, S, w.sk_part, m->Vp, st));
                }
                if (V > 6144) {
                    GVD_STAGE(sample ? "decode.sample" : "decode.pick", vocab_tail(w.sk_part, S, m->P("logit.bias"), sk_core ? w.xcat_att : w.xt,
                                                                                   sk16 ? w.xp_att : nullptr));
                } else if (sample) {
                    GVD_STAGE("decode.sample", gvd_reduce_sample(w.sk_part, S, m->Vp, m->P("logit.bias"), B, V, sample, t, w.it, (long long*)seq_out + t,
                                                                 logprobs_out ? logprobs_out + t : nullptr, L, m->P("embed.0.weight"),
                                                                 sk_core ? w.xcat_att : w.xt, sk_core ? E + H : E, E, st, sk16 ? w.xp_att : nullptr, E + H));
                } else {
                    GVD_STAGE("decode.pick", gvd_reduce_pick(w.sk_part, S, m->Vp, m->P("logit.bias"), B, V, d.unk_idx, w.it, (long long*)seq_out + t,
                                                             logprobs_out ? logprobs_out + t : nullptr, L, m->P("embed.0.weight"), sk_core ? w.xcat_att : w.xt,
                                                             sk_core ? E + H : E, E, nullptr, 0, st, sk16 ? w.xp_att : nullptr, E + H));
                }
            } else {
                GVD_STAGE("decode.logit", gvd_linear(h, H, m->P("logit.weight"), H, m->P("logit.bias"), w.logits, m->Vp, B, V, H, GVD_ACT_NONE, st));
                if (V > 6144) {   // (the sliced tail also writes the image of xt, which the next step's products read)
                    GVD_STAGE(sample ? "decode.sample" : "decode.pick", vocab_tail(w.logits, 1, nullptr, tc ? (sk_core ? w.xcat_att : w.xt) : nullptr,
                                                                                   tc && sk16 ? w.xp_att : nullptr));
                } else if (sample) {   // the logits already hold the bias: one plane, no bias
                    GVD_STAGE("decode.sample", gvd_reduce_sample(w.logits, 1, m->Vp, nullptr, B, V, sample, t, w.it, (long long*)seq_out + t,
                                                                 logprobs_out ? logprobs_out + t : nullptr, L, tc ? m->P("embed.0.weight") : nullptr,
                                                                 tc ? (sk_core ? w.xcat_att : w.xt) : nullptr, sk_core ? E + H : E, E, st));
                } else {
                    GVD_STAGE("decode.pick", gvd_greedy_pick(w.logits, m->Vp, B, V, d.unk_idx, w.it, (long long*)seq_out + t, logprobs_out ? logprobs_out + t : nullptr,
                                                             L, tc ? m->P("embed.0.weight") : nullptr, tc ? (sk_core ? w.xcat_att : w.xt) : nullptr, E, st, sk_core ? E + H : E));
                }
            }
        }
    }
    return 0;
}

// The decode loop through its captured graph: built on the first call for (B, T, backend, workspace) and replayed afterwards.
static int decode_loop_run(gvd_model_t* m, const WS& w, int B, int T, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                           int64_t* seq_out, float* logprobs_out, float* att2_logits_out, cudaStream_t st, const GvdSampleParams* sample,
                           cudaGraphExec_t& exec, LoopKey& key, long long& nodes, int div = 1) {
    const int L = m->d.seq_length, R = m->R;
    // Direct enqueue when the stage profiler is on (its events cannot be captured) or when asked (GVD_NO_GRAPH: per-kernel profiling)
    static const bool no_graph = getenv("GVD_NO_GRAPH") != nullptr;
    if (no_graph || g_prof_on.load(std::memory_order_relaxed) != 0)
        return decode_greedy_enqueue(m, w, B, T, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_logits_out, st, sample, div);
    // Graph path: the loop reads the mask from / writes its results to workspace-resident buffers (fixed addresses), the caller's
    // tensors are copied in / out around the replay.
    if (!exec || key.B != B || key.T != T || key.backend != gvd_backend() || key.ws != workspace || key.ws_bytes != workspace_bytes || key.V != w.V ||
        key.div != div) {
        if (exec) { cudaGraphExecDestroy(exec); exec = nullptr; }
        if (!m->capture_stream) GVD_CHECK_CUDA(cudaStreamCreateWithFlags(&m->capture_stream, cudaStreamNonBlocking));
        cudaGraph_t graph = nullptr;
        GVD_CHECK_CUDA(cudaStreamBeginCapture(m->capture_stream, cudaStreamCaptureModeThreadLocal));
        const long long l0 = g_launches.load();
        const int rc = decode_greedy_enqueue(m, w, B, T, workspace, workspace_bytes, w.in_mask, (int64_t*)w.out_seq, w.out_logp, w.out_att2,
                                             m->capture_stream, sample, div);
        const cudaError_t ce = cudaStreamEndCapture(m->capture_stream, &graph);
        nodes = g_launches.load() - l0;
        g_launches.store(l0);                              // capturing launches nothing
        if (rc != 0) { if (graph) cudaGraphDestroy(graph); return rc; }
        GVD_CHECK_CUDA(ce);
        const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        GVD_CHECK_CUDA(ie);
        key = {B, T, gvd_backend(), workspace, workspace_bytes, w.V, div};
    }
    if (pnt_mask != w.in_mask) GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_mask, pnt_mask, (size_t)(B / div) * (R + 1), cudaMemcpyDeviceToDevice, st));
    GVD_CHECK_CUDA(cudaGraphLaunch(exec, st));
    g_launches.fetch_add(nodes, std::memory_order_relaxed);
    if (seq_out != (int64_t*)w.out_seq) GVD_CHECK_CUDA(cudaMemcpyAsync(seq_out, w.out_seq, (size_t)B * L * 8, cudaMemcpyDeviceToDevice, st));
    if (logprobs_out && logprobs_out != w.out_logp) GVD_CHECK_CUDA(cudaMemcpyAsync(logprobs_out, w.out_logp, (size_t)B * L * 4, cudaMemcpyDeviceToDevice, st));
    if (att2_logits_out != w.out_att2) GVD_CHECK_CUDA(cudaMemcpyAsync(att2_logits_out, w.out_att2, (size_t)B * L * R * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
}

extern "C" GVD_API int gvd_decode_greedy(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                                 int64_t* seq_out, float* logprobs_out, float* att2_logits_out, void* stream) {
    GVD_TRY(require_topdown(m, "decode_greedy"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w));
    GVD_REQUIRE(pnt_mask && seq_out && att2_logits_out, "decode_greedy: null argument");
    return decode_loop_run(m, w, B, T, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_logits_out, (cudaStream_t)stream, nullptr,
                           m->greedy_exec, m->greedy_key, m->greedy_nodes);
}

extern "C" GVD_API int gvd_decode_sample(gvd_model_t* m, int B, int T, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                                 uint64_t seed, float temperature, int64_t* seq_out, float* logprobs_out, float* att2_logits_out, void* stream) {
    GVD_TRY(require_topdown(m, "decode_sample"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w));
    GVD_REQUIRE(pnt_mask && seq_out && att2_logits_out, "decode_sample: null argument");
    GVD_REQUIRE(std::isfinite(temperature) && temperature > 0.f, "decode_sample: temperature must be finite and > 0 (got %g)", (double)temperature);
    cudaStream_t st = (cudaStream_t)stream;
    // the parameter block is copied in on the caller's stream ahead of the loop (pageable source: staged before this call returns)
    const GvdSampleParams par{(uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32), temperature, 0u};
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.sample_par, &par, sizeof(par), cudaMemcpyHostToDevice, st));
    return decode_loop_run(m, w, B, T, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_logits_out, st, w.sample_par,
                           m->sample_exec, m->sample_key, m->sample_nodes);
}

extern "C" GVD_API int gvd_decode_sample_n(gvd_model_t* m, int B, int T, int n, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                                           uint64_t seed, float temperature, int64_t* seq_out, float* logprobs_out, float* att2_logits_out,
                                           void* stream) {
    GVD_REQUIRE(n >= 1, "decode_sample_n: n must be >= 1 (got %d)", n);
    if (n == 1)
        return gvd_decode_sample(m, B, T, workspace, workspace_bytes, pnt_mask, seed, temperature, seq_out, logprobs_out, att2_logits_out, stream);
    GVD_TRY(require_topdown(m, "decode_sample_n"));
    GVD_REQUIRE(B <= INT_MAX / n, "decode_sample_n: B * n overflows");
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w, n, 0, -1, false, true));
    GVD_REQUIRE(pnt_mask && seq_out && att2_logits_out, "decode_sample_n: null argument");
    GVD_REQUIRE(std::isfinite(temperature) && temperature > 0.f, "decode_sample_n: temperature must be finite and > 0 (got %g)", (double)temperature);
    cudaStream_t st = (cudaStream_t)stream;
    const GvdSampleParams par{(uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32), temperature, 0u};
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.sample_par, &par, sizeof(par), cudaMemcpyHostToDevice, st));
    return decode_loop_run(m, w, B * n, T, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_logits_out, st, w.sample_par,
                           m->sample_n_exec, m->sample_n_key, m->sample_n_nodes, n);
}

namespace {
__global__ void copy_token_column_kernel(const long long* seq, long long* out, int B, int L1, int i) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) out[b] = seq[(long long)b * L1 + i];
}
}  // namespace

// T1-T6 / G1: teacher-forced forward (misc/model.py:283-489), eval-mode arithmetic.  mode 0 = 'MLE' (four losses),
// mode 1 = 'GRD' (per-frame argmax of attention and grounding logits + region-class predictions).
extern "C" GVD_API int gvd_teacher_fwd(gvd_model_t* m, int B, int T, int nbox, int S, int mode, void* workspace, size_t workspace_bytes,
                                       const int64_t* seq, const int64_t* input_cls, const float* ppls, const float* gt_boxes,
                                       const uint8_t* mask_boxes, const uint8_t* frm_mask, const uint8_t* pnt_mask, float* losses_out,
                                       int64_t* att_idx_out, int64_t* grd_idx_out, int32_t* sim_target_out, int32_t* cls_pred_out, void* stream) {
    GVD_TRY(require_topdown(m, "teacher_fwd"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w, 1, nbox));
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, V = d.vocab_size, L = d.seq_length, R = m->R, L1 = L + 1;
    GVD_REQUIRE(seq && input_cls && ppls && gt_boxes && frm_mask && pnt_mask, "teacher_fwd: null input");
    GVD_REQUIRE(S >= 1 && S <= L && nbox >= 1, "teacher_fwd: need 1 <= S <= seq_length and nbox >= 1 (S=%d nbox=%d)", S, nbox);
    GVD_REQUIRE(mode == 1 || (mask_boxes && losses_out), "teacher_fwd: MLE needs mask_boxes and losses_out");
    GVD_REQUIRE(mode == 0 || (att_idx_out && grd_idx_out), "teacher_fwd: GRD needs the index outputs");
    cudaStream_t st = (cudaStream_t)stream;
    // IoU of every proposal with every GT box, frame + proposal masks applied (model.py:317-318)
    GVD_STAGE("teacher.iou", gvd_bbox_overlaps(ppls, gt_boxes, frm_mask, pnt_mask, w.ov, B, R, nbox, st));
    GVD_STAGE("teacher.cls", gvd_cls_target(w.ov, gt_boxes, w.simT, w.target, w.part_sum, w.part_cnt, B, R, nbox, m->NC, m->NCp, st));
    if (mode == 0) {
        GVD_STAGE("teacher.reduce", gvd_finish_mean(w.part_sum, w.part_cnt, B * nbox, -1.f, losses_out + 3, st));     // cls_loss (model.py:348-350)
        GVD_STAGE("teacher.targets", gvd_step_targets(w.ov, mask_boxes, frm_mask, pnt_mask, w.labels, w.fm, B, S, R, nbox, L1, st));
    } else {
        if (sim_target_out) GVD_CHECK_CUDA(cudaMemcpyAsync(sim_target_out, w.target, (size_t)B * nbox * R * 4, cudaMemcpyDeviceToDevice, st));
        if (cls_pred_out) GVD_STAGE("teacher.cls", gvd_class_argmax(w.simT, (int*)cls_pred_out, (long long)B * R, m->NC, m->NCp, st));
    }
    // teacher-forced loop: step i feeds seq[:, i] (model.py:421-453); S is the reference's early-exit count
    GVD_TRY(gvd_decode_reset_state(m, B, T, workspace, workspace_bytes, stream));
    for (int i = 0; i < S; ++i) {
        copy_token_column_kernel<<<gvd_cdiv(B, 128), 128, 0, st>>>((const long long*)seq, w.tok_col, B, L1, i);
        GVD_CHECK_LAUNCH();
        // MLE: softmax mask = proposal mask, returned logits additionally masked with the step's frame mask (model.py:441-443);
        // GRD: both are the proposal mask (model.py:446-448)
        const unsigned char* out_mask = mode == 0 ? w.fm + (size_t)i * (R + 1) : pnt_mask;
        const long long out_stride = mode == 0 ? (long long)S * (R + 1) : (long long)(R + 1);
        GVD_TRY(core_step(m, w, B, T, i, w.tok_col, pnt_mask, out_mask, w.z_all + (size_t)i * R, (long long)S * R, st, 1, out_stride));
        const float* h = w.h_lang + (size_t)((i + 1) & 1) * B * H;
        GVD_CHECK_CUDA(cudaMemcpy2DAsync(w.outs + (size_t)i * H, (size_t)S * H * 4, h, (size_t)H * 4, (size_t)H * 4, B, cudaMemcpyDeviceToDevice, st));
    }
    // grounding logits: ReLU(vis_embed)[cls] . g_pool^T + bias[cls] + att2 logits, masked (model.py:469-486); no bias term in transfer_mode
    // 'none' (P() is NULL)
    GVD_STAGE("teacher.ground", gvd_gather_class_rows(m->vis_relu, (const long long*)input_cls, w.emb, w.cls_idx, B, S, L1, V, 2048, m->NC, st));
    {
        GemmArgs g{};
        g.A = w.emb; g.lda = 2048; g.sAb = (long long)S * 2048;
        g.W = w.g_pool; g.ldw = 2048; g.sWb = (long long)R * 2048;
        g.C = w.G; g.ldc = R; g.sCb = (long long)S * R;
        g.M = S; g.N = R; g.K = 2048; g.nh = 1; g.alpha = 1.f;
        GVD_STAGE("teacher.ground", gvd_gemm_nt(g, B, st));
    }
    if (mode == 0) {
        GVD_STAGE("teacher.ground", gvd_grounding_finish(w.G, w.z_all, m->P("vis_classifiers_bias"), w.cls_idx, w.fm, R + 1, 1, B, S, R, st));
        // batched vocabulary head over all (clip, step) rows + LM loss (model.py:464-465, utils.py:122-136)
        GVD_STAGE("teacher.logit", gvd_linear(w.outs, H, m->P("logit.weight"), H, m->P("logit.bias"), w.logits_all, m->Vp, B * S, V, H, GVD_ACT_NONE, st));
        GVD_STAGE("teacher.loss", gvd_lm_nll(w.logits_all, m->Vp, (const long long*)seq, B, S, L1, V, w.part_sum, w.part_cnt, st));
        GVD_STAGE("teacher.reduce", gvd_finish_mean(w.part_sum, w.part_cnt, B * S, 1.f, losses_out + 0, st));
        GVD_STAGE("teacher.loss", gvd_att_nll(w.z_all, w.labels, (long long)B * S, R, w.part_sum, w.part_cnt, st));       // utils.py:139
        GVD_STAGE("teacher.reduce", gvd_finish_mean(w.part_sum, w.part_cnt, B * S, -1.f, losses_out + 1, st));
        GVD_STAGE("teacher.loss", gvd_att_nll(w.G, w.labels, (long long)B * S, R, w.part_sum, w.part_cnt, st));           // utils.py:142
        GVD_STAGE("teacher.reduce", gvd_finish_mean(w.part_sum, w.part_cnt, B * S, -1.f, losses_out + 2, st));
    } else {
        GVD_STAGE("teacher.ground", gvd_grounding_finish(w.G, w.z_all, m->P("vis_classifiers_bias"), w.cls_idx, pnt_mask, R + 1, 0, B, S, R, st));
        GVD_STAGE("teacher.argmax", gvd_frame_argmax(w.z_all, (long long*)att_idx_out, (long long)B * S, d.num_sampled_frm, d.num_prop_per_frm, st));
        GVD_STAGE("teacher.argmax", gvd_frame_argmax(w.G, (long long*)grd_idx_out, (long long)B * S, d.num_sampled_frm, d.num_prop_per_frm, st));
    }
    return 0;
}

// The bookkeeping of the beam search around the model, shared by gvd_beam_decode and its scripted test hook (gvd_op_beam_search_scripted):
//   bookkeeping init (<bos> tokens 0, beam_seq 0, att2 indices -1, sums 0); scores(0) = the <bos> step's region scores, row_argmax;
//   then for t = 0 .. L-1: logits(t), beam_topk, beam_update and, but at the last step (the reference runs one more, unused, core step),
//   the recurrent rows of state(t) reordered to the surviving beams (CaptionModelBU.py:85-89), scores(t + 1), row_argmax; finally beam_finish.
// scores(t) runs model step t on bb.tokens and returns its region scores [B*K, R]; logits(t, &ld) returns step t's logits [B*K, V] (pitch
// ld); state(t, bufs) fills at most 4 recurrent [B*K, H] buffers and returns their number.  bb.parent_hist / bb.done_step (optional) keep
// every step's parents and the finishing step.  att2_out (optional, needs both): the region scores of the returned caption [B, L, R]
// gathered along its ancestor chain by beam_backtrack; scores(t) must then have left step t's scores at z_hist + t * B*K*R.
template <class Scores, class Logits, class State>
static int beam_search_run(const BeamBufs& bb, int* bos_att, float* gather_tmp, int B, int K, int L, int V, int R, int H, int64_t* seq_out,
                           float* lp_out, int64_t* att_out, const float* z_hist, float* att2_out, cudaStream_t st, Scores scores, Logits logits,
                           State state) {
    const int BK = B * K;
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.tokens, 0, (size_t)BK * 8, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.seq, 0, (size_t)B * L * K * 4, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.lp, 0, (size_t)B * L * K * 4, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.att, 0xFF, (size_t)B * L * K * 4, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.att_ind, 0xFF, (size_t)BK * 4, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.sums, 0, (size_t)B * K * 4, st));
    GVD_CHECK_CUDA(cudaMemsetAsync(bb.done_flag, 0, (size_t)B * 4, st));
    const float* z = nullptr;
    GVD_TRY(scores(0, &z));
    GVD_STAGE("beam.argmax", gvd_row_argmax(z, R, BK, R, bos_att, st));
    for (int t = 0; t < L; ++t) {
        const float* lg = nullptr;
        long long ld = 0;
        GVD_TRY(logits(t, &lg, &ld));
        GVD_STAGE("beam.topk", gvd_beam_topk(lg, ld, BK, V, K, bb.topv, bb.topi, st));
        GVD_STAGE("beam.update", gvd_beam_update(bb, B, K, L, t, st));
        if (t == L - 1) break;
        float* bufs[4];
        const int n = state(t, bufs);
        for (int i = 0; i < n; ++i) {
            GVD_STAGE("beam.gather", gvd_beam_gather_rows(bufs[i], gather_tmp, bb.parent, B, K, H, st));
            GVD_CHECK_CUDA(cudaMemcpyAsync(bufs[i], gather_tmp, (size_t)BK * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
        GVD_TRY(scores(t + 1, &z));
        GVD_STAGE("beam.argmax", gvd_row_argmax(z, R, BK, R, bb.att_ind, st));
    }
    GVD_STAGE("beam.finish", gvd_beam_finish(bb, bos_att, B, K, L, (long long*)seq_out, lp_out, (long long*)att_out, st));
    if (att2_out) GVD_STAGE("beam.backtrack", gvd_beam_backtrack(bb, z_hist, (long long)BK * R, B, K, L, R, att2_out, st));
    return 0;
}

// B1/B2: beam search for every clip at once (misc/model.py:700-742 + misc/CaptionModelBU.py:104-185, repaired semantics).  att2_logits_out
// (gvd_beam_decode_att2): each step's region scores land in the workspace's history instead of z_rows, and the returned caption's rows are
// gathered from it at the end.
static int beam_decode(gvd_model_t* m, int B, int T, int beam_size, void* workspace, size_t workspace_bytes, const uint8_t* pnt_mask,
                       int64_t* seq_out, float* logprobs_out, int64_t* att2_idx_out, float* att2_logits_out, void* stream) {
    GVD_TRY(require_topdown(m, "beam_decode"));
    GVD_REQUIRE(beam_size >= 2, "beam_decode: beam_size must be >= 2 (use gvd_decode_greedy for 1)");
    WS w;
    const bool hist = att2_logits_out != nullptr;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w, beam_size, 0, -1, hist));
    GVD_REQUIRE(pnt_mask && seq_out && logprobs_out && att2_idx_out, "beam_decode: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const gvd_dims_t& d = m->d;
    const int H = d.rnn_size, V = d.vocab_size, L = d.seq_length, R = m->R, K = beam_size, BK = B * K;
    const size_t BKH = (size_t)BK * H;
    {   // zero state and attention tickets (the bookkeeping is initialised by beam_search_run)
        const size_t n = BKH * sizeof(float);
        GVD_CHECK_CUDA(cudaMemsetAsync(w.h_att, 0, 2 * n, st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.c_att, 0, n, st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.h_lang, 0, 2 * n, st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.c_lang, 0, n, st));
        GVD_CHECK_CUDA(cudaMemsetAsync(w.ticket, 0, (size_t)BK * sizeof(int), st));
    }
    // core step t on the beam tokens; step 0 is the <bos> step (model.py:723-733), whose K rows of a clip are identical
    auto scores = [&](int t, const float** z) {
        float* zt = hist ? w.att2_hist + (size_t)t * BK * R : w.z_rows;
        *z = zt;
        return core_step(m, w, BK, T, t, w.bb.tokens, pnt_mask, pnt_mask, zt, R, st, K);
    };
    auto logits = [&](int t, const float** lg, long long* ld) {
        const float* h_lang = w.h_lang + (size_t)((t + 1) & 1) * BKH;   // state parity written by the previous core step
        *lg = w.logits;
        *ld = m->Vp;
        GVD_STAGE("decode.logit", gvd_linear(h_lang, H, m->P("logit.weight"), H, m->P("logit.bias"), w.logits, m->Vp, BK, V, H, GVD_ACT_NONE, st));
        return 0;
    };
    auto state = [&](int t, float** bufs) {
        const int par = (t + 1) & 1;
        bufs[0] = w.h_att + (size_t)par * BKH; bufs[1] = w.c_att; bufs[2] = w.h_lang + (size_t)par * BKH; bufs[3] = w.c_lang;
        return 4;
    };
    return beam_search_run(w.bb, w.bos_att, w.gather_tmp, B, K, L, V, R, H, seq_out, logprobs_out, att2_idx_out, w.att2_hist, att2_logits_out, st,
                           scores, logits, state);
}
extern "C" GVD_API int gvd_beam_decode(gvd_model_t* m, int B, int T, int beam_size, void* workspace, size_t workspace_bytes,
                                       const uint8_t* pnt_mask, int64_t* seq_out, float* logprobs_out, int64_t* att2_idx_out, void* stream) {
    return beam_decode(m, B, T, beam_size, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_idx_out, nullptr, stream);
}
extern "C" GVD_API int gvd_beam_decode_att2(gvd_model_t* m, int B, int T, int beam_size, void* workspace, size_t workspace_bytes,
                                            const uint8_t* pnt_mask, int64_t* seq_out, float* logprobs_out, int64_t* att2_idx_out,
                                            float* att2_logits_out, void* stream) {
    GVD_REQUIRE(att2_logits_out, "beam_decode_att2: null att2_logits_out");
    return beam_decode(m, B, T, beam_size, workspace, workspace_bytes, pnt_mask, seq_out, logprobs_out, att2_idx_out, att2_logits_out, stream);
}

// Clip chunks of the host-buffer entry point.  The pipeline starts with one attention sub-batch (`unit` clips: the first kernel waits for the
// first copy) and grows 1, 2, 3, 6, 9, 12, 12 ... units, so that the copy engine stays ahead of the compute stream; a short remainder joins
// the last chunk.  The growth rule has not been re-tuned for the H100.
static std::vector<int> h2d_schedule(int B, int unit) {
    std::vector<int> s;
    int left = B;
    auto push = [&](int n) { n = std::max(1, std::min(n, left)); s.push_back(n); left -= n; };
    const int grow[5] = {1, 2, 3, 6, 9};
    for (int i = 0; i < 5 && left > 0; ++i) push(left < (grow[i] + 2) * unit ? left : grow[i] * unit);
    while (left > 0) push(left < 16 * unit ? left : 12 * unit);
    return s;
}

extern "C" GVD_API int gvd_plan_h2d_chunks(int batch_clips, int unit, int* chunks_out, int cap) {
    if (!(batch_clips >= 1 && unit >= 1 && chunks_out && cap >= 1)) { gvd_set_error("plan_h2d_chunks: bad arguments"); return -1; }
    const std::vector<int> s = h2d_schedule(batch_clips, std::min(unit, batch_clips));
    if ((int)s.size() > cap) { gvd_set_error("plan_h2d_chunks: %d chunks do not fit the caller's array of %d", (int)s.size(), cap); return -1; }
    for (size_t i = 0; i < s.size(); ++i) chunks_out[i] = s[i];
    return (int)s.size();
}

// V = 0: per-clip batch; V > 0: video-indexed batch, h_segs_feat [V,T,F] (V videos' frames cross PCIe instead of B copies)
static int sample_greedy_host_run(gvd_model_t* m, int B, int V, int T, const float* h_segs_feat, const float* h_ppls, const int64_t* h_num,
                                  const float* h_ppls_feat, const int64_t* h_sample_idx, const int64_t* h_video_idx, const uint8_t* h_pnt_mask,
                                  void* workspace, size_t workspace_bytes, int64_t* h_seq_out, float* h_logprobs_out, float* h_att2_out,
                                  float* h_sim_mat_out, void* stream) {
    GVD_TRY(require_topdown(m, "sample_greedy_host"));
    WS w;
    GVD_TRY(check_ws(m, B, T, workspace, workspace_bytes, &w, 1, 0, V));
    GVD_REQUIRE(h_segs_feat && h_ppls && h_num && h_ppls_feat && h_sample_idx && h_pnt_mask && h_seq_out && (V == 0 || h_video_idx),
                "sample_greedy_host: null argument");
    for (int b = 0; b < (V > 0 ? B : 0); ++b)
        GVD_REQUIRE(h_video_idx[b] >= 0 && h_video_idx[b] < V, "sample_greedy_host: video_idx[%d] = %lld outside [0, %d)", b, (long long)h_video_idx[b], V);
    cudaStream_t st = (cudaStream_t)stream;
    const gvd_dims_t& d = m->d;
    const int R = m->R, L = d.seq_length, FC = d.fc_feat_size;
    const size_t BR = (size_t)B * R, BT = (size_t)(V > 0 ? V : B) * T;     // BT: frame rows that cross PCIe
    // The fc6 region features are ~98 % of the input bytes (819 MB at B=100) and every region stage is per-clip independent,
    // so they cross PCIe in clip chunks on a second stream while the previous chunk runs P2-P6 on the compute stream.
    const std::vector<int> sched = h2d_schedule(B, w.clip_chunk);
    const int nchunks = (int)sched.size();
    if (!m->copy_stream) GVD_CHECK_CUDA(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
    while ((int)m->events.size() < nchunks + 3) {
        cudaEvent_t e;
        GVD_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        m->events.push_back(e);
    }
    cudaEvent_t ev_start = m->events[nchunks], ev_sim = m->events[nchunks + 1], ev_segs = m->events[nchunks + 2];
    // Frame stages (P1 + P7) on their own stream next to the region stages (see frame_fork).  Long clips (reference default T = 480: 590 MB of
    // frame features, a long GRU chain): the frame features cross PCIe after the first ~30 % of the region chunks — early enough for the
    // chain to end with the region stages, late enough for those to have work while the features travel.  Without the second stream they
    // travel last and the frame stages run last.
    const bool overlap = frame_overlap_on();
    const bool big_segs = BT * (size_t)FC * 4 > ((size_t)64 << 20);
    int segs_after = 0;                                   // chunks copied before the frame features (big_segs only)
    if (big_segs) {
        segs_after = nchunks;
        if (overlap) {
            const int want = (3 * B + 9) / 10;      // clips
            int acc = 0;
            segs_after = 0;
            while (segs_after < nchunks && acc < want) acc += sched[segs_after++];
        }
    }
    GVD_CHECK_CUDA(cudaEventRecord(ev_start, st));                       // the workspace may still be in use by earlier work on `st`
    GVD_CHECK_CUDA(cudaStreamWaitEvent(m->copy_stream, ev_start, 0));
    if (!big_segs) GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_segs, h_segs_feat, BT * FC * 4, cudaMemcpyHostToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_ppls, h_ppls, BR * 7 * 4, cudaMemcpyHostToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_num, h_num, (size_t)B * 7 * 8, cudaMemcpyHostToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_sidx, h_sample_idx, (size_t)B * 2 * 8, cudaMemcpyHostToDevice, st));
    GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_mask, h_pnt_mask, (size_t)B * (R + 1), cudaMemcpyHostToDevice, st));
    if (V > 0) GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_vid, h_video_idx, (size_t)B * 8, cudaMemcpyHostToDevice, st));
    set_video(m, workspace, B, T, V);
    cudaStream_t fst = st;
    if (overlap) { GVD_TRY(frame_fork(m, st)); fst = m->frame_stream; }          // (forked behind the small copies: the frame stages read num / sample_idx)
    // the big chunk copies are enqueued AFTER the small ones: the H2D copy engine is one FIFO across streams, and the first
    // kernels on `st` need the small tensors
    auto copy_segs = [&]() -> int {
        GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_segs, h_segs_feat, BT * FC * 4, cudaMemcpyHostToDevice, m->copy_stream));
        GVD_CHECK_CUDA(cudaEventRecord(ev_segs, m->copy_stream));
        return 0;
    };
    {
        size_t c0 = 0;
        for (int c = 0; c < nchunks; ++c) {
            if (big_segs && c == segs_after) GVD_TRY(copy_segs());
            const size_t cb = (size_t)sched[c];
            GVD_CHECK_CUDA(cudaMemcpyAsync(w.in_feat + c0 * R * d.att_feat_size, h_ppls_feat + c0 * R * d.att_feat_size, cb * R * d.att_feat_size * 4,
                                           cudaMemcpyHostToDevice, m->copy_stream));
            GVD_CHECK_CUDA(cudaEventRecord(m->events[c], m->copy_stream));
            c0 += cb;
        }
        if (big_segs && segs_after >= nchunks) GVD_TRY(copy_segs());
    }
    int rc = 0;
    bool frame_done = false;
    auto run_frame = [&]() -> int {
        frame_done = true;
        if (big_segs) GVD_CHECK_CUDA(cudaStreamWaitEvent(fst, ev_segs, 0));
        return frame_stages(m, w, B, T, w.in_segs, w.in_num, w.in_sidx, fst, V > 0 ? w.in_vid : nullptr);
    };
    if (!big_segs) rc = run_frame();
    {
        int c0 = 0;
        for (int c = 0; c < nchunks && rc == 0; ++c) {
            // on one stream the frame stages go last (they would hold up the region chunks behind the frame-feature copy)
            if (big_segs && overlap && c == segs_after && !frame_done) { rc = run_frame(); if (rc) break; }
            const int cb = sched[c];
            GVD_CHECK_CUDA(cudaStreamWaitEvent(st, m->events[c], 0));
            rc = region_prologue(m, w, c0, cb, w.in_ppls + (size_t)c0 * R * 7, w.in_feat + (size_t)c0 * R * d.att_feat_size,
                                 w.in_mask + (size_t)c0 * (R + 1), h_sim_mat_out ? w.out_sim + (size_t)c0 * m->NC * R : nullptr, st);
            c0 += cb;
        }
    }
    if (rc == 0 && !frame_done) rc = run_frame();
    if (overlap) { const int jr = frame_join(m, st); if (rc == 0) rc = jr; }
    if (rc != 0) { cudaStreamSynchronize(m->copy_stream); return rc; }            // (the copies read caller memory: never return with them in flight)
    if (h_sim_mat_out) {   // the similarity matrix is final here: its D2H overlaps the 20-step decode loop
        GVD_CHECK_CUDA(cudaEventRecord(ev_sim, st));
        GVD_CHECK_CUDA(cudaStreamWaitEvent(m->copy_stream, ev_sim, 0));
        GVD_CHECK_CUDA(cudaMemcpyAsync(h_sim_mat_out, w.out_sim, (size_t)B * m->NC * R * 4, cudaMemcpyDeviceToHost, m->copy_stream));
    }
    GVD_TRY(gvd_decode_greedy(m, B, T, workspace, workspace_bytes, w.in_mask, (int64_t*)w.out_seq, w.out_logp, w.out_att2, stream));
    GVD_CHECK_CUDA(cudaMemcpyAsync(h_seq_out, w.out_seq, (size_t)B * L * 8, cudaMemcpyDeviceToHost, st));
    if (h_logprobs_out) GVD_CHECK_CUDA(cudaMemcpyAsync(h_logprobs_out, w.out_logp, (size_t)B * L * 4, cudaMemcpyDeviceToHost, st));
    if (h_att2_out) GVD_CHECK_CUDA(cudaMemcpyAsync(h_att2_out, w.out_att2, (size_t)B * L * R * 4, cudaMemcpyDeviceToHost, st));
    GVD_CHECK_CUDA(cudaStreamSynchronize(st));
    GVD_CHECK_CUDA(cudaStreamSynchronize(m->copy_stream));
    return 0;
}
extern "C" GVD_API int gvd_sample_greedy_host(gvd_model_t* m, int B, int T, const float* h_segs_feat, const float* h_ppls, const int64_t* h_num,
                                      const float* h_ppls_feat, const int64_t* h_sample_idx, const uint8_t* h_pnt_mask, void* workspace,
                                      size_t workspace_bytes, int64_t* h_seq_out, float* h_logprobs_out, float* h_att2_out,
                                      float* h_sim_mat_out, void* stream) {
    return sample_greedy_host_run(m, B, 0, T, h_segs_feat, h_ppls, h_num, h_ppls_feat, h_sample_idx, nullptr, h_pnt_mask, workspace, workspace_bytes,
                                  h_seq_out, h_logprobs_out, h_att2_out, h_sim_mat_out, stream);
}
extern "C" GVD_API int gvd_sample_greedy_host_video(gvd_model_t* m, int B, int V, int T, const float* h_segs_feat, const float* h_ppls,
                                                    const int64_t* h_num, const float* h_ppls_feat, const int64_t* h_sample_idx,
                                                    const int64_t* h_video_idx, const uint8_t* h_pnt_mask, void* workspace, size_t workspace_bytes,
                                                    int64_t* h_seq_out, float* h_logprobs_out, float* h_att2_out, float* h_sim_mat_out, void* stream) {
    GVD_REQUIRE(V >= 1, "sample_greedy_host_video: V=%d must be >= 1", V);
    return sample_greedy_host_run(m, B, V, T, h_segs_feat, h_ppls, h_num, h_ppls_feat, h_sample_idx, h_video_idx, h_pnt_mask, workspace,
                                  workspace_bytes, h_seq_out, h_logprobs_out, h_att2_out, h_sim_mat_out, stream);
}

// Post-decode grounding extraction (main.py:364-370, SURVEY 8(f) rank 2): for every generated word and every sampled frame the
// proposal with the largest region-attention logit, and its box row.  att2 [B, L, F*P] (the second output of 'sample'),
// ppls [B, F*P, 7]; idx_out [B, L, F] int64, boxes_out [B, L, F, 7] (may be null).  Ties -> lowest index (torch.max on CPU).
extern "C" GVD_API int gvd_grounding_extract(const float* att2, const float* ppls, int B, int L, int num_frames, int num_prop, int64_t* idx_out,
                                             float* boxes_out, void* stream) {
    GVD_REQUIRE(att2 && ppls && idx_out && B > 0 && L > 0 && num_frames > 0 && num_prop > 0, "grounding_extract: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    GVD_TRY(gvd_frame_argmax(att2, (long long*)idx_out, (long long)B * L, num_frames, num_prop, st));
    if (boxes_out) GVD_TRY(gvd_grounding_gather(ppls, (const long long*)idx_out, boxes_out, B, L, num_frames, num_prop, 7, st));
    return 0;
}

// Grounding-evaluator hit test (tools/anet_entities/scripts/eval_grd_anet_entities.py:95-102, SURVEY 8(f) rank 3), batched over
// words: pred [N,F,5] (x1,y1,x2,y2,frame), ref [N,K,5] with the first nref[n] rows valid -> max IoU [N] and hit [N] = max > thresh.
extern "C" GVD_API int gvd_grounding_eval(const float* pred, const float* ref, const int* nref, int N, int F, int K, float iou_thresh,
                                          float* max_iou_out, unsigned char* hit_out, void* stream) {
    GVD_REQUIRE(pred && ref && nref && max_iou_out && hit_out && N > 0 && F > 0 && K > 0, "grounding_eval: bad arguments");
    return gvd_grounding_eval_hits(pred, ref, nref, max_iou_out, hit_out, N, F, K, iou_thresh, (cudaStream_t)stream);
}

// K-split plan of the operand-swapped skinny products (host logic only, no device access): number of splits, 0 = shape not supported
extern "C" GVD_API int gvd_plan_skinny_splits(int weight_rows, int k_total, int batch_rows) { return gvd_skinny_splits(weight_rows, k_total, batch_rows); }

// ------------------------------------------------------------------------------------ single ops
extern "C" GVD_API int gvd_op_linear(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc, int M,
                             int N, int K, int act, void* stream) {
    GVD_REQUIRE(A && W && C, "op_linear: null argument");
    return gvd_linear(A, lda, W, ldw, bias, C, ldc, M, N, K, act, (cudaStream_t)stream);
}
extern "C" GVD_API int gvd_op_linear_tc(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc,
                                        int M, int N, int K, int act, void* stream) {
    GVD_REQUIRE(A && W && C, "op_linear_tc: null argument");
    GvdF16Scope f16;                               // test hook of a forward product: backend bit 4 selects the fp16x3 variant
    GemmArgs g{};
    g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.C = C; g.ldc = ldc; g.bias = bias;
    g.M = M; g.N = N; g.K = K; g.nh = 1; g.act = act; g.alpha = 1.f;
    return gvd_gemm_nt_tc(g, 1, (cudaStream_t)stream);
}
// The conversion-free prologue GEMM (ss_gemm_kernel) on its own: both operands are packed into fp16x3 images here (scratch from the
// stream-ordered allocator), optionally with the fp16x3 image of the output (img_out [M, rup32(N)] words) next to / instead of C.
// nh > 0: the Q|K|V projection of the region encoder (N = 3 nh hs, clips of R rows, no bias / activation): Q to C[:, 0:HP), K to the
// per-head image k_img [M, nh, rup32(hs)] words, V to the image of V^T per clip vt_img [M / R, HP, rup32(R)] words.  qkv_ref: the same
// images from the fp32 product in C[M, N] followed by the pack passes of the unfused path.  Test hook.
extern "C" GVD_API int gvd_op_linear_f16ss(const float* A, int64_t lda, const float* W, int64_t ldw, const float* bias, float* C, int64_t ldc,
                                           float* img_out, int M, int N, int K, int act, int nh, int hs, int R, float* k_img, float* vt_img,
                                           int qkv_ref, void* stream) {
    GVD_REQUIRE(A && W && (C || img_out) && M > 0 && N > 0 && K > 0, "op_linear_f16ss: null argument");
    GVD_REQUIRE(nh == 0 || (nh > 0 && hs > 0 && R > 0 && M % R == 0 && N == 3 * nh * hs && k_img && vt_img && C && !img_out),
                "op_linear_f16ss: Q|K|V mode needs N = 3 nh hs, whole clips, C, k_img and vt_img");
    cudaStream_t st = (cudaStream_t)stream;
    const long long Kp = (K + 31) / 32 * 32, Np = (N + 31) / 32 * 32;
    float *Ai = nullptr, *Wi = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&Ai, (size_t)M * Kp * 4, st));
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&Wi, (size_t)N * Kp * 4, st));
    int rc = gvd_pack_f16x3(A, lda, M, K, Ai, Kp, st, GVD_F16_SA);
    if (!rc) rc = gvd_pack_f16x3(W, ldw, N, K, Wi, Kp, st, GVD_F16_SW);
    const int HP = nh * hs, KH = (hs + 31) / 32 * 32, Rp = (R + 31) / 32 * 32;
    if (!rc && nh && !qkv_ref) {
        GvdQkvImages qi{HP, hs, KH, nh, R, Rp, k_img, vt_img, GVD_ATT_SK, GVD_ATT_SV};
        rc = gvd_gemm_f16ss(Ai, Kp, Wi, Kp, bias, nullptr, nullptr, act, C, ldc, M, N, K, st, nullptr, 0, &qi);
    } else if (!rc) {
        rc = gvd_gemm_f16ss(Ai, Kp, Wi, Kp, bias, nullptr, nullptr, act, C, ldc, M, N, K, st, img_out, img_out ? Np : 0);
        if (!rc && nh) rc = gvd_pack_heads_f16x3(C + HP, ldc, M, nh, hs, hs, KH, GVD_ATT_SK, k_img, st);
        if (!rc && nh) rc = gvd_transpose_pack_f16x3(C + 2 * HP, vt_img, M / R, R, HP, (int)ldc, Rp, GVD_ATT_SV, st);
    }
    cudaFreeAsync(Ai, st);
    cudaFreeAsync(Wi, st);
    return rc;
}
// One LSTMCell step from up to two dense input segments [x0 | x1] (weights w0 [4H,K0], w1 [4H,K1]); backend 0 = CUDA cores, 1 = wgmma
extern "C" GVD_API int gvd_op_lstm_step(int B, int H, const float* x0, int K0, const float* w0, int64_t ldw0, const float* x1, int K1,
                                        const float* w1, int64_t ldw1, const float* bias1, const float* bias2, const float* c_prev,
                                        float* h_out, float* c_out, int backend, void* stream) {
    GVD_REQUIRE(x0 && w0 && c_prev && h_out && c_out, "op_lstm_step: null argument");
    GvdF16Scope f16;
    LstmArgs a{};
    a.nseg = x1 ? 2 : 1;
    a.seg[0] = LstmSeg{x0, K0, nullptr, 0, w0, ldw0, K0};
    if (x1) a.seg[1] = LstmSeg{x1, K1, nullptr, 0, w1, ldw1, K1};
    a.bias1 = bias1; a.bias2 = bias2; a.c_prev = c_prev; a.h_out = h_out; a.c_out = c_out; a.B = B; a.H = H;
    return backend ? gvd_lstm_step_tc(a, (cudaStream_t)stream) : gvd_lstm_step(a, (cudaStream_t)stream);
}
// The decode step's operand-swapped split-K product on its own: part[s][b][n] = sum over the K range of split s of W[n][k] X[b][k].
// f16_images = 0: gvd_skinny_splitk (operands split in the kernel, 3xTF32 or fp16x3 by backend bit 4); 1: both operands packed into fp16x3
// images here and multiplied by the conversion-free gvd_skinny_f16.  S = 0 takes the plan of gvd_skinny_splits.  Test hook.
extern "C" GVD_API int gvd_op_skinny_partials(const float* W, int Nw, int K, const float* X, int64_t ldx, int B, int S, int f16_images,
                                              float* part, int ldp, void* stream) {
    GVD_REQUIRE(W && X && part && Nw > 0 && K > 0 && B >= 1 && B <= 128 && S >= 0, "op_skinny_partials: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (S == 0) S = gvd_skinny_splits(Nw, K, B);
    GVD_REQUIRE(S >= 1, "op_skinny_partials: no split plan for %d x %d weights and %d rows", Nw, K, B);
    GvdF16Scope f16;
    if (!f16_images) return gvd_skinny_splitk(W, Nw, K, X, ldx, B, S, part, ldp, st);
    GVD_REQUIRE(K % 32 == 0, "op_skinny_partials: operand images need K %% 32 == 0");
    float *Wi = nullptr, *Xi = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&Wi, (size_t)Nw * K * 4, st));
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&Xi, (size_t)B * K * 4, st));
    int rc = gvd_pack_f16x3(W, K, Nw, K, Wi, K, st, GVD_F16_SW);
    if (!rc) rc = gvd_pack_f16x3(X, ldx, B, K, Xi, K, st, GVD_F16_SA);
    if (!rc) rc = gvd_skinny_f16(Wi, K, Nw, Xi, K, B, K, S, part, ldp, st);
    cudaFreeAsync(Wi, st);
    cudaFreeAsync(Xi, st);
    return rc;
}
// The three reductions of the split-K partial planes and the CUDA-core sampler with their launchers' own arguments.  Test hooks.
extern "C" GVD_API int gvd_op_reduce_lstm(const float* part, int S, int ldp, const float* pre, int pre_div, const float* bias1, const float* bias2,
                                          const float* c_prev, float* c_out, float* h0, int64_t ldh0, float* h1, int64_t ldh1, float* h2,
                                          int64_t ldh2, int B, int H, float* pk1, int64_t ldpk1, float* pk2, int64_t ldpk2, void* stream) {
    GVD_REQUIRE(part && c_prev && c_out && h0 && S >= 1 && B >= 1 && H >= 1, "op_reduce_lstm: bad arguments");
    return gvd_reduce_lstm(part, S, ldp, pre, pre_div, bias1, bias2, c_prev, c_out, h0, ldh0, h1, ldh1, h2, ldh2, B, H, (cudaStream_t)stream, pk1, ldpk1,
                           pk2, ldpk2);
}
extern "C" GVD_API int gvd_op_reduce_bias(const float* part, int S, int Nw, int ldp, const float* bias, float* out, int64_t ld_out, int B,
                                          void* stream) {
    GVD_REQUIRE(part && out && S >= 1 && B >= 1 && Nw >= 1, "op_reduce_bias: bad arguments");
    return gvd_reduce_bias(part, S, Nw, ldp, bias, out, ld_out, B, (cudaStream_t)stream);
}
extern "C" GVD_API int gvd_op_reduce_pick(const float* part, int S, int ldp, const float* bias, int B, int V, int unk_idx, int64_t* it_out,
                                          int64_t* seq_out, float* logp_out, int64_t out_stride, const float* embed, float* xt, int64_t ld_xt,
                                          int E, float* logits_out, int64_t ld_logits, float* xt_pk, int64_t ld_xt_pk, void* stream) {
    GVD_REQUIRE(part && S >= 1 && B >= 1 && (!xt || embed), "op_reduce_pick: bad arguments");
    return gvd_reduce_pick(part, S, ldp, bias, B, V, unk_idx, (long long*)it_out, (long long*)seq_out, logp_out, out_stride, embed, xt, ld_xt, E,
                           logits_out, ld_logits, (cudaStream_t)stream, xt_pk, ld_xt_pk);
}
extern "C" GVD_API int gvd_op_reduce_sample(const float* part, int S, int ldp, const float* bias, int B, int V, float temperature, uint64_t seed,
                                            int step, int64_t* it_out, int64_t* seq_out, float* logp_out, int64_t out_stride, const float* embed,
                                            float* xt, int64_t ld_xt, int E, float* xt_pk, int64_t ld_xt_pk, void* stream) {
    GVD_REQUIRE(part && S >= 1 && B >= 1 && (!xt || embed), "op_reduce_sample: bad arguments");
    GVD_REQUIRE(std::isfinite(temperature) && temperature > 0.f, "op_reduce_sample: temperature must be finite and > 0 (got %g)", (double)temperature);
    cudaStream_t st = (cudaStream_t)stream;
    const GvdSampleParams par{(uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32), temperature, 0u};
    GvdSampleParams* dpar = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&dpar, sizeof(par), st));
    int rc = 0;
    if (cudaMemcpyAsync(dpar, &par, sizeof(par), cudaMemcpyHostToDevice, st) != cudaSuccess) { gvd_set_error("op_reduce_sample: copy failed"); rc = 2; }
    if (!rc) rc = gvd_reduce_sample(part, S, ldp, bias, B, V, dpar, step, (long long*)it_out, (long long*)seq_out, logp_out, out_stride, embed, xt, ld_xt,
                                    E, st, xt_pk, ld_xt_pk);
    cudaFreeAsync(dpar, st);
    return rc;
}
static_assert(VOCAB_GREEDY == GVD_VOCAB_GREEDY && VOCAB_SAMPLE == GVD_VOCAB_SAMPLE && VOCAB_ARGMAX == GVD_VOCAB_ARGMAX, "vocabulary tail modes");
extern "C" GVD_API int gvd_op_reduce_pick_split(const float* part, int S, int ldp, const float* bias, int B, int V, int mode, int unk_idx,
                                                float temperature, uint64_t seed, int step, int64_t* it_out, int64_t* seq_out, float* logp_out,
                                                int64_t out_stride, const float* embed, float* xt, int64_t ld_xt, int E, float* logits_out,
                                                int64_t ld_logits, float* xt_pk, int64_t ld_xt_pk, void* stream) {
    GVD_REQUIRE(part && S >= 1 && B >= 1 && V >= 2 && it_out && (!xt || embed), "op_reduce_pick_split: bad arguments");
    GVD_REQUIRE(mode != GVD_VOCAB_SAMPLE || (std::isfinite(temperature) && temperature > 0.f),
                "op_reduce_pick_split: temperature must be finite and > 0 (got %g)", (double)temperature);
    cudaStream_t st = (cudaStream_t)stream;
    // records | tickets | sampler parameter block, in one allocation
    const size_t rec_bytes = gvd_vocab_rec_floats(B, V) * 4, tk_bytes = ((size_t)B * 4 + 15) / 16 * 16;
    char* buf = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&buf, rec_bytes + tk_bytes + sizeof(GvdSampleParams), st));
    const GvdSampleParams par{(uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32), temperature, 0u};
    VocabTailArgs a{};
    a.part = part; a.S = S; a.plane = (long long)B * ldp; a.ldp = ldp; a.bias = bias; a.B = B; a.V = V;
    a.mode = mode; a.unk_idx = unk_idx; a.par = reinterpret_cast<GvdSampleParams*>(buf + rec_bytes + tk_bytes); a.step = step;
    a.it_out = (long long*)it_out; a.seq_out = (long long*)seq_out; a.logp_out = logp_out; a.out_stride = out_stride;
    a.embed = embed; a.xt = xt; a.ld_xt = ld_xt; a.E = E; a.xt_pk = xt_pk; a.ld_xt_pk = ld_xt_pk; a.logits_out = logits_out; a.ld_logits = ld_logits;
    a.rec = reinterpret_cast<float*>(buf); a.ticket = reinterpret_cast<int*>(buf + rec_bytes);
    int rc = 0;
    if (cudaMemsetAsync(a.ticket, 0, tk_bytes, st) != cudaSuccess ||
        cudaMemcpyAsync(buf + rec_bytes + tk_bytes, &par, sizeof(par), cudaMemcpyHostToDevice, st) != cudaSuccess) {
        gvd_set_error("op_reduce_pick_split: staging failed");
        rc = 2;
    }
    if (!rc) rc = gvd_vocab_tail(a, st);
    cudaFreeAsync(buf, st);
    return rc;
}
extern "C" GVD_API int gvd_op_greedy_pick(const float* logits, int64_t ld, int B, int V, int unk_idx, int64_t* it_out, int64_t* seq_out,
                                          float* logp_out, int64_t out_stride, const float* embed, float* xt, int64_t ld_xt, int E, void* stream) {
    GVD_REQUIRE(logits && it_out && B >= 1 && (!xt || embed), "op_greedy_pick: bad arguments");
    return gvd_greedy_pick(logits, ld, B, V, unk_idx, (long long*)it_out, (long long*)seq_out, logp_out, out_stride, embed, xt, E,
                           (cudaStream_t)stream, ld_xt);
}
// Vocabulary head with the sampler in the GEMM epilogue (MODE_PICK of wg_gemm_kernel): the per-CTA partials and the zeroed ticket are
// allocated here.  Test hook.
extern "C" GVD_API int gvd_op_logit_pick_tc(const float* h, int64_t ldh, const float* W, int64_t ldw, const float* bias, int B, int V, int K,
                                            int unk_idx, const float* embed, int E, int64_t* it_out, int64_t* seq_out, float* logp_out,
                                            int64_t out_stride, float* xt, void* stream) {
    GVD_REQUIRE(h && W && bias && it_out && B >= 1 && V >= 2 && K > 0 && (!xt || embed), "op_logit_pick_tc: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    GvdF16Scope f16;
    const size_t part_bytes = (size_t)gvd_cdiv(V, 64) * B * 8 * sizeof(float);
    float* part = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&part, part_bytes + 16, st));
    int* ticket = reinterpret_cast<int*>(reinterpret_cast<char*>(part) + part_bytes);
    int rc = 0;
    if (cudaMemsetAsync(part, 0, part_bytes + 16, st) != cudaSuccess) { gvd_set_error("op_logit_pick_tc: memset failed"); rc = 2; }
    if (!rc) rc = gvd_logit_pick_tc(h, ldh, W, ldw, bias, B, V, K, unk_idx, part, ticket, (long long*)it_out, (long long*)seq_out, logp_out, out_stride,
                                    embed, xt, E, st);
    cudaFreeAsync(part, st);
    return rc;
}
// One bidirectional GRU layer (model.py:150-154) from given input projections gi [B,T,6G]: path 1 = the tensor-core layer (W_hh packed
// into its fp16x3 image here), path 0 = the per-step GEMM + pointwise loop (gvd_gemm_nt follows the backend switch).  Test hook.
extern "C" GVD_API int gvd_op_gru_layer(int path, const float* gi, const float* Whh, const float* bhh, const int64_t* sample_idx, int B, int T,
                                        int G, float* out, void* stream) {
    GVD_REQUIRE(gi && Whh && bhh && out && B >= 1 && T >= 1 && G >= 4 && G % 4 == 0 && (path == 0 || path == 1), "op_gru_layer: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    GvdF16Scope f16;
    const size_t state = (size_t)2 * 2 * B * G, nw = (size_t)6 * G * G, ngh = (size_t)2 * B * 3 * G;
    float* buf = nullptr;                                           // hstate | h image or gh | W_hh image
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&buf, (2 * state + (path ? nw : ngh)) * sizeof(float), st));
    float *hstate = buf, *h_img = buf + state, *tail = buf + 2 * state;
    int rc = 0;
    if (path) {
        rc = gvd_pack_f16x3(Whh, G, 6 * G, G, tail, G, st, GVD_F16_SW);
        if (!rc) rc = gvd_gru_layer_f16(gi, tail, bhh, hstate, h_img, out, (const long long*)sample_idx, B, T, G, st);
    } else {
        if (cudaMemsetAsync(hstate, 0, state * sizeof(float), st) != cudaSuccess) { gvd_set_error("op_gru_layer: memset failed"); rc = 2; }
        if (!rc) rc = gru_layer_steps(gi, Whh, bhh, hstate, tail, out, (const long long*)sample_idx, B, T, G, st);
    }
    cudaFreeAsync(buf, st);
    return rc;
}
// The decode attention (attn_partial_kernel) with every AttnArgs field the decode step sets.  ticket != NULL: the last chunk CTA of each row
// merges the partials (the decode step's fused path; the caller zeroes the tickets once); ticket == NULL: attn_combine_kernel merges them
// after the partial launch, into x_out at pitch H.  Test hook.
static int op_attention(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                        const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                        const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                        int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                        int B, int R, int T, int A, int H, int RC, int TC, int feat_div, int att_input_mode,
                        const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld, int region_attn_mode,
                        const int64_t* video_idx, const int64_t* sample_idx, const float* ctx_bias, void* stream, int path = 0) {
    GVD_REQUIRE(att_input_mode == GVD_ATT_INPUT_BOTH || att_input_mode == GVD_ATT_INPUT_FEATMAP || att_input_mode == GVD_ATT_INPUT_DUAL_REGION,
                "op_attention: unknown att_input_mode %d", att_input_mode);
    GVD_REQUIRE(region_attn_mode == GVD_REGION_ATTN_MIX || region_attn_mode == GVD_REGION_ATTN_MIX_MUL || region_attn_mode == GVD_REGION_ATTN_DP,
                "op_attention: unknown region_attn_mode %d", region_attn_mode);
    const bool dual = att_input_mode == GVD_ATT_INPUT_DUAL_REGION, dp = region_attn_mode == GVD_REGION_ATTN_DP;
    GVD_REQUIRE(p_pool && (pool || att_input_mode == GVD_ATT_INPUT_FEATMAP) && ((p_conv && conv) || dual) && ((w1 && b1) || (dual && dp)) &&
                ((w2 && b2) || dp) && att_mask && out_mask && z_out && partial && x_out && B >= 1 && R >= 1 && T >= 1 && feat_div >= 1 && B % feat_div == 0, "op_attention: bad arguments");
    GVD_REQUIRE(!dual || (ticket && gate_w && gate_b && gate_h && gate_ld >= H), "op_attention: dual_region needs the tickets and the gate");
    GVD_REQUIRE(q ? !q_part : (q_part && q_bias && q_S >= 1), "op_attention: give either q or (q_part, q_S >= 1, q_bias)");
    GVD_REQUIRE(z_stride_b >= R && (out_mask_stride == 0 || out_mask_stride >= R + 1), "op_attention: bad z / out_mask pitch");
    GVD_REQUIRE(x_ld == 0 || (x_ld >= H && x_ld % 4 == 0), "op_attention: x_ld must be 0 or a multiple of 4 covering H");
    GVD_REQUIRE(!x_pk || (x_pk_ld % 32 == 0 && x_pk_ld >= (H + 31) / 32 * 32), "op_attention: x_pk_ld must be a 32-multiple covering H");
    GVD_REQUIRE(ticket || ((x_ld == 0 || x_ld == H) && !x_pk), "op_attention: the separate combine writes x_out at pitch H and no image");
    AttnArgs a{};
    a.p_pool = p_pool; a.pool = pool; a.p_conv = p_conv; a.conv = conv; a.q = q;
    if (!q) { a.q_part = q_part; a.q_S = q_S; a.q_plane = (long long)B * 2 * A; a.q_bias = q_bias; }
    a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
    a.att_mask = att_mask; a.out_mask = out_mask; a.out_mask_stride = out_mask_stride; a.z_out = z_out; a.z_stride_b = z_stride_b;
    a.partial = partial; a.ticket = ticket; a.x_out = x_out; a.x_ld = x_ld; a.x_pk = x_pk; a.x_pk_ld = x_pk_ld;
    a.B = B; a.R = R; a.T = T; a.A = A; a.H = H; a.RC = RC; a.TC = TC; a.feat_div = feat_div; a.mode = att_input_mode;
    a.gate_w = gate_w; a.gate_b = gate_b; a.gate_h = gate_h; a.gate_ld = gate_ld; a.form = region_attn_mode;
    if (dp) { a.w2 = a.b2 = nullptr; if (dual) a.w1 = a.b1 = nullptr; }          // the kernel must not need them
    a.vid = (const long long*)video_idx; a.win = (const long long*)sample_idx; a.ctx_bias = ctx_bias;
    cudaStream_t st = (cudaStream_t)stream;
    GVD_TRY(gvd_attn_partial_path(a, path, st));
    if (ticket) return 0;
    int nch_r, nch_t;
    gvd_attn_chunks(R, T, RC, TC, &nch_r, &nch_t);
    return gvd_attn_combine(partial, x_out, B, H, nch_r, nch_t, att_input_mode, st);
}
extern "C" GVD_API int gvd_op_attention_form(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                                             const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                                             const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                                             int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                                             int B, int R, int T, int A, int H, int RC, int TC, int feat_div, int att_input_mode,
                                             const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld, int region_attn_mode,
                                             void* stream) {
    return op_attention(p_pool, pool, p_conv, conv, q, q_part, q_S, q_bias, w1, b1, w2, b2, att_mask, out_mask, out_mask_stride, z_out,
                        z_stride_b, partial, ticket, x_out, x_ld, x_pk, x_pk_ld, B, R, T, A, H, RC, TC, feat_div, att_input_mode, gate_w,
                        gate_b, gate_h, gate_ld, region_attn_mode, nullptr, nullptr, nullptr, stream);
}
extern "C" GVD_API int gvd_op_attention_video(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                                              const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                                              const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                                              int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                                              int B, int R, int T, int A, int H, int RC, int TC, int feat_div, int att_input_mode,
                                              const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld, int region_attn_mode,
                                              const int64_t* video_idx, const int64_t* sample_idx, const float* ctx_bias, void* stream) {
    GVD_REQUIRE(video_idx && sample_idx && ctx_bias, "op_attention_video: video_idx, sample_idx and ctx_bias are required");
    return op_attention(p_pool, pool, p_conv, conv, q, q_part, q_S, q_bias, w1, b1, w2, b2, att_mask, out_mask, out_mask_stride, z_out,
                        z_stride_b, partial, ticket, x_out, x_ld, x_pk, x_pk_ld, B, R, T, A, H, RC, TC, feat_div, att_input_mode, gate_w,
                        gate_b, gate_h, gate_ld, region_attn_mode, video_idx, sample_idx, ctx_bias, stream);
}
// gvd_op_attention_video's arguments (video_idx / sample_idx / ctx_bias may be NULL: per-clip features) and the kernel: path 0 =
// attn_partial_kernel (one CTA per row, what the decode runs), 1 = attn_group_kernel (one CTA per group of a clip's rows).  Test and
// measurement hook.
extern "C" GVD_API int gvd_op_attention_path(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                                             const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                                             const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                                             int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                                             int B, int R, int T, int A, int H, int RC, int TC, int feat_div, int att_input_mode,
                                             const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld, int region_attn_mode,
                                             const int64_t* video_idx, const int64_t* sample_idx, const float* ctx_bias, int path, void* stream) {
    GVD_REQUIRE(path == 0 || path == 1, "op_attention_path: path must be 0 (per row) or 1 (row groups), got %d", path);
    GVD_REQUIRE(!video_idx || (sample_idx && ctx_bias), "op_attention_path: video rows need sample_idx and ctx_bias");
    return op_attention(p_pool, pool, p_conv, conv, q, q_part, q_S, q_bias, w1, b1, w2, b2, att_mask, out_mask, out_mask_stride, z_out,
                        z_stride_b, partial, ticket, x_out, x_ld, x_pk, x_pk_ld, B, R, T, A, H, RC, TC, feat_div, att_input_mode, gate_w,
                        gate_b, gate_h, gate_ld, region_attn_mode, video_idx, sample_idx, ctx_bias, stream, path);
}
extern "C" GVD_API int gvd_op_attention_mode(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                                             const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                                             const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                                             int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                                             int B, int R, int T, int A, int H, int RC, int TC, int feat_div, int att_input_mode,
                                             const float* gate_w, const float* gate_b, const float* gate_h, int64_t gate_ld, void* stream) {
    GVD_REQUIRE(w1 && b1 && w2 && b2, "op_attention: bad arguments");
    return gvd_op_attention_form(p_pool, pool, p_conv, conv, q, q_part, q_S, q_bias, w1, b1, w2, b2, att_mask, out_mask, out_mask_stride, z_out,
                                 z_stride_b, partial, ticket, x_out, x_ld, x_pk, x_pk_ld, B, R, T, A, H, RC, TC, feat_div, att_input_mode, gate_w,
                                 gate_b, gate_h, gate_ld, GVD_REGION_ATTN_MIX, stream);
}
extern "C" GVD_API int gvd_op_attention(const float* p_pool, const float* pool, const float* p_conv, const float* conv, const float* q,
                                        const float* q_part, int q_S, const float* q_bias, const float* w1, const float* b1, const float* w2,
                                        const float* b2, const uint8_t* att_mask, const uint8_t* out_mask, int64_t out_mask_stride, float* z_out,
                                        int64_t z_stride_b, float* partial, int* ticket, float* x_out, int64_t x_ld, float* x_pk, int64_t x_pk_ld,
                                        int B, int R, int T, int A, int H, int RC, int TC, int feat_div, void* stream) {
    GVD_REQUIRE(pool, "op_attention: bad arguments");
    return gvd_op_attention_mode(p_pool, pool, p_conv, conv, q, q_part, q_S, q_bias, w1, b1, w2, b2, att_mask, out_mask, out_mask_stride, z_out,
                                 z_stride_b, partial, ticket, x_out, x_ld, x_pk, x_pk_ld, B, R, T, A, H, RC, TC, feat_div, GVD_ATT_INPUT_BOTH,
                                 nullptr, nullptr, nullptr, 0, stream);
}
// beam_topk / row_argmax on their own.  Test hooks.
extern "C" GVD_API int gvd_op_beam_topk(const float* logits, int64_t ld, int rows, int V, int K, float* topv, int* topi, void* stream) {
    GVD_REQUIRE(logits && topv && topi && rows >= 1 && ld >= V, "op_beam_topk: bad arguments");
    return gvd_beam_topk(logits, ld, rows, V, K, topv, topi, (cudaStream_t)stream);
}
extern "C" GVD_API int gvd_op_row_argmax(const float* z, int64_t ld, int rows, int R, int* idx, void* stream) {
    GVD_REQUIRE(z && idx && rows >= 1 && R >= 1 && ld >= R, "op_row_argmax: bad arguments");
    return gvd_row_argmax(z, ld, rows, R, idx, (cudaStream_t)stream);
}
// gvd_beam_decode's bookkeeping (beam_search_run) with the model replaced by a script: step t's logits are logits[t] [B*K, V], the region
// scores of core step t are z[t] [B*K, R] (t = 0: <bos>), and the recurrent state is one probe buffer [B*K, H] that is reordered like the
// model's state.  The bookkeeping buffers are allocated here.  Test hook.
static int beam_search_scripted(const float* logits, const float* z, float* probe, int B, int K, int L, int V, int R, int H, int64_t* seq_out,
                                float* logp_out, int64_t* att2_idx_out, int* parents_out, float* att2_out, void* stream) {
    GVD_REQUIRE(logits && z && probe && seq_out && logp_out && att2_idx_out && parents_out && B >= 1 && V >= 1 && R >= 1 && H >= 4 && H % 4 == 0,
                "op_beam_search_scripted: bad arguments");
    GVD_REQUIRE(K >= 1 && L >= 1, "op_beam_search_scripted: beam_size and seq_length must be >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t BK = (size_t)B * K, BLK = (size_t)B * L * K;
    const size_t n4 = 3 * BLK + 2 * BK * K + 4 * BK + 3 * (size_t)B + 2 * (size_t)B * L;   // 4-byte words after the gather rows and tokens
    char* buf = nullptr;
    GVD_CHECK_CUDA(cudaMallocAsync((void**)&buf, BK * H * 4 + BK * 8 + n4 * 4, st));
    float* gather_tmp = (float*)buf;                                 // [B*K, H], 16-byte rows
    BeamBufs bb{};
    bb.tokens = (long long*)(buf + BK * H * 4);
    int* p = (int*)(bb.tokens + BK);
    auto take = [&](size_t n) { int* r = p; p += n; return r; };
    bb.seq = take(BLK); bb.att = take(BLK); bb.lp = (float*)take(BLK); bb.topv = (float*)take(BK * K); bb.topi = take(BK * K);
    bb.sums = (float*)take(BK); bb.parent = take(BK); bb.att_ind = take(BK);
    int* bos_att = take(BK);
    bb.done_flag = take(B); bb.done_slot = take(B); bb.done_step = take(B); bb.done_seq = take((size_t)B * L); bb.done_lp = (float*)take((size_t)B * L);
    bb.parent_hist = parents_out;
    auto scores = [&](int t, const float** zt) { *zt = z + (size_t)t * BK * R; return 0; };
    auto step_logits = [&](int t, const float** lg, long long* ld) { *lg = logits + (size_t)t * BK * V; *ld = V; return 0; };
    auto state = [&](int, float** bufs) { bufs[0] = probe; return 1; };
    const int rc = beam_search_run(bb, bos_att, gather_tmp, B, K, L, V, R, H, seq_out, logp_out, att2_idx_out, z, att2_out, st, scores, step_logits,
                                   state);
    cudaFreeAsync(buf, st);
    return rc;
}
extern "C" GVD_API int gvd_op_beam_search_scripted(const float* logits, const float* z, float* probe, int B, int K, int L, int V, int R, int H,
                                                   int64_t* seq_out, float* logp_out, int64_t* att2_idx_out, int* parents_out, void* stream) {
    return beam_search_scripted(logits, z, probe, B, K, L, V, R, H, seq_out, logp_out, att2_idx_out, parents_out, nullptr, stream);
}
// ... and the region scores of the returned caption, gathered along its ancestor chain from the script's z (gvd_beam_decode_att2's
// att2_logits_out).  Test hook.
extern "C" GVD_API int gvd_op_beam_att2_scripted(const float* logits, const float* z, float* probe, int B, int K, int L, int V, int R, int H,
                                                 int64_t* seq_out, float* logp_out, int64_t* att2_idx_out, int* parents_out, float* att2_out,
                                                 void* stream) {
    GVD_REQUIRE(att2_out, "op_beam_att2_scripted: null att2_out");
    return beam_search_scripted(logits, z, probe, B, K, L, V, R, H, seq_out, logp_out, att2_idx_out, parents_out, att2_out, stream);
}
// Batched short-K product C[b,h] = A[b,:,h*hs:(h+1)*hs] . W[b,:,h*hs:(h+1)*hs]^T through the A-stationary kernel (the attention-score shape)
extern "C" GVD_API int gvd_op_scores_tc(const float* A, const float* W, float* C, int nb, int nh, int M, int N, int hs, int64_t ld, void* stream) {
    GVD_REQUIRE(A && W && C, "op_scores_tc: null argument");
    GemmArgs g{};
    g.A = A; g.lda = ld; g.sAb = (long long)M * ld; g.sAh = hs;
    g.W = W; g.ldw = ld; g.sWb = (long long)N * ld; g.sWh = hs;
    g.C = C; g.ldc = N; g.sCb = (long long)nh * M * N; g.sCh = (long long)M * N;
    g.M = M; g.N = N; g.K = hs; g.nh = nh; g.alpha = 1.f;
    return gvd_gemm_nt_astat(g, nb * nh, (cudaStream_t)stream);
}
// Self-attention core of one encoder layer on a packed projection buffer qkv [nb, R, 3*HP] (Q | K | V, heads of width hs at
// column h*hs):  out[nb, R, HP] = concat_h softmax(Q_h K_h^T * scale) V_h through the fused wgmma pair.  Test hook: the
// scratch buffers are allocated here.  E [nb,nh,R,R] (numerators) and F [nb,nh,ceil(R/32),R] (group factors) are caller
// buffers; stages: bit 0 = scores (writes E, F), bit 1 = P.V (reads E, F, writes out).
extern "C" GVD_API int gvd_op_self_attention_tc(const float* qkv, float* out, int nb, int nh, int R, int hs, int HP, float scale, float* E,
                                                float* F, int stages, void* stream) {
    GVD_REQUIRE(qkv && out && E && F && nb > 0 && nh > 0 && R > 0 && R % 4 == 0 && HP % 4 == 0 && nh * hs <= HP, "op_self_attention_tc: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t BR = (size_t)nb * R;
    float *khi = nullptr, *klo = nullptr, *vh = nullptr, *vl = nullptr;
    const bool att16 = gvd_backend_on(BK_ATT_F16);          // fp16x3 images instead of tf32 planes (same switch as the prologue)
    const int KH = (hs + 31) / 32 * 32, Rp = (R + 31) / 32 * 32;
    auto body16 = [&]() -> int {
        GVD_CHECK_CUDA(cudaMalloc(&khi, BR * nh * KH * 4)); GVD_CHECK_CUDA(cudaMalloc(&vh, (size_t)nb * HP * Rp * 4));
        if (stages & 1) {
            GVD_TRY(gvd_pack_heads_f16x3(qkv + HP, 3 * HP, (long long)BR, nh, hs, hs, KH, GVD_ATT_SK, khi, st));
            GemmArgs g{};
            g.A = qkv; g.lda = 3 * HP; g.sAb = (long long)R * 3 * HP; g.sAh = hs;
            g.W = khi; g.ldw = (long long)nh * KH; g.sWb = (long long)R * nh * KH; g.sWh = KH;
            g.C = E; g.ldc = R; g.sCb = (long long)nh * R * R; g.sCh = (long long)R * R;
            g.M = R; g.N = R; g.K = hs; g.nh = nh; g.alpha = 1.f;
            GVD_TRY(gvd_attn_scores_tc(g, nullptr, F, scale, nb * nh, st, 1));
        }
        if (stages & 2) {
            GVD_TRY(gvd_transpose_pack_f16x3(qkv + 2 * HP, vh, nb, R, HP, 3 * HP, Rp, GVD_ATT_SV, st));
            GemmArgs v{};
            v.A = E; v.lda = R; v.sAb = (long long)nh * R * R; v.sAh = (long long)R * R;
            v.W = vh; v.ldw = Rp; v.sWb = (long long)HP * Rp; v.sWh = (long long)hs * Rp;
            v.C = out; v.ldc = HP; v.sCb = (long long)R * HP; v.sCh = hs;
            v.M = R; v.N = hs; v.K = R; v.nh = nh; v.alpha = 1.f;
            GVD_TRY(gvd_attn_pv_tc(v, nullptr, F, nb * nh, st, 1));
        }
        GVD_CHECK_CUDA(cudaStreamSynchronize(st));
        return 0;
    };
    auto body = [&]() -> int {
        GVD_CHECK_CUDA(cudaMalloc(&khi, BR * HP * 4)); GVD_CHECK_CUDA(cudaMalloc(&klo, BR * HP * 4));
        GVD_CHECK_CUDA(cudaMalloc(&vh, BR * HP * 4)); GVD_CHECK_CUDA(cudaMalloc(&vl, BR * HP * 4));
        if (stages & 1) {
            GVD_TRY(gvd_split_hilo(qkv + HP, 3 * HP, khi, klo, HP, (long long)BR, HP, st));
            GemmArgs g{};
            g.A = qkv; g.lda = 3 * HP; g.sAb = (long long)R * 3 * HP; g.sAh = hs;
            g.W = khi; g.ldw = HP; g.sWb = (long long)R * HP; g.sWh = hs;
            g.C = E; g.ldc = R; g.sCb = (long long)nh * R * R; g.sCh = (long long)R * R;
            g.M = R; g.N = R; g.K = hs; g.nh = nh; g.alpha = 1.f;
            GVD_TRY(gvd_attn_scores_tc(g, klo, F, scale, nb * nh, st));
        }
        if (stages & 2) {
            GVD_TRY(gvd_transpose_split(qkv + 2 * HP, vh, vl, nb, R, HP, 3 * HP, st));
            GemmArgs v{};
            v.A = E; v.lda = R; v.sAb = (long long)nh * R * R; v.sAh = (long long)R * R;
            v.W = vh; v.ldw = R; v.sWb = (long long)HP * R; v.sWh = (long long)hs * R;
            v.C = out; v.ldc = HP; v.sCb = (long long)R * HP; v.sCh = hs;
            v.M = R; v.N = hs; v.K = R; v.nh = nh; v.alpha = 1.f;
            GVD_TRY(gvd_attn_pv_tc(v, vl, F, nb * nh, st));
        }
        GVD_CHECK_CUDA(cudaStreamSynchronize(st));
        return 0;
    };
    const int rc = att16 ? body16() : body();
    cudaFree(khi); cudaFree(klo); cudaFree(vh); cudaFree(vl);
    return rc;
}
// Self-attention core through the fused kernel (gvd_attn.cu): key / V^T images built here, O as fp32 (out) or as its operand image (img).
extern "C" GVD_API int gvd_op_self_attention_fused(const float* qkv, float* out, int nb, int nh, int R, int hs, int HP, float scale, float* img,
                                                   int64_t img_ld, void* stream) {
    GVD_REQUIRE(qkv && (out || img) && nb > 0 && nh > 0 && R > 0 && HP % 4 == 0 && nh * hs <= HP, "op_self_attention_fused: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t BR = (size_t)nb * R;
    const int KH = (hs + 31) / 32 * 32, Rp = (R + 31) / 32 * 32;
    float *kimg = nullptr, *vimg = nullptr;
    auto body = [&]() -> int {
        GVD_CHECK_CUDA(cudaMalloc(&kimg, BR * nh * KH * 4));
        GVD_CHECK_CUDA(cudaMalloc(&vimg, (size_t)nb * HP * Rp * 4));
        GVD_TRY(gvd_pack_heads_f16x3(qkv + HP, 3 * HP, (long long)BR, nh, hs, hs, KH, GVD_ATT_SK, kimg, st));
        GVD_TRY(gvd_transpose_pack_f16x3(qkv + 2 * HP, vimg, nb, R, HP, 3 * HP, Rp, GVD_ATT_SV, st));
        GVD_TRY(gvd_self_attn_fused(qkv, 3 * HP, kimg, vimg, nb, R, nh, hs, HP, scale, out, HP, img, img_ld, st));
        GVD_CHECK_CUDA(cudaStreamSynchronize(st));
        return 0;
    };
    const int rc = body();
    cudaFree(kimg); cudaFree(vimg);
    return rc;
}
extern "C" GVD_API int gvd_op_tanh(const float* x, float* y, int n, void* stream) { return gvd_tanh_test(x, y, n, (cudaStream_t)stream); }
