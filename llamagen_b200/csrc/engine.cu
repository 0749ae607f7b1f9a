// C-ABI entry points of the AR transformer engine (see include/llamagen_b200.h).
//
// Replaces, for inference only:
//   autoregressive/models/gpt.py:316-330  Transformer.setup_caches   -> lg_engine_set_workspace
//   autoregressive/models/gpt.py:341-368  Transformer.forward        -> Engine::forward
//   autoregressive/models/generate.py:77-176 prefill/decode/generate -> lg_prefill / lg_decode_step / lg_generate
// The decode loop never leaves the device: sampled tokens, the position and the step counter live in
// HBM, so one captured CUDA graph of a decode step is replayed S-2 times with no host round trip.
#include "kernels.cuh"
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

std::string& lg_err_slot() {
    static thread_local std::string s;
    return s;
}
int lg_fail(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    lg_err_slot() = buf;
    return -1;
}
std::atomic<uint64_t> g_lg_launches{0};
int g_lg_pdl = -1;
int lg_env_flag(const char* name, int dflt) {
    const char* e = getenv(name);
    if (!e || !e[0]) return dflt;
    return atoi(e);
}
bool lg_debug_sync() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("LG_DEBUG_SYNC"); v = (e && e[0] == '1') ? 1 : 0; }
    return v == 1;
}

// ---------------------------------------------------------------------------------------------------
// event-pair profiler
namespace {
struct ProfState {
    bool on = false;
    std::vector<cudaEvent_t> pool;      // flat pairs
    std::vector<int> cls;               // class of each recorded pair
    size_t used = 0;                    // pairs recorded since the last drain
    double total_ms[PC_COUNT] = {0};
    uint64_t count[PC_COUNT] = {0};
    int cur = -1;
};
ProfState g_prof;
void prof_drain() {
    if (g_prof.used == 0) return;
    cudaDeviceSynchronize();
    for (size_t i = 0; i < g_prof.used; ++i) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, g_prof.pool[2 * i], g_prof.pool[2 * i + 1]) == cudaSuccess) {
            g_prof.total_ms[g_prof.cls[i]] += ms;
            g_prof.count[g_prof.cls[i]] += 1;
        }
    }
    g_prof.used = 0;
}
}  // namespace
bool prof_enabled() { return g_prof.on; }
void prof_begin(int cls, cudaStream_t st) {
    if (!g_prof.on) return;
    if (g_prof.used >= 16384) prof_drain();
    if (g_prof.pool.size() < 2 * (g_prof.used + 1)) {
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        g_prof.pool.push_back(a);
        g_prof.pool.push_back(b);
        g_prof.cls.push_back(cls);
    }
    g_prof.cls[g_prof.used] = cls;
    g_prof.cur = (int)g_prof.used;
    cudaEventRecord(g_prof.pool[2 * g_prof.used], st);
}
void prof_end(cudaStream_t st) {
    if (!g_prof.on || g_prof.cur < 0) return;
    cudaEventRecord(g_prof.pool[2 * g_prof.cur + 1], st);
    g_prof.used += 1;
    g_prof.cur = -1;
}

namespace {

struct Tensor {
    const void* p = nullptr;
    int64_t shape[4] = {0, 0, 0, 0};
    int ndim = 0;
    int dtype = 0;
};

size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

struct Workspace {
    char* base = nullptr;
    size_t bytes = 0;
    int rows = 0, max_seq = 0;
    // carved pointers
    char *kcache = nullptr, *vcache = nullptr;
    char *h = nullptr, *xn = nullptr, *q = nullptr, *attn = nullptr, *ff = nullptr, *x0 = nullptr;
    float *partial = nullptr, *logits = nullptr;
    int32_t* tokens = nullptr;
    int* counters = nullptr;  // [0] = pos, [1] = step (chain g of a split uses [2g], [2g+1])
    size_t layer_cache_bytes = 0;
    size_t partial_floats = 0;
    alignas(64) unsigned char kmap[128];   // CUtensorMap over the K / V cache regions (bf16 / fp16 only)
    alignas(64) unsigned char vmap[128];
    alignas(64) unsigned char kmap16[128];  // same regions, 16-row boxes (tail chunk of the decode attention)
    alignas(64) unsigned char vmap16[128];
    bool have_maps = false;
};

struct Layer {
    const void *wqkv, *wo, *w1, *w3, *w2, *attn_norm, *ffn_norm;
};

}  // namespace

struct lg_engine {
    lg_model_cfg cfg;
    int device = 0;
    int hd = 0;
    int hdp = 0;                          // KV-cache row width in elements: hd, or 112 for head_dim 100 in bf16 / fp16 (GPT-3B) so that the rows
                                          // are 16-byte multiples and the TMA attention kernel can stream them (dims 100..111 stay zero)
    size_t esz = 2;
    // KV-cache storage (lg_engine_set_kv_cache): the model dtype, or fp8 e4m3 with per-layer power-of-two (k, v) scales
    bool kv_f8 = false;
    size_t kv_esz = 2;                    // bytes per cached element
    std::vector<float> kv_scales;         // [n_layer][2] (fp8 only)
    std::unordered_map<std::string, Tensor> w;
    std::vector<Layer> layers;
    const void *tok_emb = nullptr, *cls_table = nullptr, *cap_fc1 = nullptr, *cap_fc2 = nullptr, *uncond = nullptr;
    const void *final_norm = nullptr, *output = nullptr;
    const float* freqs = nullptr;
    bool finalized = false;
    Workspace ws;                         // ACTIVE workspace (full, or one of the two halves while a group is issued)
    static constexpr int kMaxChains = 8;
    Workspace full, sub[kMaxChains];      // sub[g]: rows/n_sub each, carved INSIDE the regions of `full` (multi-chain decode)
    int n_sub = 0;                        // 0: no split available
    bool use_graph = true;
    bool ws_needs_zero = false;           // KV cache + counters of `full` still have to be zero-filled (done on the caller's stream)
    bool skip_first_norm = false;         // set by the decode loop when the sample kernel's fused tail already wrote xn = RMSNorm_0(h)
    cudaStream_t works[kMaxChains] = {};   // engine-owned streams (one per chain)
    cudaEvent_t ev_fork = nullptr, ev_joins[kMaxChains] = {};
    ~lg_engine() {
        for (int i = 0; i < kMaxChains; ++i) {
            if (works[i]) cudaStreamDestroy(works[i]);
            if (ev_joins[i]) cudaEventDestroy(ev_joins[i]);
        }
        if (ev_fork) cudaEventDestroy(ev_fork);
    }

    // R <= 8 decode steps on the column-owner GEMV path (gemv_small.cu); shared by forward() and the decode loop's fused tail
    bool small_row_path(int M, const AttnArgs& aa) const {
        const int D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size, dt = cfg.dtype;
        return M <= 8 && lg_env_flag("LG_SMALL_R", 1) && lg_env_flag("LG_FUSE_QKV", 1) && attn_tma_enabled() && attn_tma_supported(aa) &&
               gemv_small_supported(M, 3 * D, D, dt, false) && gemv_small_supported(M, D, D, dt, false) &&
               gemv_small_supported(M, F, D, dt, true) && gemv_small_supported(M, D, F, dt, false) && gemv_small_supported(M, V, D, dt, false);
    }
    size_t carve(Workspace& o, char* base, int rows, int max_seq) const;
    int zero_fill_if_needed(cudaStream_t st) {
        if (!ws_needs_zero || !full.base) return 0;
        LG_CUDA_OK(cudaMemsetAsync(full.kcache, 0, 2 * ((full.layer_cache_bytes * cfg.n_layer + 255) / 256 * 256), st));
        LG_CUDA_OK(cudaMemsetAsync(full.counters, 0, 128 * sizeof(int), st));
        ws_needs_zero = false;
        return 0;
    }
    int forward(int M, int Tq, PosArg pos, const float* emb_mask, int B, float* logits_out, bool round_out,
                cudaStream_t st);
    int embed_cond(const void* cond, int B, int R, int T, cudaStream_t st);
    int gemm(const void* x, int M, int N, int K, const void* wa, const void* wb, int n_split, int* ksplit,
             float* direct_out, cudaStream_t st, const GemmNext* next = nullptr);
};

size_t lg_engine::carve(Workspace& o, char* base, int rows, int max_seq) const {
    const int L = cfg.n_layer, D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size, H = cfg.n_head;
    const int Tc = cfg.model_type == LG_MODEL_T2I ? cfg.cls_token_num : 1;
    const size_t Mmax = (size_t)rows * Tc;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* p = base ? base + off : nullptr;
        off += align_up(bytes);
        return p;
    };
    o.layer_cache_bytes = (size_t)rows * H * max_seq * hdp * kv_esz;
    o.kcache = take(o.layer_cache_bytes * L);
    o.vcache = take(o.layer_cache_bytes * L);
    o.h = take(Mmax * D * esz);
    o.xn = take(Mmax * D * esz);
    o.q = take(Mmax * D * esz);
    o.attn = take(Mmax * D * esz);
    o.ff = take(Mmax * F * esz);
    o.x0 = take(cfg.model_type == LG_MODEL_T2I ? Mmax * cfg.caption_dim * esz : 0);
    size_t pf = 0;
    const int Ms[2] = {rows, (int)Mmax};
    for (int i = 0; i < 2; ++i) {
        const int M = Ms[i];
        pf = std::max(pf, gemm_partial_floats(M, 3 * D, D, cfg.dtype));
        pf = std::max(pf, gemm_partial_floats(M, D, D, cfg.dtype));
        pf = std::max(pf, gemm_partial_floats(M, 2 * F, D, cfg.dtype));
        pf = std::max(pf, gemm_partial_floats(M, D, F, cfg.dtype));
        if (cfg.model_type == LG_MODEL_T2I) pf = std::max(pf, gemm_partial_floats(M, D, cfg.caption_dim, cfg.dtype));
    }
    pf = std::max(pf, gemm_partial_floats(rows, V, D, cfg.dtype));
    o.partial_floats = pf;
    o.partial = (float*)take(pf * sizeof(float));
    o.logits = (float*)take((size_t)rows * V * sizeof(float));
    o.tokens = (int32_t*)take((size_t)rows * sizeof(int32_t));
    o.counters = (int*)take(128 * sizeof(int));   // [0, 16): pos/step per chain (<= 8 chains)
    o.rows = rows;
    o.max_seq = max_seq;
    return off;
}

int lg_engine::gemm(const void* x, int M, int N, int K, const void* wa, const void* wb, int n_split, int* ksplit,
                    float* direct_out, cudaStream_t st, const GemmNext* next) {
    // when the plan needs a single slab the GEMM can write straight into `direct_out`
    const size_t need = gemm_partial_floats(M, N, K, cfg.dtype);
    const size_t slabs = need / ((size_t)M * N);
    float* dst = (direct_out && slabs == 1) ? direct_out : ws.partial;
    // the plan (k-slices) is not monotone in M and depends on run-time switches: never trust the carve-time sizing blindly
    LG_REQUIRE(dst == direct_out || need <= ws.partial_floats, "gemm %dx%dx%d needs %zu partial floats, workspace holds %zu", M, N, K, need,
               ws.partial_floats);
    GemmPlan plan;
    LG_TRY(gemm_partial(x, K, wa, wb, n_split, M, N, K, cfg.dtype, dst, &plan, st, next));
    *ksplit = plan.ksplit;
    return dst == direct_out ? 1 : 0;
}

int lg_engine::forward(int M, int Tq, PosArg pos, const float* emb_mask, int B, float* logits_out, bool round_out,
                       cudaStream_t st) {
    const int L = cfg.n_layer, D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size, H = cfg.n_head;
    const int R = M / Tq;
    const int dt = cfg.dtype;
    int ks = 1;
    auto attn_args = [&](int l) {
        AttnArgs aa;
        aa.q = ws.q; aa.kcache = ws.kcache + (size_t)l * ws.layer_cache_bytes; aa.vcache = ws.vcache + (size_t)l * ws.layer_cache_bytes;
        aa.out = ws.attn; aa.R = R; aa.Tq = Tq; aa.H = H; aa.hd = hd;
        aa.maxS = ws.max_seq; aa.pos = pos; aa.emb_mask = emb_mask; aa.B = B; aa.hdp = hdp;
        aa.Tc = cfg.cls_token_num; aa.scale = 1.0f / sqrtf((float)hd); aa.dtype = dt;
        if (kv_f8) {   // the K scale folds into the softmax scale, the V scale into O / L, the writers divide by them
            const float ks = kv_scales[2 * l], vs = kv_scales[2 * l + 1];
            aa.kv_f8 = 1; aa.scale *= ks; aa.k_inv = 1.0f / ks; aa.v_inv = 1.0f / vs; aa.v_scale = vs;
        }
        if (ws.have_maps) {
            aa.kmap = ws.kmap; aa.vmap = ws.vmap; aa.kmap16 = ws.kmap16; aa.vmap16 = ws.vmap16;
            aa.cache_row_base = (long long)l * ws.rows * H * ws.max_seq;
        }
        return aa;
    };
    // ---- R <= 8 decode step (batch-1 latency path, gemv_small.cu): 5 dependent kernels per layer, no slabs
    if (Tq == 1 && small_row_path(M, attn_args(0))) {
        skip_first_norm = false;
        for (int l = 0; l < L; ++l) {
            const Layer& ly = layers[l];
            GemvSmall gq{ly.wqkv, nullptr, 3 * D, D, M, ws.h, ly.attn_norm, cfg.norm_eps, ws.partial, nullptr, nullptr, dt};
            LG_PROF(PC_GEMM_QKV, st, launch_gemv_small(gq, st));
            AttnArgs aa = attn_args(l);
            aa.qkv_partial = ws.partial; aa.qkv_ksplit = 1; aa.freqs = freqs;
            LG_PROF(PC_ATTENTION, st, launch_attention(aa, st));
            GemvSmall go{ly.wo, nullptr, D, D, M, ws.attn, nullptr, 0.f, nullptr, ws.h, nullptr, dt};
            LG_PROF(PC_GEMM_WO, st, launch_gemv_small(go, st));
            GemvSmall g13{ly.w1, ly.w3, F, D, M, ws.h, ly.ffn_norm, cfg.norm_eps, nullptr, nullptr, ws.ff, dt};
            LG_PROF(PC_GEMM_W13, st, launch_gemv_small(g13, st));
            GemvSmall g2{ly.w2, nullptr, D, F, M, ws.ff, nullptr, 0.f, nullptr, ws.h, nullptr, dt};
            LG_PROF(PC_GEMM_W2, st, launch_gemv_small(g2, st));
        }
        GemvSmall gh{output, nullptr, V, D, M, ws.h, final_norm, cfg.norm_eps, logits_out, nullptr, nullptr, dt};
        LG_PROF(PC_GEMM_HEAD, st, launch_gemv_small(gh, st));
        return 0;
    }
    if (!skip_first_norm) LG_PROF(PC_EMBED_MISC, st, launch_rmsnorm(ws.h, layers[0].attn_norm, ws.xn, M, D, cfg.norm_eps, dt, st));
    skip_first_norm = false;
    for (int l = 0; l < L; ++l) {
        const Layer& ly = layers[l];
        char* kc = ws.kcache + (size_t)l * ws.layer_cache_bytes;
        char* vc = ws.vcache + (size_t)l * ws.layer_cache_bytes;
        const size_t eb = esz;
        GemmNext nx_wo{ly.wo, (size_t)D * D * eb, nullptr, 0};
        GemmNext nx_w13{ly.w1, (size_t)F * D * eb, ly.w3, (size_t)F * D * eb};
        GemmNext nx_w2{ly.w2, (size_t)D * F * eb, nullptr, 0};
        GemmNext nx_qkv{(l + 1 < L) ? layers[l + 1].wqkv : output, (l + 1 < L) ? (size_t)3 * D * D * eb : (size_t)V * D * eb, nullptr, 0};
        LG_PROF(PC_GEMM_QKV, st, gemm(ws.xn, M, 3 * D, D, ly.wqkv, nullptr, 0, &ks, nullptr, st, &nx_wo));
        QkvEpiArgs qa;
        qa.partial = ws.partial; qa.ksplit = ks; qa.M = M; qa.Tq = Tq; qa.D = D; qa.H = H; qa.hd = hd;
        qa.pos = pos; qa.freqs = freqs; qa.q = ws.q; qa.kcache = kc; qa.vcache = vc; qa.maxS = ws.max_seq; qa.dtype = dt; qa.hdp = hdp;
        AttnArgs aa = attn_args(l);
        qa.kv_f8 = aa.kv_f8; qa.k_inv = aa.k_inv; qa.v_inv = aa.v_inv;
        // decode steps on the TMA path: the attention kernel is also the QKV epilogue (one dependent kernel less)
        const bool fuse_qkv = lg_env_flag("LG_FUSE_QKV", 1) && attn_tma_enabled() && attn_tma_supported(aa);
        if (fuse_qkv) {
            aa.qkv_partial = ws.partial; aa.qkv_ksplit = ks; aa.freqs = freqs;
        } else {
            LG_PROF(PC_QKV_EPI, st, launch_qkv_epilogue(qa, st));
        }
        LG_PROF(PC_ATTENTION, st, launch_attention(aa, st));
        LG_PROF(PC_GEMM_WO, st, gemm(ws.attn, M, D, D, ly.wo, nullptr, 0, &ks, nullptr, st, &nx_w13));
        LG_PROF(PC_RESNORM, st, launch_residual_norm(ws.partial, ks, M, D, ws.h, ly.ffn_norm, ws.xn, cfg.norm_eps, dt, st));
        LG_PROF(PC_GEMM_W13, st, gemm(ws.xn, M, 2 * F, D, ly.w1, ly.w3, F, &ks, nullptr, st, &nx_w2));
        LG_PROF(PC_SILU, st, launch_silu_mul(ws.partial, ks, M, F, ws.ff, dt, st));
        LG_PROF(PC_GEMM_W2, st, gemm(ws.ff, M, D, F, ly.w2, nullptr, 0, &ks, nullptr, st, &nx_qkv));
        const void* next_norm = (l + 1 < L) ? layers[l + 1].attn_norm : final_norm;
        LG_PROF(PC_RESNORM, st, launch_residual_norm(ws.partial, ks, M, D, ws.h, next_norm, ws.xn, cfg.norm_eps, dt, st));
    }
    // head on the last position only (generate.py:58 reads logits[:, -1])
    const void* xlast = ws.xn;
    if (Tq > 1) {
        LG_TRY(launch_gather_last(ws.xn, R, Tq, D, dt, ws.q, st));
        xlast = ws.q;
    }
    (void)round_out;
    prof_begin(PC_GEMM_HEAD, st);
    GemmNext nx_first{layers[0].wqkv, (size_t)3 * D * D * esz, nullptr, 0};   // the next decode step starts with layer 0
    const int direct = gemm(xlast, R, V, D, output, nullptr, 0, &ks, logits_out, st, &nx_first);
    prof_end(st);
    if (direct < 0) return direct;
    if (direct == 0) LG_TRY(launch_reduce_f32(ws.partial, ks, R, V, logits_out, st));
    return 0;
}

int lg_engine::embed_cond(const void* cond, int B, int R, int T, cudaStream_t st) {
    const int D = cfg.dim, dt = cfg.dtype;
    if (cfg.model_type == LG_MODEL_C2I) {
        // LabelEmbedder (gpt.py:78-83); null class = num_classes (generate.py:130)
        return launch_embed(cls_table, (const int32_t*)cond, B, R, cfg.num_classes, D, dt, ws.h, st);
    }
    // CaptionEmbedder: cap_proj = fc2(gelu_tanh(fc1(x))) (gpt.py:110-131); uncond rows = uncond_embedding
    const int C = cfg.caption_dim, M = R * T;
    int ks = 1;
    LG_TRY(launch_build_caption_rows(cond, uncond, B, R, T, C, dt, ws.x0, st));
    LG_TRY(gemm(ws.x0, M, D, C, cap_fc1, nullptr, 0, &ks, nullptr, st));
    LG_TRY(launch_store_act(ws.partial, ks, M, D, ws.attn, 1, dt, st));
    LG_TRY(gemm(ws.attn, M, D, D, cap_fc2, nullptr, 0, &ks, nullptr, st));
    LG_TRY(launch_store_act(ws.partial, ks, M, D, ws.h, 0, dt, st));
    return 0;
}

// ---------------------------------------------------------------------------------------------------
extern "C" {

int lg_version(void) { return LG_ABI_VERSION; }
const char* lg_last_error(void) { return lg_err_slot().c_str(); }
uint64_t lg_launch_count(void) { return g_lg_launches.load(); }
void lg_reset_launch_count(void) { g_lg_launches.store(0); }

int lg_engine_create(const lg_model_cfg* cfg, int device, lg_engine** out) {
    LG_REQUIRE(cfg && out, "lg_engine_create: null argument");
    LG_REQUIRE(cfg->dtype == LG_DTYPE_F32 || lg_dtype_is16(cfg->dtype), "unsupported dtype %d (f32, bf16 and f16 only)", cfg->dtype);
    LG_REQUIRE(cfg->model_type == LG_MODEL_C2I || cfg->model_type == LG_MODEL_T2I, "please check model type");
    LG_REQUIRE(cfg->n_layer > 0 && cfg->n_head > 0 && cfg->dim > 0 && cfg->dim % cfg->n_head == 0, "bad model dims");
    const int hd = cfg->dim / cfg->n_head;
    LG_REQUIRE(hd == 64 || hd == 100 || hd == 128, "unsupported head_dim %d (64, 100, 128)", hd);
    LG_REQUIRE(cfg->dim % 8 == 0 && cfg->ffn_dim % 8 == 0 && cfg->vocab_size % 2 == 0, "dims must be multiples of 8");
    lg_engine* e = new lg_engine();
    e->cfg = *cfg;
    e->device = device;
    e->hd = hd;
    e->hdp = attn_kv_row_width(cfg->dtype, hd);
    e->esz = (size_t)lg_dtype_info(cfg->dtype).esz;
    e->kv_esz = e->esz;
    const char* ng = getenv("LG_NO_GRAPH");
    e->use_graph = !(ng && ng[0] == '1');
    *out = e;
    return 0;
}

void lg_engine_destroy(lg_engine* e) {
    if (!e) return;
    DeviceGuard guard(e->device);
    delete e;
}

int lg_engine_bind_weight(lg_engine* e, const char* name, const void* dev_ptr, const int64_t* shape, int ndim,
                          int dtype) {
    LG_REQUIRE(e && name && dev_ptr && shape && ndim >= 1 && ndim <= 4, "lg_engine_bind_weight: bad argument");
    Tensor t;
    t.p = dev_ptr;
    t.ndim = ndim;
    t.dtype = dtype;
    for (int i = 0; i < ndim; ++i) t.shape[i] = shape[i];
    e->w[name] = t;
    e->finalized = false;
    return 0;
}

static int need(lg_engine* e, const std::string& name, int dtype, std::initializer_list<int64_t> shape,
                const void** out) {
    auto it = e->w.find(name);
    LG_REQUIRE(it != e->w.end(), "missing weight '%s'", name.c_str());
    const Tensor& t = it->second;
    LG_REQUIRE(t.dtype == dtype, "weight '%s' has dtype %d, expected %d", name.c_str(), t.dtype, dtype);
    LG_REQUIRE(t.ndim == (int)shape.size(), "weight '%s' has %d dims, expected %d", name.c_str(), t.ndim, (int)shape.size());
    int i = 0;
    for (int64_t s : shape) {
        LG_REQUIRE(t.shape[i] == s, "weight '%s' dim %d is %lld, expected %lld", name.c_str(), i, (long long)t.shape[i], (long long)s);
        ++i;
    }
    LG_REQUIRE(((uintptr_t)t.p & 15) == 0, "weight '%s' is not 16-byte aligned", name.c_str());
    *out = t.p;
    return 0;
}

int lg_engine_finalize(lg_engine* e) {
    LG_REQUIRE(e, "null engine");
    const lg_model_cfg& c = e->cfg;
    const int D = c.dim, F = c.ffn_dim, V = c.vocab_size, dt = c.dtype;
    e->layers.resize(c.n_layer);
    for (int l = 0; l < c.n_layer; ++l) {
        const std::string p = "layers." + std::to_string(l) + ".";
        Layer& ly = e->layers[l];
        LG_TRY(need(e, p + "attention.wqkv.weight", dt, {3 * D, D}, &ly.wqkv));
        LG_TRY(need(e, p + "attention.wo.weight", dt, {D, D}, &ly.wo));
        LG_TRY(need(e, p + "feed_forward.w1.weight", dt, {F, D}, &ly.w1));
        LG_TRY(need(e, p + "feed_forward.w3.weight", dt, {F, D}, &ly.w3));
        LG_TRY(need(e, p + "feed_forward.w2.weight", dt, {D, F}, &ly.w2));
        LG_TRY(need(e, p + "attention_norm.weight", dt, {D}, &ly.attn_norm));
        LG_TRY(need(e, p + "ffn_norm.weight", dt, {D}, &ly.ffn_norm));
    }
    LG_TRY(need(e, "tok_embeddings.weight", dt, {V, D}, &e->tok_emb));
    LG_TRY(need(e, "norm.weight", dt, {D}, &e->final_norm));
    LG_TRY(need(e, "output.weight", dt, {V, D}, &e->output));
    if (c.model_type == LG_MODEL_C2I) {
        auto it = e->w.find("cls_embedding.embedding_table.weight");
        LG_REQUIRE(it != e->w.end(), "missing weight 'cls_embedding.embedding_table.weight'");
        LG_REQUIRE(it->second.dtype == dt && it->second.ndim == 2 && it->second.shape[1] == D &&
                       it->second.shape[0] > c.num_classes,
                   "cls_embedding.embedding_table.weight must be [>num_classes, dim] (needs the CFG null row)");
        e->cls_table = it->second.p;
    } else {
        LG_TRY(need(e, "cls_embedding.cap_proj.fc1.weight", dt, {D, c.caption_dim}, &e->cap_fc1));
        LG_TRY(need(e, "cls_embedding.cap_proj.fc2.weight", dt, {D, D}, &e->cap_fc2));
        LG_TRY(need(e, "cls_embedding.uncond_embedding", dt, {c.cls_token_num, c.caption_dim}, &e->uncond));
    }
    const void* fr = nullptr;
    LG_TRY(need(e, "freqs_cis", LG_DTYPE_F32, {c.cls_token_num + c.block_size, e->hd / 2, 2}, &fr));
    e->freqs = (const float*)fr;
    e->finalized = true;
    return 0;
}

int lg_engine_workspace_bytes(lg_engine* e, int rows, int max_seq, size_t* bytes) {
    LG_REQUIRE(e && bytes && rows > 0 && max_seq > 0, "lg_engine_workspace_bytes: bad argument");
    Workspace tmp;
    *bytes = e->carve(tmp, nullptr, rows, max_seq);
    return 0;
}

int lg_engine_set_workspace(lg_engine* e, void* dev_ws, size_t bytes, int rows, int max_seq) {
    LG_REQUIRE(e && dev_ws, "lg_engine_set_workspace: null argument");
    DeviceGuard guard(e->device);
    LG_REQUIRE(((uintptr_t)dev_ws & 255) == 0, "workspace must be 256-byte aligned");
    Workspace tmp;
    const size_t needb = e->carve(tmp, (char*)dev_ws, rows, max_seq);
    LG_REQUIRE(bytes >= needb, "workspace too small: %zu < %zu", bytes, needb);
    tmp.base = (char*)dev_ws;
    tmp.bytes = bytes;
    // The reference zero-fills the KV cache (gpt.py:174-175). The tensor-core attention multiplies masked
    // probabilities (exactly 0) with whatever sits in not-yet-written V rows, so those rows must be finite.
    // The zero-fill is enqueued on the CALLER'S stream by the first prefill / decode / generate that uses this workspace
    // (zero_fill_if_needed): a legacy-NULL-stream memset here would not be ordered against non-blocking streams that may
    // still be running kernels on memory the caching allocator has just recycled.
    e->ws_needs_zero = true;
    tmp.have_maps = false;
    const int dt = e->cfg.dtype;
    const int kvdt = e->kv_f8 ? LG_DTYPE_E4M3 : dt;   // storage type of the cache regions
    const long long total_rows = (long long)e->cfg.n_layer * rows * e->cfg.n_head * max_seq;
    if (attn_tma_maps_usable(dt, e->hd, e->hdp, total_rows)) {
        LG_TRY(attn_tma_make_map(tmp.kmap, tmp.kcache, total_rows, e->hdp, kvdt));
        LG_TRY(attn_tma_make_map(tmp.vmap, tmp.vcache, total_rows, e->hdp, kvdt));
        LG_TRY(attn_tma_make_map(tmp.kmap16, tmp.kcache, total_rows, e->hdp, kvdt, 1));
        LG_TRY(attn_tma_make_map(tmp.vmap16, tmp.vcache, total_rows, e->hdp, kvdt, 1));
        tmp.have_maps = true;
    }
    e->full = tmp;
    e->ws = tmp;
    // n equal sub-batch workspaces inside the same memory (every region scales with rows, so chain g takes the g-th
    // 1/n of every region; the K/V parts stay inside the zero-initialised cache regions).
    e->n_sub = 0;
    // Chain-count policy: every chain streams ALL the weights, so two chains only pay while a layer's weights survive in L2 between
    // the chains' visits, next to the KV and activation traffic of the other chain; otherwise they double the HBM weight traffic.
    // Two chains run while a layer is at most a third of the L2. On an H100 80GB HBM3 (50 MB L2; both settings alternated twice in
    // one run) one chain is faster for GPT-L (27 MB per layer, c2i 256 px, B = 64: 431 vs 469 ms/step) and GPT-XL (39 MB, 384 px,
    // B = 32: 1659 vs 1849 ms/step).
    // LG_SPLIT forces the chain count.
    const double layer_bytes = (4.0 * e->cfg.dim * e->cfg.dim + 3.0 * e->cfg.dim * e->cfg.ffn_dim) * e->esz;
    int l2_bytes = 0, dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, dev) != cudaSuccess) l2_bytes = 0;
    int n = lg_env_flag("LG_SPLIT", 3.0 * layer_bytes <= (double)l2_bytes ? 2 : 1);
    if (n > lg_engine::kMaxChains) n = lg_engine::kMaxChains;
    while (n >= 2 && (rows % n != 0 || (rows / n) % 2 != 0 || rows / n < 16)) --n;
    if (n >= 2 && lg_dtype_is16(dt) && tmp.have_maps) {
        const lg_model_cfg& c = e->cfg;
        const int hr = rows / n;
        const int Tc = c.model_type == LG_MODEL_T2I ? c.cls_token_num : 1;
        const size_t Mh = (size_t)hr * Tc, esz = e->esz;
        Workspace probe;
        e->carve(probe, nullptr, hr, max_seq);
        const size_t pf_full = tmp.partial_floats, pf_part = probe.partial_floats;
        const size_t pf_slot = pf_full / n / 64 * 64;
        if (pf_part <= pf_slot) {
            for (int g = 0; g < n; ++g) {
                Workspace w = tmp;
                w.rows = hr;
                w.layer_cache_bytes = (size_t)hr * c.n_head * max_seq * e->hdp * e->kv_esz;
                w.kcache = tmp.kcache + (size_t)g * w.layer_cache_bytes * c.n_layer;
                w.vcache = tmp.vcache + (size_t)g * w.layer_cache_bytes * c.n_layer;
                w.h = tmp.h + (size_t)g * Mh * c.dim * esz;
                w.xn = tmp.xn + (size_t)g * Mh * c.dim * esz;
                w.q = tmp.q + (size_t)g * Mh * c.dim * esz;
                w.attn = tmp.attn + (size_t)g * Mh * c.dim * esz;
                w.ff = tmp.ff + (size_t)g * Mh * c.ffn_dim * esz;
                w.x0 = tmp.x0 ? tmp.x0 + (size_t)g * Mh * c.caption_dim * esz : nullptr;
                w.partial = tmp.partial + (size_t)g * pf_slot;
                w.logits = tmp.logits + (size_t)g * hr * c.vocab_size;
                w.tokens = tmp.tokens + (size_t)g * hr;
                w.counters = tmp.counters + 2 * g;
                const long long total_rows = (long long)c.n_layer * hr * c.n_head * max_seq;
                LG_TRY(attn_tma_make_map(w.kmap, w.kcache, total_rows, e->hdp, kvdt));
                LG_TRY(attn_tma_make_map(w.vmap, w.vcache, total_rows, e->hdp, kvdt));
                LG_TRY(attn_tma_make_map(w.kmap16, w.kcache, total_rows, e->hdp, kvdt, 1));
                LG_TRY(attn_tma_make_map(w.vmap16, w.vcache, total_rows, e->hdp, kvdt, 1));
                w.have_maps = true;
                e->sub[g] = w;
            }
            e->n_sub = n;
        }
    }
    return 0;
}

// powers of two keep x / s exact and e4m3 * s exact in bf16 and fp16 (448 * 2^7 < 65504)
static bool kv_scale_ok(float s) {
    int ex = 0;
    return std::isfinite(s) && s > 0.f && std::frexp(s, &ex) == 0.5f && ex - 1 >= -8 && ex - 1 <= 7;
}

int lg_engine_set_kv_cache(lg_engine* e, int kv_dtype, const float* scales) {
    LG_REQUIRE(e, "lg_engine_set_kv_cache: null engine");
    const int dt = e->cfg.dtype;
    LG_REQUIRE(lg_dtype_is16(dt), "lg_engine_set_kv_cache: an fp8 KV cache needs a bf16 or fp16 model (model dtype %d)", dt);
    LG_REQUIRE(kv_dtype == dt || kv_dtype == LG_DTYPE_E4M3,
               "lg_engine_set_kv_cache: unsupported KV-cache dtype %d (LG_DTYPE_E4M3 or the model dtype %d)", kv_dtype, dt);
    std::vector<float> sc;
    if (kv_dtype == LG_DTYPE_E4M3) {
        sc.assign((size_t)2 * e->cfg.n_layer, 1.0f);
        for (size_t i = 0; scales && i < sc.size(); ++i) {
            const float s = scales[i];
            LG_REQUIRE(kv_scale_ok(s), "lg_engine_set_kv_cache: %s scale of layer %d is %g; scales must be powers of two in [2^-8, 2^7]",
                       i % 2 ? "V" : "K", (int)(i / 2), (double)s);
            sc[i] = s;
        }
    }
    // the carving and the tensor maps depend on the element size: the caller sets a new workspace
    e->kv_f8 = kv_dtype == LG_DTYPE_E4M3;
    e->kv_esz = e->kv_f8 ? 1 : e->esz;
    e->kv_scales = sc;
    e->full = Workspace();
    e->ws = Workspace();
    e->n_sub = 0;
    e->ws_needs_zero = false;
    return 0;
}

static int check_ready(lg_engine* e, int rows, int seq) {
    LG_REQUIRE(e && e->finalized, "engine not finalized");
    LG_REQUIRE(e->full.base, "workspace not set");
    e->ws = e->full;
    LG_REQUIRE(rows <= e->ws.rows, "rows %d exceed workspace rows %d", rows, e->ws.rows);
    LG_REQUIRE(seq <= e->ws.max_seq, "sequence %d exceeds workspace max_seq %d", seq, e->ws.max_seq);
    LG_REQUIRE(seq <= e->cfg.cls_token_num + e->cfg.block_size, "sequence %d exceeds the RoPE table (%d)", seq,
               e->cfg.cls_token_num + e->cfg.block_size);
    return 0;
}

// 16-bit engines: the head's logits are a bf16 / fp16 tensor in the reference (gpt.py:368 `.float()` of it); no-op for fp32
static int round_logits_inplace(float* logits, size_t n, int dtype, cudaStream_t st);

int lg_prefill(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int use_cfg, float* logits_out,
               void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int R = use_cfg ? 2 * B : B;
    LG_REQUIRE(e, "lg_prefill: null engine");
    DeviceGuard guard(e->device);
    LG_TRY(check_ready(e, R, T));
    LG_TRY(e->zero_fill_if_needed(st));
    LG_REQUIRE(cond && logits_out && B > 0, "lg_prefill: bad argument");
    LG_REQUIRE(T == e->cfg.cls_token_num, "lg_prefill: T=%d must equal cls_token_num=%d", T, e->cfg.cls_token_num);
    LG_TRY(e->embed_cond(cond, B, R, T, st));
    PosArg pos{nullptr, 0};
    LG_TRY(e->forward(R * T, T, pos, emb_mask, B, logits_out, false, st));
    LG_TRY(round_logits_inplace(logits_out, (size_t)R * e->cfg.vocab_size, e->cfg.dtype, st));
    return 0;
}

int lg_decode_step(lg_engine* e, const int32_t* tokens, int B, int pos, int use_cfg, float* logits_out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int R = use_cfg ? 2 * B : B;
    LG_REQUIRE(e, "lg_decode_step: null engine");
    DeviceGuard guard(e->device);
    LG_TRY(check_ready(e, R, pos + 1));
    LG_TRY(e->zero_fill_if_needed(st));
    LG_REQUIRE(tokens && logits_out && B > 0 && pos >= 0, "lg_decode_step: bad argument");
    LG_TRY(launch_embed(e->tok_emb, tokens, B, R, -1, e->cfg.dim, e->cfg.dtype, e->ws.h, st));
    PosArg p{nullptr, pos};
    LG_TRY(e->forward(R, 1, p, nullptr, B, logits_out, false, st));
    LG_TRY(round_logits_inplace(logits_out, (size_t)R * e->cfg.vocab_size, e->cfg.dtype, st));
    return 0;
}

int lg_decode_rows(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, int B, int use_cfg, float* logits_out, void* stream) {
    // Iteration-level scheduling (serve/llm_engine.py:511 step()): one forward for R rows that sit at DIFFERENT depths. A row at
    // position 0 is a request that has just joined: it takes its class embedding (the c2i "prefill" is that single position).
    cudaStream_t st = (cudaStream_t)stream;
    const int R = use_cfg ? 2 * B : B;
    LG_REQUIRE(e, "lg_decode_rows: null engine");
    DeviceGuard guard(e->device);
    LG_TRY(check_ready(e, R, 1));
    LG_TRY(e->zero_fill_if_needed(st));
    LG_REQUIRE(tokens && pos_rows && logits_out && B > 0, "lg_decode_rows: bad argument");
    LG_REQUIRE(e->cfg.model_type == LG_MODEL_C2I && e->cfg.cls_token_num == 1, "lg_decode_rows: class-conditional models only");
    LG_TRY(launch_embed_rows(e->cls_table, e->tok_emb, tokens, pos_rows, B, R, e->cfg.num_classes, e->cfg.dim, e->cfg.dtype, e->ws.h, st));
    PosArg p{nullptr, 0, pos_rows};
    LG_TRY(e->forward(R, 1, p, nullptr, B, logits_out, false, st));
    LG_TRY(round_logits_inplace(logits_out, (size_t)R * e->cfg.vocab_size, e->cfg.dtype, st));
    return 0;
}

int lg_sample_rows(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                   const int32_t* step_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream) {
    LG_REQUIRE(logits && sc && seed_rows && step_rows && (out_idx || out_seq), "lg_sample_rows: null argument");
    SampleArgs a{};
    a.logits = logits; a.B = B; a.V = V; a.mix_cfg = mix_cfg; a.round_dtype = lg_dtype_is16(round_dtype) ? round_dtype : LG_DTYPE_F32;
    a.cfg_scale = sc->cfg_scale; a.cfg_interval = sc->cfg_interval; a.temperature = sc->temperature;
    a.top_k = sc->top_k; a.top_p = sc->top_p; a.greedy = sc->greedy; a.seed = sc->seed; a.step = 0;
    a.seed_rows = seed_rows; a.step_rows = step_rows;
    a.out_idx = out_idx; a.out_seq = out_seq; a.seq_stride = seq_stride;
    return launch_sample(a, (cudaStream_t)stream);
}

int lg_sample(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, uint64_t step,
              int32_t* out_idx, float* out_probs, void* stream) {
    LG_REQUIRE(logits && sc && out_idx, "lg_sample: null argument");
    SampleArgs a{};
    a.logits = logits; a.B = B; a.V = V; a.mix_cfg = mix_cfg; a.round_dtype = lg_dtype_is16(round_dtype) ? round_dtype : LG_DTYPE_F32;
    a.cfg_scale = sc->cfg_scale; a.cfg_interval = sc->cfg_interval; a.temperature = sc->temperature;
    a.top_k = sc->top_k; a.top_p = sc->top_p; a.greedy = sc->greedy; a.seed = sc->seed; a.step = step;
    a.out_idx = out_idx; a.out_probs = out_probs;
    return launch_sample(a, (cudaStream_t)stream);
}

static int generate_impl(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S,
                         const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher,
                         cudaStream_t st);

int lg_generate(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc,
                int32_t* out_tokens, float* dbg_logits, const int32_t* teacher, void* stream) {
    // The loop runs on engine-owned non-blocking streams forked from / joined to the caller's stream with
    // events: the caller's stream may be the legacy default stream (torch's default), which cannot be captured
    // into a CUDA graph. Semantics for the caller stay "asynchronous on the given stream".
    cudaStream_t caller = (cudaStream_t)stream;
    LG_REQUIRE(e, "lg_generate: null engine");
    DeviceGuard guard(e->device);
    if (!e->works[0]) {
        // highest priority: when the VQ decode of the previous batch runs beside the sampler (pipeline.py), a freed SM slot goes to the
        // sampler's short dependent kernels first
        int prio_lo = 0, prio_hi = 0;
        LG_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        for (int i = 0; i < lg_engine::kMaxChains; ++i) {
            LG_CUDA_OK(cudaStreamCreateWithPriority(&e->works[i], cudaStreamNonBlocking, prio_hi));
            LG_CUDA_OK(cudaEventCreateWithFlags(&e->ev_joins[i], cudaEventDisableTiming));
        }
        LG_CUDA_OK(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
    }
    LG_TRY(e->zero_fill_if_needed(caller));
    LG_CUDA_OK(cudaEventRecord(e->ev_fork, caller));
    for (int i = 0; i < lg_engine::kMaxChains; ++i) LG_CUDA_OK(cudaStreamWaitEvent(e->works[i], e->ev_fork, 0));
    const int rc = generate_impl(e, cond, emb_mask, B, T, S, sc, out_tokens, dbg_logits, teacher, e->works[0]);
    for (int i = 0; i < lg_engine::kMaxChains; ++i) {
        cudaEventRecord(e->ev_joins[i], e->works[i]);
        cudaStreamWaitEvent(caller, e->ev_joins[i], 0);
    }
    if (e->full.base) e->ws = e->full;
    return rc;
}

namespace {
// One independent decode chain (a contiguous group of images with its own workspace half, stream and graph).
struct Chain {
    Workspace w;
    cudaStream_t st = nullptr;
    const void* cond = nullptr;
    const float* emb_mask = nullptr;
    int B = 0, R = 0;
    SampleArgs sa{};
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    uint64_t per_step = 0;
};
}  // namespace

static int generate_impl(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S,
                         const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher,
                         cudaStream_t st0) {
    LG_REQUIRE(cond && sc && out_tokens && B > 0 && S > 0, "lg_generate: bad argument");
    const bool use_cfg = sc->cfg_scale > 1.0f;  // generate.py:128
    const int R = use_cfg ? 2 * B : B;
    LG_TRY(check_ready(e, R, T + S));
    LG_REQUIRE(T == e->cfg.cls_token_num, "lg_generate: T=%d must equal cls_token_num=%d", T, e->cfg.cls_token_num);
    if (emb_mask) LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "emb_masks only apply to t2i models");
    const lg_model_cfg& c = e->cfg;

    // Multi-chain decode: at large batch every kernel of a decode step is latency-bound (a few microseconds of
    // dependent load -> compute -> store), so the batch is cut into n_sub independent chains (the chain-count policy of
    // lg_engine_set_workspace, which LG_SPLIT overrides; each chain has its own KV-cache slice, stream and CUDA graph) whose kernels interleave on the GPU. Each image's arithmetic is unchanged, so the result
    // is bit-identical to the single-chain run.
    const bool split = e->n_sub >= 2 && lg_env_flag("LG_SPLIT", 2) >= 2 && R == e->full.rows && B % e->n_sub == 0 &&
                       !prof_enabled() && !lg_debug_sync();
    const int nchains = split ? e->n_sub : 1;
    Chain ch[lg_engine::kMaxChains];
    for (int g = 0; g < nchains; ++g) {
        Chain& k = ch[g];
        k.w = split ? e->sub[g] : e->full;
        k.st = g == 0 ? st0 : e->works[g];
        k.B = B / nchains;
        k.R = R / nchains;
        const size_t boff = (size_t)g * k.B;
        k.cond = c.model_type == LG_MODEL_C2I ? (const void*)((const int32_t*)cond + boff)
                                              : (const void*)((const char*)cond + boff * T * c.caption_dim * e->esz);
        k.emb_mask = emb_mask ? emb_mask + boff * T : nullptr;
        SampleArgs& sa = k.sa;
        sa.logits = k.w.logits; sa.B = k.B; sa.V = c.vocab_size; sa.mix_cfg = use_cfg;
        sa.round_dtype = c.dtype;   // LG_DTYPE_F32 (0): no rounding
        sa.cfg_scale = sc->cfg_scale; sa.cfg_interval = sc->cfg_interval; sa.temperature = sc->temperature;
        sa.top_k = sc->top_k; sa.top_p = sc->top_p; sa.greedy = sc->greedy; sa.seed = sc->seed;
        sa.row_offset = (int)boff;
        sa.out_seq = out_tokens + boff * S; sa.seq_stride = S; sa.next_tokens = k.w.tokens;
        sa.teacher = teacher ? teacher + boff * S : nullptr;
        sa.dbg_logits = dbg_logits; sa.dbg_batch = B;
    }

    // Fused tail (bf16 / fp16): the sample kernel writes the next step's input rows (token embedding, and on the batched path the layer-0
    // RMSNorm) and advances the device-resident counters, so a decode iteration loses its embed / rmsnorm / advance kernels.
    const bool fuse_tail = lg_dtype_is16(c.dtype) && lg_env_flag("LG_FUSE_TAIL", 1) && c.dim % 2 == 0;
    auto arm_tail = [&](Chain& k, bool advance) {
        SampleArgs& sa = k.sa;
        e->ws = k.w;
        AttnArgs aa{};
        aa.R = k.R; aa.Tq = 1; aa.H = c.n_head; aa.hd = e->hd; aa.hdp = e->hdp; aa.dtype = c.dtype;
        if (k.w.have_maps) { aa.kmap = k.w.kmap; aa.vmap = k.w.vmap; aa.kmap16 = k.w.kmap16; aa.vmap16 = k.w.vmap16; }
        const bool small = e->small_row_path(k.R, aa);
        sa.emb_table = e->tok_emb; sa.emb_h = k.w.h; sa.emb_D = c.dim; sa.emb_rows = k.R;
        sa.emb_xn = small ? nullptr : k.w.xn;
        sa.emb_norm_w = e->layers[0].attn_norm; sa.emb_eps = c.norm_eps;
        sa.adv_pos = advance ? k.w.counters : nullptr;
        sa.adv_step = advance ? k.w.counters + 1 : nullptr;
        sa.adv_ticket = advance ? reinterpret_cast<unsigned int*>(k.w.counters + 64) : nullptr;
    };
    auto body = [&](Chain& k) -> int {
        e->ws = k.w;
        int* d_pos = k.w.counters;
        int* d_step = k.w.counters + 1;
        if (fuse_tail) {
            e->skip_first_norm = k.sa.emb_xn != nullptr;     // the previous iteration's sample kernel left h (and xn) in place
        } else {
            LG_PROF(PC_EMBED_MISC, k.st, launch_embed(e->tok_emb, k.w.tokens, k.B, k.R, -1, c.dim, c.dtype, k.w.h, k.st));
        }
        LG_TRY(e->forward(k.R, 1, PosArg{d_pos, 0}, k.emb_mask, k.B, k.w.logits, false, k.st));
        LG_PROF(PC_SAMPLE, k.st, launch_sample(k.sa, k.st));
        if (!fuse_tail) LG_PROF(PC_EMBED_MISC, k.st, launch_advance(d_pos, d_step, k.st));
        return 0;
    };

    // ---- prefill (generate.py:167-169) + first decode step, eagerly, per chain
    for (int g = 0; g < nchains; ++g) {
        Chain& k = ch[g];
        e->ws = k.w;
        LG_TRY(e->embed_cond(k.cond, k.B, k.R, T, k.st));
        LG_TRY(e->forward(k.R * T, T, PosArg{nullptr, 0}, k.emb_mask, k.B, k.w.logits, false, k.st));
        k.sa.step = 0; k.sa.step_dev = nullptr;
        const bool tail = S > 1 && fuse_tail;
        if (tail) arm_tail(k, false);            // the prefill's sample prepares the first decode step's rows; counters are set below
        LG_TRY(launch_sample(k.sa, k.st));
        if (S == 1) continue;
        LG_TRY(launch_set_counters(k.w.counters, T, k.w.counters + 1, 1, k.st));
        k.sa.step_dev = k.w.counters + 1;
        if (tail) arm_tail(k, true);
        LG_TRY(body(k));   // first decode step runs eagerly (also sets every kernel attribute outside capture)
    }
    const int remaining = S - 2;
    if (remaining <= 0) return 0;
    if (!e->use_graph || remaining < 3 || prof_enabled() || lg_debug_sync()) {
        for (int i = 0; i < remaining; ++i)
            for (int g = 0; g < nchains; ++g) LG_TRY(body(ch[g]));
        return 0;
    }
    // ---- decode loop (generate.py:105-123): per chain one captured graph of one decode step (the loop state is
    // device-resident, so every step has identical kernel arguments), replayed, chains interleaved: with two chains the
    // gap between graph launches of one chain is covered by the other chain's kernels.
    int ret = 0;
    auto capture = [&](Chain& k, cudaGraph_t* graph, cudaGraphExec_t* exec, uint64_t* launches) -> int {
        cudaError_t ce = cudaStreamBeginCapture(k.st, cudaStreamCaptureModeRelaxed);
        if (ce != cudaSuccess) return lg_fail("cudaStreamBeginCapture failed: %s", cudaGetErrorString(ce));
        const uint64_t before = g_lg_launches.load();
        const int rc = body(k);
        *launches = g_lg_launches.load() - before;
        ce = cudaStreamEndCapture(k.st, graph);
        g_lg_launches.fetch_sub(*launches);  // the capture pass launched nothing
        if (rc < 0) return rc;
        if (ce != cudaSuccess || !*graph) return lg_fail("stream capture failed: %s", cudaGetErrorString(ce));
        ce = cudaGraphInstantiate(exec, *graph, 0);
        if (ce != cudaSuccess) return lg_fail("cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
        return 0;
    };
    for (int g = 0; g < nchains && ret == 0; ++g) ret = capture(ch[g], &ch[g].graph, &ch[g].exec, &ch[g].per_step);
    for (int i = 0; i < remaining && ret == 0; ++i) {
        for (int g = 0; g < nchains; ++g) {
            const cudaError_t ce = cudaGraphLaunch(ch[g].exec, ch[g].st);
            if (ce != cudaSuccess) { ret = lg_fail("cudaGraphLaunch failed: %s", cudaGetErrorString(ce)); break; }
            g_lg_launches.fetch_add(ch[g].per_step);
        }
    }
    for (int g = 0; g < nchains; ++g) {
        if (ch[g].exec) cudaGraphExecDestroy(ch[g].exec);
        if (ch[g].graph) cudaGraphDestroy(ch[g].graph);
    }
    return ret;
}

int lg_vq_set_cta_budget(int ctas) {
    conv_tc_set_cta_budget(ctas < 0 ? 0 : ctas);
    return 0;
}
int lg_set_pdl(int on) {
    g_lg_pdl = on ? 1 : 0;
    return 0;
}
int lg_profile_enable(int on) {
    if (!on) prof_drain();
    g_prof.on = on != 0;
    return 0;
}
int lg_profile_reset(void) {
    prof_drain();
    for (int i = 0; i < PC_COUNT; ++i) { g_prof.total_ms[i] = 0; g_prof.count[i] = 0; }
    return 0;
}
int lg_profile_read(int cls, double* total_ms, uint64_t* launches) {
    LG_REQUIRE(cls >= 0 && cls < PC_COUNT && total_ms && launches, "lg_profile_read: bad argument");
    prof_drain();
    *total_ms = g_prof.total_ms[cls];
    *launches = g_prof.count[cls];
    return 0;
}
const char* lg_profile_class_name(int cls) {
    static const char* names[PC_COUNT] = {"gemm_qkv", "qkv_rope_kvwrite", "attention", "gemm_wo", "residual_rmsnorm",
                                          "gemm_w13", "silu_mul", "gemm_w2", "gemm_head", "sample", "embed_misc",
                                          "vq_conv_gemm", "vq_gn_stats", "vq_gn_apply", "vq_attn", "vq_misc"};
    return (cls >= 0 && cls < PC_COUNT) ? names[cls] : nullptr;
}

int lg_test_gemm(const void* x, const void* w, int M, int N, int K, int dtype, float* y, void* dev_scratch,
                 size_t scratch_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(x && w && y && dev_scratch, "lg_test_gemm: null argument");
    const size_t needf = gemm_partial_floats(M, N, K, dtype);
    LG_REQUIRE(scratch_bytes >= needf * sizeof(float), "lg_test_gemm: scratch %zu < %zu", scratch_bytes, needf * sizeof(float));
    GemmPlan plan;
    LG_TRY(gemm_partial(x, K, w, nullptr, 0, M, N, K, dtype, (float*)dev_scratch, &plan, st));
    return launch_reduce_f32((const float*)dev_scratch, plan.ksplit, M, N, y, st);
}

int lg_test_attention(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                      void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                      const int32_t* pos_rows, const float* emb_mask, int B, int Tc, const void* q, const float* qkv_partial,
                      int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    auto a16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    const bool f8 = kv_dtype == LG_DTYPE_E4M3;
    LG_REQUIRE(dtype == LG_DTYPE_F32 || lg_dtype_is16(dtype), "lg_test_attention: unsupported model dtype %d", dtype);
    LG_REQUIRE(kv_dtype == dtype || (f8 && lg_dtype_is16(dtype)),
               "lg_test_attention: KV dtype %d with model dtype %d (the model dtype, or LG_DTYPE_E4M3 for a bf16 / fp16 model)", kv_dtype,
               dtype);
    LG_REQUIRE(f8 ? kv_scale_ok(k_scale) && kv_scale_ok(v_scale) : k_scale == 1.f && v_scale == 1.f,
               "lg_test_attention: K / V scales %g / %g (fp8: powers of two in [2^-8, 2^7], otherwise 1)", (double)k_scale, (double)v_scale);
    LG_REQUIRE(R > 0 && Tq > 0 && H > 0 && max_seq > 0 && n_layer > 0 && layer >= 0 && layer < n_layer && (long long)R * Tq <= 65535,
               "lg_test_attention: bad shape R=%d Tq=%d H=%d max_seq=%d layer %d of %d", R, Tq, H, max_seq, layer, n_layer);
    LG_REQUIRE(hd == 64 || hd == 100 || hd == 128, "lg_test_attention: unsupported head_dim %d (64, 100, 128)", hd);
    LG_REQUIRE(hdp == attn_kv_row_width(dtype, hd), "lg_test_attention: row width %d for head_dim %d", hdp, hd);
    LG_REQUIRE(kcache && vcache && out && a16(kcache) && a16(vcache) && a16(out) && a16(q) && a16(q_out) && a16(qkv_partial) && a16(freqs),
               "lg_test_attention: null or misaligned (16 bytes) buffer");
    if (pos_rows) {
        LG_REQUIRE(pos_dev == nullptr && pos_value == 0, "lg_test_attention: per-row positions take no counter and no value");
    } else {
        LG_REQUIRE(pos_value >= 0 && (pos_dev || pos_value + Tq <= max_seq), "lg_test_attention: position %d + Tq %d exceeds max_seq %d",
                   pos_value, Tq, max_seq);
    }
    LG_REQUIRE(!emb_mask || (B > 0 && Tc > 0 && Tc <= max_seq), "lg_test_attention: emb_mask needs B > 0 and 0 < Tc <= max_seq (B=%d Tc=%d)",
               B, Tc);
    LG_REQUIRE((q != nullptr) != (qkv_partial != nullptr), "lg_test_attention: pass exactly one of q and qkv_partial");
    LG_REQUIRE(q ? fuse == 0 : (ksplit > 0 && freqs && (fuse == 1 || (fuse == 0 && q_out))),
               "lg_test_attention: q takes fuse = 0; qkv_partial needs ksplit > 0, freqs and fuse = 1 or q_out");
    const long long total_rows = (long long)n_layer * R * H * max_seq;
    const size_t layer_bytes = (size_t)R * H * max_seq * hdp * (f8 ? 1 : lg_dtype_info(dtype).esz);
    AttnArgs aa;
    aa.q = q ? q : q_out; aa.out = out;
    aa.kcache = (char*)kcache + (size_t)layer * layer_bytes; aa.vcache = (char*)vcache + (size_t)layer * layer_bytes;
    aa.R = R; aa.Tq = Tq; aa.H = H; aa.hd = hd; aa.maxS = max_seq; aa.hdp = hdp;
    aa.pos = PosArg{pos_dev, pos_value, pos_rows};
    aa.emb_mask = emb_mask; aa.B = emb_mask ? B : 1; aa.Tc = emb_mask ? Tc : 0;
    aa.scale = 1.0f / sqrtf((float)hd); aa.dtype = dtype;
    if (f8) { aa.kv_f8 = 1; aa.scale *= k_scale; aa.k_inv = 1.0f / k_scale; aa.v_inv = 1.0f / v_scale; aa.v_scale = v_scale; }
    alignas(64) unsigned char maps[4][128];   // as lg_engine_set_workspace builds them: over every layer of the buffer
    if (attn_tma_maps_usable(dtype, hd, hdp, total_rows)) {
        const int kvdt = f8 ? LG_DTYPE_E4M3 : dtype;
        LG_TRY(attn_tma_make_map(maps[0], kcache, total_rows, hdp, kvdt));
        LG_TRY(attn_tma_make_map(maps[1], vcache, total_rows, hdp, kvdt));
        LG_TRY(attn_tma_make_map(maps[2], kcache, total_rows, hdp, kvdt, 1));
        LG_TRY(attn_tma_make_map(maps[3], vcache, total_rows, hdp, kvdt, 1));
        aa.kmap = maps[0]; aa.vmap = maps[1]; aa.kmap16 = maps[2]; aa.vmap16 = maps[3];
        aa.cache_row_base = (long long)layer * R * H * max_seq;
    }
    if (qkv_partial) {
        if (fuse) {
            LG_REQUIRE(attn_tma_enabled() && attn_tma_supported(aa), "lg_test_attention: the fused QKV epilogue needs the TMA decode kernel");
            aa.qkv_partial = qkv_partial; aa.qkv_ksplit = ksplit; aa.freqs = freqs;
        } else {
            QkvEpiArgs qa;
            qa.partial = qkv_partial; qa.ksplit = ksplit; qa.M = R * Tq; qa.Tq = Tq; qa.D = H * hd; qa.H = H; qa.hd = hd;
            qa.pos = aa.pos; qa.freqs = freqs; qa.q = q_out; qa.kcache = const_cast<void*>(aa.kcache); qa.vcache = const_cast<void*>(aa.vcache);
            qa.maxS = max_seq; qa.dtype = dtype; qa.hdp = hdp;
            qa.kv_f8 = aa.kv_f8; qa.k_inv = aa.k_inv; qa.v_inv = aa.v_inv;
            LG_TRY(launch_qkv_epilogue(qa, st));
        }
    }
    return launch_attention(aa, st, path);
}

}  // extern "C"

namespace {
__global__ void round_bf16_kernel(float* p, size_t n) {
    lg_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        p[i] = round_bf16(p[i]);
}
__global__ void round_f16_kernel(float* p, size_t n) {
    lg_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        p[i] = ElemTraits<f16>::round(p[i]);   // past +-65504 -> +-inf, like torch's fp16 head
}
}  // namespace
static int round_logits_inplace(float* logits, size_t n, int dtype, cudaStream_t st) {
    if (!lg_dtype_is16(dtype)) return 0;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 132 * 8);
    (void)lg_launch(dtype == LG_DTYPE_F16 ? round_f16_kernel : round_bf16_kernel, dim3(blocks), dim3(256), 0, st, logits, n);
    LG_LAUNCH_CHECK();
    return 0;
}
