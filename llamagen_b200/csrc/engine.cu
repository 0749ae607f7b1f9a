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

constexpr int kCounterInts = 128;   // device loop state: pos / step of chain g at [2g, 2g+1], the sampler's ticket at 64 + 2g

// CUtensorMaps over a whole K and a whole V cache region: kKC-row boxes, and 16-row boxes for the tail chunk of the decode attention
struct alignas(64) KvMaps {
    unsigned char k[128], v[128], k16[128], v16[128];
    bool usable = false;   // built: a bf16 / fp16 cache the TMA attention kernels can stream (attn_tma_maps_usable)
};

// Fills `m` for a K / V cache pair of total_rows rows of hdp elements each, stored in kv_dtype, of a model in `dtype` with head_dim hd
int make_kv_maps(KvMaps& m, int dtype, int hd, int hdp, int kv_dtype, const void* kcache, const void* vcache, long long total_rows) {
    m.usable = attn_tma_maps_usable(dtype, hd, hdp, total_rows);
    if (!m.usable) return 0;
    LG_TRY(attn_tma_make_map(m.k, kcache, total_rows, hdp, kv_dtype));
    LG_TRY(attn_tma_make_map(m.v, vcache, total_rows, hdp, kv_dtype));
    LG_TRY(attn_tma_make_map(m.k16, kcache, total_rows, hdp, kv_dtype, 1));
    LG_TRY(attn_tma_make_map(m.v16, vcache, total_rows, hdp, kv_dtype, 1));
    return 0;
}

// One attention call over layer `layer` of a K / V cache pair laid out [layer][rows, H, max_seq, hdp] (DESIGN §3): the geometry, the
// softmax scale with an fp8 cache's scales folded in (kv_scales: this layer's {K, V} scales, null for a cache in the model dtype) and
// the tensor maps over the whole pair. The call's row r is cache row first_row + r: the cache pointers and the maps' first row move
// alike. The caller sets q, out, the positions and the emb-mask.
AttnArgs make_attn_args(int dtype, int H, int hd, int hdp, int rows, int max_seq, char* kcache, char* vcache, const KvMaps& maps,
                        const float* kv_scales, int layer, int R, int Tq, int first_row = 0) {
    AttnArgs aa{};
    const long long row0 = ((long long)layer * rows + first_row) * H * max_seq;
    const size_t row_bytes = (size_t)hdp * (kv_scales ? 1 : lg_dtype_info(dtype).esz);
    aa.kcache = kcache + (size_t)row0 * row_bytes; aa.vcache = vcache + (size_t)row0 * row_bytes;
    aa.R = R; aa.Tq = Tq; aa.H = H; aa.hd = hd; aa.hdp = hdp; aa.maxS = max_seq; aa.dtype = dtype;
    aa.scale = 1.0f / sqrtf((float)hd);
    if (kv_scales) {   // the K scale folds into the softmax scale, the V scale into O / L, the writers divide by them
        const float ks = kv_scales[0], vs = kv_scales[1];
        aa.kv_f8 = 1; aa.scale *= ks; aa.k_inv = 1.0f / ks; aa.v_inv = 1.0f / vs; aa.v_scale = vs;
    }
    if (maps.usable) {
        aa.kmap = maps.k; aa.vmap = maps.v; aa.kmap16 = maps.k16; aa.vmap16 = maps.v16;
        aa.cache_row_base = row0;
    }
    return aa;
}

// The separate QKV epilogue that writes q and the K / V rows `aa` attends over, from the QKV GEMM's split-K slabs
QkvEpiArgs make_qkv_epi_args(const AttnArgs& aa, const float* partial, int ksplit, const float* freqs) {
    QkvEpiArgs qa;
    qa.partial = partial; qa.ksplit = ksplit; qa.M = aa.R * aa.Tq; qa.Tq = aa.Tq; qa.D = aa.H * aa.hd; qa.H = aa.H; qa.hd = aa.hd;
    qa.pos = aa.pos; qa.freqs = freqs; qa.q = const_cast<void*>(aa.q);
    qa.kcache = const_cast<void*>(aa.kcache); qa.vcache = const_cast<void*>(aa.vcache);
    qa.maxS = aa.maxS; qa.dtype = aa.dtype; qa.hdp = aa.hdp;
    qa.kv_f8 = aa.kv_f8; qa.k_inv = aa.k_inv; qa.v_inv = aa.v_inv;
    return qa;
}

// Whether the attention kernel of `aa` (a call without QKV slabs) is also its QKV epilogue, one dependent kernel less: decode steps
// that run on the TMA decode kernel
bool fuse_qkv(const AttnArgs& aa) { return lg_env_flag("LG_FUSE_QKV", 1) && attn_plan(aa).kernel == 1; }

SampleArgs make_sample_args(const lg_sample_cfg& sc, const float* logits, int B, int V, int mix_cfg, int round_dtype) {
    SampleArgs a{};
    a.logits = logits; a.B = B; a.V = V; a.mix_cfg = mix_cfg; a.round_dtype = lg_dtype_is16(round_dtype) ? round_dtype : LG_DTYPE_F32;
    a.cfg_scale = sc.cfg_scale; a.cfg_interval = sc.cfg_interval; a.temperature = sc.temperature;
    a.top_k = sc.top_k; a.top_p = sc.top_p; a.greedy = sc.greedy; a.seed = sc.seed;
    a.temp_rows = sc.temperature_rows; a.topk_rows = sc.top_k_rows; a.topp_rows = sc.top_p_rows; a.greedy_rows = sc.greedy_rows;
    return a;
}

// A K / V cache pair laid out [layer][rows, H, max_seq, hdp] (DESIGN §3) and its tensor maps
struct KvCache {
    char *kcache = nullptr, *vcache = nullptr;
    size_t cache_bytes = 0;   // the K and V regions together, from kcache on (what the first use zero-fills)
    int rows = 0, max_seq = 0;
    int layers = 0;           // n_layer, or 1 for a cache that every layer rewrites before its attention reads it
    bool kv_f8 = false;       // e4m3 with the engine's per-layer scales, else the model dtype
    int first_row = 0;        // attention row 0 of a forward through this view is this cache row (a chunk of a prefix prefill)
    KvMaps maps;
};

// The activations, GEMM split-K partials and logits of a forward pass
struct RowBuffers {
    char *h = nullptr, *xn = nullptr, *q = nullptr, *attn = nullptr, *ff = nullptr, *x0 = nullptr;
    float *partial = nullptr, *logits = nullptr;
    size_t partial_floats = 0;
};

// The workspace (lg_engine::carve), one decode chain's view of it, or a scratch view (lg_score, lg_generate_sjd)
struct Workspace : KvCache, RowBuffers {
    char* base = nullptr;     // start of the whole workspace
    int32_t* tokens = nullptr;
    int* counters = nullptr;  // [0] = pos, [1] = step, [64] = the fused sampler tail's ticket
    int head_rows = 0;        // lg_score: rows per head GEMM
};

// The class of a scratch region (lg_test_scratch_regions): float or 16-bit data, int32 / uint64 state, KV cache
enum RegionClass { kRegionData = 0, kRegionInt = 1, kRegionKv = 2 };

// lg_test_scratch_regions' log of the regions carved while it is set: {offset, bytes, class, chain} per region, offsets from the
// scratch's start (`shift` is added: a layout carved from a point inside the scratch)
struct RegionLog {
    std::vector<int64_t> rows;
    size_t shift = 0;
    int chain = -1;   // >= 0: the chain of every region logged (one chain's layout carved on its own), else the carver's g
};
thread_local RegionLog* t_region_log = nullptr;

// Bump allocator over a workspace from `base` (null: sizes only), 256-byte aligned regions, for chain g of n
struct Carver {
    char* base;
    int g = 0, n = 1;
    size_t off = 0;
    // a region of `bytes`, of which chain g takes the part from g * chain_stride on (chain_stride bytes of it with n > 1; `used` bytes
    // of it with n = 1, when less than the whole region is ever used)
    char* shared(size_t bytes, size_t chain_stride, int cls = kRegionData, size_t used = SIZE_MAX) {
        char* p = base ? base + off + g * chain_stride : nullptr;
        if (t_region_log)
            t_region_log->rows.insert(t_region_log->rows.end(), {(int64_t)(t_region_log->shift + off + g * chain_stride),
                                                                 (int64_t)(n > 1 ? chain_stride : std::min(bytes, used)), cls,
                                                                 t_region_log->chain >= 0 ? t_region_log->chain : g});
        off += align_up(bytes);
        return p;
    }
    // a region that scales with rows: chain g takes its g-th n-th
    char* split(size_t bytes, int cls = kRegionData) { return shared(bytes, bytes / n, cls); }
};

// A captured CUDA graph of one stream's work and its executable graph
struct Graph {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    uint64_t launches = 0;    // kernel launches per replay
    Graph() = default;
    Graph(const Graph&) = delete;
    Graph& operator=(const Graph&) = delete;
    ~Graph() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
    }
    template <class Body>
    int capture(cudaStream_t st, Body&& body) {
        cudaError_t ce = cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed);
        if (ce != cudaSuccess) return lg_fail("cudaStreamBeginCapture failed: %s", cudaGetErrorString(ce));
        const uint64_t before = g_lg_launches.load();
        const int rc = body();
        launches = g_lg_launches.load() - before;
        ce = cudaStreamEndCapture(st, &graph);
        g_lg_launches.fetch_sub(launches);   // the capture pass launched nothing
        if (rc < 0) return rc;
        if (ce != cudaSuccess || !graph) return lg_fail("stream capture failed: %s", cudaGetErrorString(ce));
        ce = cudaGraphInstantiate(&exec, graph, 0);
        if (ce != cudaSuccess) return lg_fail("cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
        return 0;
    }
    int launch(cudaStream_t st) {
        const cudaError_t ce = cudaGraphLaunch(exec, st);
        if (ce != cudaSuccess) return lg_fail("cudaGraphLaunch failed: %s", cudaGetErrorString(ce));
        g_lg_launches.fetch_add(launches);
        return 0;
    }
};

// A negative prompt of the *_neg entry points: the condition of the unconditional CFG rows, cond [B, T, caption_dim] in the model
// dtype (one per image), and their emb-mask [B, T] (null: the rows read emb_mask's, as without a negative). cond null: the null
// condition uncond_embedding, today's unconditional rows.
struct Negative {
    const void* cond = nullptr;
    const float* mask = nullptr;
};

struct Layer {
    GemmWeight wqkv, wo, w1, w3, w2;   // each in the model dtype or fp8 (w1 and w3 alike: one GEMM streams both)
    const void *attn_norm, *ffn_norm;
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
    std::vector<float> kv_scales;         // [n_layer][2] (fp8 only)
    std::unordered_map<std::string, Tensor> w;
    std::vector<Layer> layers;
    const void *tok_emb = nullptr, *cls_table = nullptr, *cap_fc1 = nullptr, *cap_fc2 = nullptr, *uncond = nullptr;
    const void* final_norm = nullptr;
    GemmWeight output;
    size_t layer_weight_bytes = 0;        // GEMM weight bytes of the largest layer as bound (the chain-count policy's measure)
    const float* freqs = nullptr;
    bool finalized = false;
    static constexpr int kMaxChains = 2;   // carve_rows' chain slices are exact while every chain count divides this
    Workspace full, sub[kMaxChains];      // sub[g]: chain g's view of `full` (multi-chain decode)
    int n_sub = 0;                        // 0: no split available
    bool use_graph = true;
    bool ws_needs_zero = false;           // KV cache + counters of `full` still have to be zero-filled (done on the caller's stream)
    cudaStream_t works[kMaxChains] = {};   // engine-owned streams (one per chain)
    cudaEvent_t ev_fork = nullptr, ev_joins[kMaxChains] = {};
    cudaEvent_t ev_prefill = nullptr;     // lg_generate_prefix: every chain's prefill (one scratch) is done
    int prefix_chunks = 0;                // chunks the last lg_generate_prefix ran its prefill in (lg_test_prefix_chunks)
    int prefix_chains = 0;                // decode chains of that call
    int* sjd_done_host = nullptr;         // pinned copy of lg_generate_sjd's done flag
    cudaEvent_t ev_pass[2] = {};
    int32_t* given_host = nullptr;        // lg_generate_given's pinned staging of the head of its scratch (given_host_bytes)
    size_t given_host_bytes = 0;
    cudaEvent_t ev_given = nullptr;       // the last upload from given_host has been read
    // given_host with room for `bytes`, once the previous upload from it has read it
    int stage_given(size_t bytes) {
        if (!ev_given) LG_CUDA_OK(cudaEventCreateWithFlags(&ev_given, cudaEventDisableTiming));
        else LG_CUDA_OK(cudaEventSynchronize(ev_given));
        if (bytes <= given_host_bytes) return 0;
        if (given_host) LG_CUDA_OK(cudaFreeHost(given_host));
        given_host = nullptr;
        given_host_bytes = 0;
        LG_CUDA_OK(cudaHostAlloc((void**)&given_host, bytes, cudaHostAllocDefault));
        given_host_bytes = bytes;
        return 0;
    }
    ~lg_engine() {
        for (int i = 0; i < kMaxChains; ++i) {
            if (works[i]) cudaStreamDestroy(works[i]);
            if (ev_joins[i]) cudaEventDestroy(ev_joins[i]);
        }
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_prefill) cudaEventDestroy(ev_prefill);
        for (cudaEvent_t ev : ev_pass)
            if (ev) cudaEventDestroy(ev);
        if (sjd_done_host) cudaFreeHost(sjd_done_host);
        if (given_host) cudaFreeHost(given_host);
        if (ev_given) cudaEventDestroy(ev_given);
    }
    // the engine-owned streams the loops run on, created on first use
    int ensure_streams() {
        if (works[0]) return 0;
        // highest priority: when the VQ decode of the previous batch runs beside the sampler (pipeline.py), a freed SM slot goes to the
        // sampler's short dependent kernels first
        int prio_lo = 0, prio_hi = 0;
        LG_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
        for (int i = 0; i < kMaxChains; ++i) {
            LG_CUDA_OK(cudaStreamCreateWithPriority(&works[i], cudaStreamNonBlocking, prio_hi));
            LG_CUDA_OK(cudaEventCreateWithFlags(&ev_joins[i], cudaEventDisableTiming));
        }
        LG_CUDA_OK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        LG_CUDA_OK(cudaEventCreateWithFlags(&ev_prefill, cudaEventDisableTiming));
        return 0;
    }
    // Runs body(works[0]) with works[0..n) forked from and joined to the caller's stream by events: the caller's stream may be the
    // legacy default stream (torch's default), which cannot be captured into a CUDA graph. Semantics for the caller stay
    // "asynchronous on the given stream".
    template <class Body>
    int run_forked(cudaStream_t caller, int n, Body&& body) {
        LG_TRY(ensure_streams());
        LG_TRY(zero_fill_if_needed(caller));
        LG_CUDA_OK(cudaEventRecord(ev_fork, caller));
        for (int i = 0; i < n; ++i) LG_CUDA_OK(cudaStreamWaitEvent(works[i], ev_fork, 0));
        const int rc = body(works[0]);
        for (int i = 0; i < n; ++i) {
            cudaEventRecord(ev_joins[i], works[i]);
            cudaStreamWaitEvent(caller, ev_joins[i], 0);
        }
        return rc;
    }

    // R <= 8 decode steps on the column-owner GEMV path (gemv_small.cu); shared by forward() and the decode loop's fused tail
    bool small_row_path(int M, const AttnArgs& aa) const {
        const int D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size, dt = cfg.dtype;
        if (!(M <= 8 && lg_env_flag("LG_SMALL_R", 1) && fuse_qkv(aa) && gemv_small_supported(M, V, D, dt, false, output.scale != nullptr)))
            return false;
        for (const Layer& ly : layers)   // the storage of a weight is per layer
            if (!(gemv_small_supported(M, 3 * D, D, dt, false, ly.wqkv.scale != nullptr) &&
                  gemv_small_supported(M, D, D, dt, false, ly.wo.scale != nullptr) &&
                  gemv_small_supported(M, F, D, dt, true, ly.w1.scale != nullptr) &&
                  gemv_small_supported(M, D, F, dt, false, ly.w2.scale != nullptr)))
                return false;
        return true;
    }
    size_t carve(Workspace& o, char* base, int rows, int max_seq, int g = 0, int n = 1) const;
    size_t carve_score(Workspace& o, char* base, int rows, int seq) const;
    size_t carve_sjd(RowBuffers& o, SjdArgs& sa, char* base, int B, int nh, int L) const;
    size_t carve_sjd_slots(RowBuffers& o, SjdArgs& sa, char* base, int B, int nh, int L) const;
    size_t carve_prefix(RowBuffers& o, char* base, int rows, int seq) const;
    size_t carve_slot(RowBuffers& head, char* base, int nh, int seq) const;
    size_t carve_given_window(RowBuffers& o, int32_t** win, int32_t** pos_rows, char* base, int B, int nh, int W) const;
    void carve_kv(Carver& c, KvCache& o, int rows, int max_seq, int layers, bool f8) const;
    void carve_rows(Carver& c, RowBuffers& o, size_t M, size_t x0_rows, size_t partial_floats, size_t logits_rows, int chains = 1) const;
    // the most partial floats one of a layer's four GEMMs needs at M rows
    size_t layer_partial_floats(int M) const {
        const int D = cfg.dim, F = cfg.ffn_dim, dt = cfg.dtype;
        return std::max({gemm_partial_floats(M, 3 * D, D, 0, dt), gemm_partial_floats(M, D, D, 0, dt),
                         gemm_partial_floats(M, 2 * F, D, F, dt), gemm_partial_floats(M, D, F, 0, dt)});
    }
    // K / V tensor maps over every layer the cache holds
    int make_maps(KvCache& kv) const {
        return make_kv_maps(kv.maps, cfg.dtype, hd, hdp, kv.kv_f8 ? LG_DTYPE_E4M3 : cfg.dtype, kv.kcache, kv.vcache,
                            (long long)kv.layers * kv.rows * cfg.n_head * kv.max_seq);
    }
    AttnArgs attn_args(const KvCache& kv, int l, int R, int Tq) const {
        return make_attn_args(cfg.dtype, cfg.n_head, hd, hdp, kv.rows, kv.max_seq, kv.kcache, kv.vcache, kv.maps,
                              kv.kv_f8 ? &kv_scales[2 * l] : nullptr, l % kv.layers, R, Tq, kv.first_row);
    }
    AttnArgs layer_attn(const Workspace& w, int l, int R, int Tq, PosArg pos, const float* emb_mask, const float* neg_mask, int B) const {
        AttnArgs aa = attn_args(w, l, R, Tq);
        aa.q = w.q; aa.out = w.attn; aa.pos = pos; aa.emb_mask = emb_mask; aa.B = B; aa.Tc = cfg.cls_token_num;
        aa.emb_mask_uncond = neg_mask;
        return aa;
    }
    int zero_fill_if_needed(cudaStream_t st) {
        if (!ws_needs_zero || !full.base) return 0;
        LG_CUDA_OK(cudaMemsetAsync(full.kcache, 0, full.cache_bytes, st));
        LG_CUDA_OK(cudaMemsetAsync(full.counters, 0, kCounterInts * sizeof(int), st));
        ws_needs_zero = false;
        return 0;
    }
    // xn_ready: xn already holds RMSNorm_0(h) (the fused tail of the previous decode step's sample kernel wrote it). Rows r < B attend
    // with emb_mask, rows r >= B with neg_mask when it is set (a negative prompt's), else with emb_mask. pdl_first false: the first
    // kernel is launched without PDL (generate_impl's eager decode steps).
    int forward(const Workspace& w, int M, int Tq, PosArg pos, const float* emb_mask, const float* neg_mask, int B, float* logits_out,
                bool xn_ready, cudaStream_t st, bool pdl_first = true);
    // the transformer blocks over M = R * Tq rows of w.h, leaving RMSNorm_final(h) in w.xn (batched GEMM path)
    int run_layers(const Workspace& w, int M, int Tq, PosArg pos, const float* emb_mask, const float* neg_mask, int B, bool xn_ready,
                   cudaStream_t st, bool pdl_first = true);
    // the condition rows of R rows: rows r < B from cond, rows r >= B from neg_cond [R - B, T, C] (t2i) or the null condition
    int embed_cond(const Workspace& w, const void* cond, const void* neg_cond, int B, int R, int T, cudaStream_t st);
    int gemm(const Workspace& w, const void* x, int M, int N, int K, const GemmWeight& wa, const GemmWeight& wb, int n_split, int* ksplit,
             float* direct_out, cudaStream_t st, const GemmNext* next = nullptr, bool pdl = true);
    int head(const Workspace& w, const void* x, int M, float* logits_out, const GemmNext* next, cudaStream_t st);
};

// Lays out the workspace for `rows` rows and max_seq positions from `base` (null: sizes only) and returns its bytes. With n > 1, `o`
// becomes chain g's view of that same layout: the g-th n-th of every region that scales with rows (rows / n rows each), a 64-float
// aligned n-th of the GEMM partials, and the counters from 2g on.
size_t lg_engine::carve(Workspace& o, char* base, int rows, int max_seq, int g, int n) const {
    const int D = cfg.dim, V = cfg.vocab_size, dt = cfg.dtype;
    const bool t2i = cfg.model_type == LG_MODEL_T2I;
    const int Mmax = rows * (t2i ? cfg.cls_token_num : 1);
    size_t pf = gemm_partial_floats(rows, V, D, 0, dt);
    for (int M : {rows, Mmax}) {
        pf = std::max(pf, layer_partial_floats(M));
        if (t2i) pf = std::max(pf, gemm_partial_floats(M, D, cfg.caption_dim, 0, dt));
    }
    Carver c{base, g, n};
    carve_kv(c, o, rows, max_seq, cfg.n_layer, kv_f8);
    carve_rows(c, o, Mmax, t2i ? Mmax : 0, pf, rows, kMaxChains);
    o.tokens = (int32_t*)c.split((size_t)rows * sizeof(int32_t), kRegionInt);
    o.counters = (int*)c.shared(kCounterInts * sizeof(int), 2 * sizeof(int), kRegionInt);
    o.base = base;
    return c.off;
}

// K and V of `layers` layers of [rows, H, max_seq, hdp] elements, in e4m3 (f8) or the model dtype
void lg_engine::carve_kv(Carver& c, KvCache& o, int rows, int max_seq, int layers, bool f8) const {
    const size_t bytes = (size_t)rows * cfg.n_head * max_seq * hdp * (f8 ? 1 : esz) * layers, start = c.off;
    o.kcache = c.split(bytes, kRegionKv);
    o.vcache = c.split(bytes, kRegionKv);
    o.cache_bytes = c.off - start;
    o.rows = rows / c.n;
    o.max_seq = max_seq;
    o.layers = layers;
    o.kv_f8 = f8;
}

// The row buffers of M activation rows, x0_rows caption rows, partial_floats GEMM partials and logits_rows rows of logits. The partials
// region holds a whole number of 64-float slices for each of `chains` chains, so that chain g of n takes its n-th, 64-float aligned and
// at least an n-th of partial_floats.
void lg_engine::carve_rows(Carver& c, RowBuffers& o, size_t M, size_t x0_rows, size_t partial_floats, size_t logits_rows, int chains) const {
    o.h = c.split(M * cfg.dim * esz);
    o.xn = c.split(M * cfg.dim * esz);
    o.q = c.split(M * cfg.dim * esz);
    o.attn = c.split(M * cfg.dim * esz);
    o.ff = c.split(M * cfg.ffn_dim * esz);
    o.x0 = c.split(x0_rows * cfg.caption_dim * esz);
    const size_t region = chains == 1 ? partial_floats : (partial_floats + 64 * chains - 1) / (64 * chains) * (64 * chains);
    o.partial_floats = c.n == 1 ? partial_floats : region / c.n / 64 * 64;
    o.partial = (float*)c.shared(region * sizeof(float), o.partial_floats * sizeof(float), kRegionData, partial_floats * sizeof(float));
    o.logits = (float*)c.split(logits_rows * cfg.vocab_size * sizeof(float));
}

constexpr int kScoreHeadRows = 2048;   // rows per head GEMM of lg_score: its fp32 slabs stay ~kScoreHeadRows * V floats

// lg_score's scratch for `rows` sequences of `seq` positions, from `base` (null: sizes only): the activations of rows * seq positions,
// the GEMM partials of that M (and of the caption MLP and one head chunk), and K / V of ONE layer ([rows, H, round8(seq), hdp] in the
// model dtype, also after lg_engine_set_kv_cache): every layer rewrites it before its attention reads it.
size_t lg_engine::carve_score(Workspace& o, char* base, int rows, int seq) const {
    const int D = cfg.dim, V = cfg.vocab_size, Tc = cfg.cls_token_num, dt = cfg.dtype;
    const bool t2i = cfg.model_type == LG_MODEL_T2I;
    const int M = rows * seq;
    o.head_rows = std::min(rows * std::max(seq - Tc + 1, 1), kScoreHeadRows);
    size_t pf = std::max(layer_partial_floats(M), gemm_partial_floats(o.head_rows, V, D, 0, dt));
    if (t2i) pf = std::max({pf, gemm_partial_floats(rows * Tc, D, cfg.caption_dim, 0, dt), gemm_partial_floats(rows * Tc, D, D, 0, dt)});
    Carver c{base};
    carve_kv(c, o, rows, (seq + 7) / 8 * 8, 1, false);
    carve_rows(c, o, M, t2i ? rows * Tc : 0, pf, 0);
    o.base = base;
    return c.off;
}

// lg_generate_sjd's scratch for B images (nh rows each) and window L, from `base` (null: sizes only): the row buffers of nh * B * L
// rows, and the loop state (sa's buffers). The caller pairs `o` with the KV cache of the full workspace.
size_t lg_engine::carve_sjd(RowBuffers& o, SjdArgs& sa, char* base, int B, int nh, int L) const {
    const int V = cfg.vocab_size;
    const size_t M = (size_t)nh * B * L, BL = (size_t)B * L;
    Carver c{base};
    carve_rows(c, o, M, 0, std::max(layer_partial_floats((int)M), gemm_partial_floats((int)M, V, cfg.dim, 0, cfg.dtype)), M);
    sa.p = (const float*)c.split(BL * V * sizeof(float));
    sa.q = (float*)c.split(BL * V * sizeof(float));
    sa.seed_rows = (uint64_t*)c.split(BL * sizeof(uint64_t), kRegionInt);
    sa.qflag = (int32_t*)c.split(BL * sizeof(int32_t), kRegionInt);
    sa.x = (const int32_t*)c.split(BL * sizeof(int32_t), kRegionInt);
    sa.win = (int32_t*)c.split(BL * sizeof(int32_t), kRegionInt);
    sa.step_rows = (int32_t*)c.split(BL * sizeof(int32_t), kRegionInt);
    sa.nfin = (int32_t*)c.split(B * sizeof(int32_t), kRegionInt);
    sa.start = (int32_t*)c.split(B * sizeof(int32_t), kRegionInt);
    sa.shift = (int32_t*)c.split(B * sizeof(int32_t), kRegionInt);
    sa.pos_rows = (int32_t*)c.split((size_t)nh * B * sizeof(int32_t), kRegionInt);
    sa.state = (int32_t*)c.split(kSjdStateInts * sizeof(int32_t), kRegionInt);
    return c.off;
}

// Serving's SJD state for B slots (lg_sjd_slots_workspace_bytes), from `base` (null: sizes only): carve_sjd's scratch, then every slot's
// seed, pass counter and image index and the guidance of every window row
size_t lg_engine::carve_sjd_slots(RowBuffers& o, SjdArgs& sa, char* base, int B, int nh, int L) const {
    Carver c{base, 0, 1, carve_sjd(o, sa, base, B, nh, L)};
    const size_t BL = (size_t)B * L;
    sa.seed_slots = (uint64_t*)c.split(B * sizeof(uint64_t), kRegionInt);
    sa.pass_slots = (int32_t*)c.split(B * sizeof(int32_t), kRegionInt);
    sa.cfg_rows = (float*)c.split(BL * sizeof(float));
    sa.interval_rows = (int32_t*)c.split(BL * sizeof(int32_t), kRegionInt);
    sa.img_slots = (int32_t*)c.split(B * sizeof(int32_t), kRegionInt);
    return c.off;
}

// lg_generate_prefix's scratch for a chunk of `rows` cache rows of `seq` positions (the condition and the prefix), from `base` (null:
// sizes only): the row buffers of rows * seq positions and the GEMM partials of that M and of the caption MLP. The K / V rows go to
// the workspace's cache, the last positions to its row buffers.
size_t lg_engine::carve_prefix(RowBuffers& o, char* base, int rows, int seq) const {
    const int D = cfg.dim, Tc = cfg.cls_token_num, dt = cfg.dtype;
    const bool t2i = cfg.model_type == LG_MODEL_T2I;
    size_t pf = layer_partial_floats(rows * seq);
    if (t2i) pf = std::max({pf, gemm_partial_floats(rows * Tc, D, cfg.caption_dim, 0, dt), gemm_partial_floats(rows * Tc, D, D, 0, dt)});
    Carver c{base};
    carve_rows(c, o, (size_t)rows * seq, t2i ? (size_t)rows * Tc : 0, pf, 0);
    return c.off;
}

// lg_prefill_slot_prefix's scratch for one request of nh rows, from `base` (null: sizes only): one prefill chunk of one row of `seq`
// = T + P positions (carve_prefix, from base on), then the request's nh last positions (head.q) and the partials of the head GEMM over
// them. lg_prefill_slot's is the seq = cls_token_num case.
size_t lg_engine::carve_slot(RowBuffers& head, char* base, int nh, int seq) const {
    const int D = cfg.dim, V = cfg.vocab_size, dt = cfg.dtype;
    RowBuffers chunk;
    Carver c{base, 0, 1, carve_prefix(chunk, nullptr, 1, seq)};
    head.q = c.split((size_t)nh * D * esz);
    head.partial_floats = std::max(gemm_partial_floats(nh, V, D, 0, dt), gemm_partial_floats(nh, V, D, 0, dt, output.scale != nullptr));
    head.partial = (float*)c.split(head.partial_floats * sizeof(float));
    return c.off;
}

// lg_generate_given's extend pass of one chain of B images (nh rows each), from `base` (null: sizes only): the row buffers of nh * B
// windows of W rows, the GEMM partials of that M and of the head over the nh * B last rows, then the window's tokens [B, W] and its
// rows' positions [nh * B]. The K / V rows go to the chain's cache, the logits to its row buffers.
size_t lg_engine::carve_given_window(RowBuffers& o, int32_t** win, int32_t** pos_rows, char* base, int B, int nh, int W) const {
    const int R = nh * B, V = cfg.vocab_size, D = cfg.dim, dt = cfg.dtype;
    const size_t M = (size_t)R * W;
    const size_t pf = std::max({layer_partial_floats((int)M), gemm_partial_floats(R, V, D, 0, dt),
                                gemm_partial_floats(R, V, D, 0, dt, output.scale != nullptr)});
    Carver c{base};
    carve_rows(c, o, M, 0, pf, 0);
    *win = (int32_t*)c.split((size_t)B * W * sizeof(int32_t), kRegionInt);
    *pos_rows = (int32_t*)c.split((size_t)R * sizeof(int32_t), kRegionInt);
    return c.off;
}

int lg_engine::gemm(const Workspace& w, const void* x, int M, int N, int K, const GemmWeight& wa, const GemmWeight& wb, int n_split, int* ksplit,
                    float* direct_out, cudaStream_t st, const GemmNext* next, bool pdl) {
    // when the plan needs a single slab the GEMM can write straight into `direct_out`
    const size_t need = gemm_partial_floats(M, N, K, wb.p ? n_split : 0, cfg.dtype, wa.scale != nullptr);
    LG_REQUIRE(need > 0, "%s", gemm_plan(M, N, K, wb.p ? n_split : 0, cfg.dtype, wa.scale != nullptr).error);
    const size_t slabs = need / ((size_t)M * N);
    float* dst = (direct_out && slabs == 1) ? direct_out : w.partial;
    // the plan (k-slices) is not monotone in M and depends on run-time switches: never trust the carve-time sizing blindly
    LG_REQUIRE(dst == direct_out || need <= w.partial_floats, "gemm %dx%dx%d needs %zu partial floats, workspace holds %zu", M, N, K, need,
               w.partial_floats);
    GemmPlan plan;
    LG_TRY(gemm_partial(x, K, wa, wb, n_split, M, N, K, cfg.dtype, dst, &plan, st, next, pdl));
    *ksplit = plan.ksplit;
    return dst == direct_out ? 1 : 0;
}

int lg_engine::forward(const Workspace& w, int M, int Tq, PosArg pos, const float* emb_mask, const float* neg_mask, int B, float* logits_out,
                       bool xn_ready, cudaStream_t st, bool pdl_first) {
    const int L = cfg.n_layer, D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size;
    const int R = M / Tq;
    const int dt = cfg.dtype;
    // ---- R <= 8 decode step (batch-1 latency path, gemv_small.cu): 5 dependent kernels per layer, no slabs
    if (Tq == 1 && small_row_path(M, attn_args(w, 0, R, Tq))) {
        for (int l = 0; l < L; ++l) {
            const Layer& ly = layers[l];
            GemvSmall gq{ly.wqkv, nullptr, 3 * D, D, M, w.h, ly.attn_norm, cfg.norm_eps, w.partial, nullptr, nullptr, dt};
            gq.pdl = l > 0 || pdl_first;
            LG_PROF(PC_GEMM_QKV, st, launch_gemv_small(gq, st));
            AttnArgs aa = layer_attn(w, l, R, Tq, pos, emb_mask, neg_mask, B);
            aa.qkv_partial = w.partial; aa.qkv_ksplit = 1; aa.freqs = freqs;
            LG_PROF(PC_ATTENTION, st, launch_attention(aa, st));
            GemvSmall go{ly.wo, nullptr, D, D, M, w.attn, nullptr, 0.f, nullptr, w.h, nullptr, dt};
            LG_PROF(PC_GEMM_WO, st, launch_gemv_small(go, st));
            GemvSmall g13{ly.w1, ly.w3, F, D, M, w.h, ly.ffn_norm, cfg.norm_eps, nullptr, nullptr, w.ff, dt};
            LG_PROF(PC_GEMM_W13, st, launch_gemv_small(g13, st));
            GemvSmall g2{ly.w2, nullptr, D, F, M, w.ff, nullptr, 0.f, nullptr, w.h, nullptr, dt};
            LG_PROF(PC_GEMM_W2, st, launch_gemv_small(g2, st));
        }
        GemvSmall gh{output, nullptr, V, D, M, w.h, final_norm, cfg.norm_eps, logits_out, nullptr, nullptr, dt};
        LG_PROF(PC_GEMM_HEAD, st, launch_gemv_small(gh, st));
        return 0;
    }
    LG_TRY(run_layers(w, M, Tq, pos, emb_mask, neg_mask, B, xn_ready, st, pdl_first));
    // head on the last position only (generate.py:58 reads logits[:, -1])
    const void* xlast = w.xn;
    if (Tq > 1) {
        LG_TRY(launch_gather_last(w.xn, R, Tq, D, dt, w.q, st));
        xlast = w.q;
    }
    GemmNext nx_first{layers[0].wqkv.p, layers[0].wqkv.bytes(3 * D, D, esz), nullptr, 0};   // the next decode step starts with layer 0
    return head(w, xlast, R, logits_out, &nx_first, st);
}

// The head GEMM over M rows of x: straight into logits_out when the plan has one slab, otherwise through the partials
int lg_engine::head(const Workspace& w, const void* x, int M, float* logits_out, const GemmNext* next, cudaStream_t st) {
    const int V = cfg.vocab_size;
    int ks = 1;
    prof_begin(PC_GEMM_HEAD, st);
    const int direct = gemm(w, x, M, V, cfg.dim, output, nullptr, 0, &ks, logits_out, st, next);
    prof_end(st);
    if (direct < 0) return direct;
    if (direct == 0) LG_TRY(launch_reduce_f32(w.partial, ks, M, V, logits_out, st));
    return 0;
}

int lg_engine::run_layers(const Workspace& w, int M, int Tq, PosArg pos, const float* emb_mask, const float* neg_mask, int B, bool xn_ready,
                          cudaStream_t st, bool pdl_first) {
    const int L = cfg.n_layer, D = cfg.dim, F = cfg.ffn_dim, V = cfg.vocab_size;
    const int R = M / Tq;
    const int dt = cfg.dtype;
    int ks = 1;
    if (!xn_ready) LG_PROF(PC_EMBED_MISC, st, launch_rmsnorm(w.h, layers[0].attn_norm, w.xn, M, D, cfg.norm_eps, dt, st, pdl_first));
    for (int l = 0; l < L; ++l) {
        const Layer& ly = layers[l];
        const size_t eb = esz;
        const bool last = l + 1 == L;     // prefetch sizes are those of the tensors as bound (fp8 codes are one byte)
        GemmNext nx_wo{ly.wo.p, ly.wo.bytes(D, D, eb), nullptr, 0};
        GemmNext nx_w13{ly.w1.p, ly.w1.bytes(F, D, eb), ly.w3.p, ly.w3.bytes(F, D, eb)};
        GemmNext nx_w2{ly.w2.p, ly.w2.bytes(D, F, eb), nullptr, 0};
        GemmNext nx_qkv{last ? output.p : layers[l + 1].wqkv.p, last ? output.bytes(V, D, eb) : layers[l + 1].wqkv.bytes(3 * D, D, eb), nullptr, 0};
        LG_PROF(PC_GEMM_QKV, st, gemm(w, w.xn, M, 3 * D, D, ly.wqkv, nullptr, 0, &ks, nullptr, st, &nx_wo, l > 0 || !xn_ready || pdl_first));
        AttnArgs aa = layer_attn(w, l, R, Tq, pos, emb_mask, neg_mask, B);
        if (fuse_qkv(aa)) {
            aa.qkv_partial = w.partial; aa.qkv_ksplit = ks; aa.freqs = freqs;
        } else {
            LG_PROF(PC_QKV_EPI, st, launch_qkv_epilogue(make_qkv_epi_args(aa, w.partial, ks, freqs), st));
        }
        LG_PROF(PC_ATTENTION, st, launch_attention(aa, st));
        LG_PROF(PC_GEMM_WO, st, gemm(w, w.attn, M, D, D, ly.wo, nullptr, 0, &ks, nullptr, st, &nx_w13));
        LG_PROF(PC_RESNORM, st, launch_residual_norm(w.partial, ks, M, D, w.h, ly.ffn_norm, w.xn, cfg.norm_eps, dt, st));
        LG_PROF(PC_GEMM_W13, st, gemm(w, w.xn, M, 2 * F, D, ly.w1, ly.w3, F, &ks, nullptr, st, &nx_w2));
        LG_PROF(PC_SILU, st, launch_silu_mul(w.partial, ks, M, F, w.ff, dt, st));
        LG_PROF(PC_GEMM_W2, st, gemm(w, w.ff, M, D, F, ly.w2, nullptr, 0, &ks, nullptr, st, &nx_qkv));
        const void* next_norm = (l + 1 < L) ? layers[l + 1].attn_norm : final_norm;
        LG_PROF(PC_RESNORM, st, launch_residual_norm(w.partial, ks, M, D, w.h, next_norm, w.xn, cfg.norm_eps, dt, st));
    }
    return 0;
}

int lg_engine::embed_cond(const Workspace& w, const void* cond, const void* neg_cond, int B, int R, int T, cudaStream_t st) {
    const int D = cfg.dim, dt = cfg.dtype;
    if (cfg.model_type == LG_MODEL_C2I) {
        // LabelEmbedder (gpt.py:78-83); null class = num_classes (generate.py:130)
        return launch_embed(cls_table, (const int32_t*)cond, B, R, cfg.num_classes, D, dt, w.h, st);
    }
    // CaptionEmbedder: cap_proj = fc2(gelu_tanh(fc1(x))) (gpt.py:110-131); uncond rows = uncond_embedding, or one negative per image
    const int C = cfg.caption_dim, M = R * T;
    int ks = 1;
    LG_TRY(launch_build_caption_rows(cond, neg_cond ? neg_cond : uncond, neg_cond ? (size_t)T * C : 0, B, R, T, C, dt, w.x0, st));
    LG_TRY(gemm(w, w.x0, M, D, C, cap_fc1, nullptr, 0, &ks, nullptr, st));
    LG_TRY(launch_store_act(w.partial, ks, M, D, w.attn, 1, dt, st));
    LG_TRY(gemm(w, w.attn, M, D, D, cap_fc2, nullptr, 0, &ks, nullptr, st));
    LG_TRY(launch_store_act(w.partial, ks, M, D, w.h, 0, dt, st));
    return 0;
}

static int check_ready(lg_engine* e, int rows, int seq) {
    LG_REQUIRE(e && e->finalized, "engine not finalized");
    LG_REQUIRE(e->full.base, "workspace not set");
    LG_REQUIRE(rows <= e->full.rows, "rows %d exceed workspace rows %d", rows, e->full.rows);
    LG_REQUIRE(seq <= e->full.max_seq, "sequence %d exceeds workspace max_seq %d", seq, e->full.max_seq);
    LG_REQUIRE(seq <= e->cfg.cls_token_num + e->cfg.block_size, "sequence %d exceeds the RoPE table (%d)", seq,
               e->cfg.cls_token_num + e->cfg.block_size);
    return 0;
}

// 16-bit engines: the head's logits are a bf16 / fp16 tensor in the reference (gpt.py:368 `.float()` of it); no-op for fp32
static int round_logits_inplace(float* logits, size_t n, int dtype, cudaStream_t st);

// One eager forward of R rows of Tq positions each (up to position seq) on the full workspace for the entry point fn: `embed` checks
// fn's own arguments and writes the rows of h, then the forward writes the logits as the reference's head rounds them
template <class Embed>
static int eager_forward(const char* fn, lg_engine* e, int R, int Tq, int seq, PosArg pos, const float* emb_mask, const float* neg_mask, int B,
                         float* logits_out, void* stream, Embed&& embed) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(e, "%s: null engine", fn);
    DeviceGuard guard(e->device);
    LG_TRY(check_ready(e, R, seq));
    LG_TRY(e->zero_fill_if_needed(st));
    LG_TRY(embed(st));
    LG_TRY(e->forward(e->full, R * Tq, Tq, pos, emb_mask, neg_mask, B, logits_out, false, st));
    return round_logits_inplace(logits_out, (size_t)R * e->cfg.vocab_size, e->cfg.dtype, st);
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

// A GEMM weight [N][K] (n_split: the w1 | w3 boundary of the GEMM that streams it, 0 for one segment): in the model dtype, or bound as
// LG_DTYPE_E4M3 codes with its companion "<name>_scale" fp32 [N]. An fp8 weight is refused on an fp32 model, without its scales, with
// a scale that is not an allowed power of two, and with a shape the fp8 GEMM kernel does not take.
static int need_gemm_weight(lg_engine* e, const std::string& name, int64_t N, int64_t K, int NN, int n_split, GemmWeight* out) {
    const int dt = e->cfg.dtype;
    auto it = e->w.find(name);
    const void* p = nullptr;
    if (it == e->w.end() || it->second.dtype != LG_DTYPE_E4M3) {
        LG_TRY(need(e, name, dt, {N, K}, &p));
        *out = GemmWeight(p);
        return 0;
    }
    LG_REQUIRE(lg_dtype_is16(dt), "weight '%s' is fp8: fp8 weights need a bf16 or fp16 model (model dtype %d)", name.c_str(), dt);
    LG_TRY(need(e, name, LG_DTYPE_E4M3, {N, K}, &p));
    const void* sc = nullptr;
    LG_TRY(need(e, name + "_scale", LG_DTYPE_F32, {N}, &sc));
    const GemmPlan plan = gemm_plan(16, NN, (int)K, n_split, dt, true);
    LG_REQUIRE(plan.kernel >= 0, "weight '%s' [%lld, %lld] cannot be fp8: %s", name.c_str(), (long long)N, (long long)K, plan.error);
    DeviceGuard guard(e->device);
    LG_TRY(w8_check_scales((name + "_scale").c_str(), (const float*)sc, (int)N, dt));
    *out = GemmWeight(p, (const float*)sc);
    return 0;
}

int lg_engine_finalize(lg_engine* e) {
    LG_REQUIRE(e, "null engine");
    const lg_model_cfg& c = e->cfg;
    const int D = c.dim, F = c.ffn_dim, V = c.vocab_size, dt = c.dtype;
    e->layers.resize(c.n_layer);
    e->layer_weight_bytes = 0;
    for (int l = 0; l < c.n_layer; ++l) {
        const std::string p = "layers." + std::to_string(l) + ".";
        Layer& ly = e->layers[l];
        LG_TRY(need_gemm_weight(e, p + "attention.wqkv.weight", 3 * D, D, 3 * D, 0, &ly.wqkv));
        LG_TRY(need_gemm_weight(e, p + "attention.wo.weight", D, D, D, 0, &ly.wo));
        LG_TRY(need_gemm_weight(e, p + "feed_forward.w1.weight", F, D, 2 * F, F, &ly.w1));
        LG_TRY(need_gemm_weight(e, p + "feed_forward.w3.weight", F, D, 2 * F, F, &ly.w3));
        LG_REQUIRE((ly.w1.scale != nullptr) == (ly.w3.scale != nullptr),
                   "layer %d: feed_forward.w1 and w3 are streamed by one GEMM and must both be fp8 or both be 16-bit", l);
        LG_TRY(need_gemm_weight(e, p + "feed_forward.w2.weight", D, F, D, 0, &ly.w2));
        e->layer_weight_bytes = std::max(e->layer_weight_bytes, ly.wqkv.bytes(3 * D, D, e->esz) + ly.wo.bytes(D, D, e->esz) +
                                                                    ly.w1.bytes(F, D, e->esz) + ly.w3.bytes(F, D, e->esz) +
                                                                    ly.w2.bytes(D, F, e->esz));
        LG_TRY(need(e, p + "attention_norm.weight", dt, {D}, &ly.attn_norm));
        LG_TRY(need(e, p + "ffn_norm.weight", dt, {D}, &ly.ffn_norm));
    }
    LG_TRY(need(e, "tok_embeddings.weight", dt, {V, D}, &e->tok_emb));
    LG_TRY(need(e, "norm.weight", dt, {D}, &e->final_norm));
    LG_TRY(need_gemm_weight(e, "output.weight", V, D, V, 0, &e->output));
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
    Workspace full;
    const size_t needb = e->carve(full, (char*)dev_ws, rows, max_seq);
    LG_REQUIRE(bytes >= needb, "workspace too small: %zu < %zu", bytes, needb);
    // The reference zero-fills the KV cache (gpt.py:174-175). The tensor-core attention multiplies masked
    // probabilities (exactly 0) with whatever sits in not-yet-written V rows, so those rows must be finite.
    // The zero-fill is enqueued on the CALLER'S stream by the first prefill / decode / generate that uses this workspace
    // (zero_fill_if_needed): a legacy-NULL-stream memset here would not be ordered against non-blocking streams that may
    // still be running kernels on memory the caching allocator has just recycled.
    e->ws_needs_zero = true;
    LG_TRY(e->make_maps(full));
    e->full = full;
    e->n_sub = 0;
    // Chain-count policy: every chain streams ALL the weights, so two chains only pay while a layer's weights survive in L2 between
    // the chains' visits, next to the KV and activation traffic of the other chain; otherwise they double the HBM weight traffic.
    // Two chains run while a layer's GEMM weights as bound (fp8 weights count one byte per element) are at most a third of the L2. On an H100 80GB HBM3 (50 MB L2; both settings alternated twice in
    // one run) one chain is faster for GPT-L (27 MB per layer, c2i 256 px, B = 64: 431 vs 469 ms/step) and GPT-XL (39 MB, 384 px,
    // B = 32: 1659 vs 1849 ms/step).
    // LG_SPLIT forces the chain count (at most two).
    const double layer_bytes = e->finalized ? (double)e->layer_weight_bytes
                                            : (4.0 * e->cfg.dim * e->cfg.dim + 3.0 * e->cfg.dim * e->cfg.ffn_dim) * e->esz;
    int l2_bytes = 0, dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, dev) != cudaSuccess) l2_bytes = 0;
    int n = lg_env_flag("LG_SPLIT", 3.0 * layer_bytes <= (double)l2_bytes ? 2 : 1);
    if (n > lg_engine::kMaxChains) n = lg_engine::kMaxChains;
    while (n >= 2 && (rows % n != 0 || (rows / n) % 2 != 0 || rows / n < 16)) --n;
    if (n >= 2 && full.maps.usable) {   // chains run bf16 / fp16 models whose cache the TMA attention kernels stream
        Workspace need;                 // a chain's GEMMs must fit in its share of the partials
        e->carve(need, nullptr, rows / n, max_seq);
        for (int g = 0; g < n; ++g) e->carve(e->sub[g], (char*)dev_ws, rows, max_seq, g, n);
        if (need.partial_floats <= e->sub[0].partial_floats) {
            for (int g = 0; g < n; ++g) LG_TRY(e->make_maps(e->sub[g]));
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
    e->kv_scales = sc;
    e->full = Workspace();
    e->n_sub = 0;
    e->ws_needs_zero = false;
    return 0;
}

int lg_prefill(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int use_cfg, float* logits_out,
               void* stream) {
    const int R = use_cfg ? 2 * B : B;
    auto embed = [&](cudaStream_t st) -> int {
        LG_REQUIRE(cond && logits_out && B > 0, "lg_prefill: bad argument");
        LG_REQUIRE(T == e->cfg.cls_token_num, "lg_prefill: T=%d must equal cls_token_num=%d", T, e->cfg.cls_token_num);
        return e->embed_cond(e->full, cond, nullptr, B, R, T, st);
    };
    return eager_forward("lg_prefill", e, R, T, T, PosArg{nullptr, 0}, emb_mask, nullptr, B, logits_out, stream, embed);
}

int lg_decode_step(lg_engine* e, const int32_t* tokens, int B, int pos, int use_cfg, float* logits_out, void* stream) {
    const int R = use_cfg ? 2 * B : B;
    auto embed = [&](cudaStream_t st) -> int {
        LG_REQUIRE(tokens && logits_out && B > 0 && pos >= 0, "lg_decode_step: bad argument");
        return launch_embed(e->tok_emb, tokens, B, R, -1, e->cfg.dim, e->cfg.dtype, e->full.h, st);
    };
    return eager_forward("lg_decode_step", e, R, 1, pos + 1, PosArg{nullptr, pos}, nullptr, nullptr, B, logits_out, stream, embed);
}

int lg_decode_rows(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, int B, int use_cfg, float* logits_out, void* stream) {
    // Iteration-level scheduling (serve/llm_engine.py:511 step()): one forward for R rows that sit at DIFFERENT depths. A row at
    // position 0 is a request that has just joined: it takes its class embedding (the c2i "prefill" is that single position).
    const int R = use_cfg ? 2 * B : B;
    auto embed = [&](cudaStream_t st) -> int {
        LG_REQUIRE(tokens && pos_rows && logits_out && B > 0, "lg_decode_rows: bad argument");
        LG_REQUIRE(e->cfg.model_type == LG_MODEL_C2I && e->cfg.cls_token_num == 1, "lg_decode_rows: class-conditional models only");
        const lg_model_cfg& c = e->cfg;
        return launch_embed_rows(e->cls_table, e->tok_emb, tokens, pos_rows, B, R, c.num_classes, c.dim, c.dtype, e->full.h, st);
    };
    return eager_forward("lg_decode_rows", e, R, 1, 1, PosArg{nullptr, 0, pos_rows}, nullptr, nullptr, B, logits_out, stream, embed);
}

}  // extern "C"

// The checks an entry point fn that takes a negative makes of it before any launch (e non-null)
static int check_negative(const char* fn, const lg_engine* e, const Negative& neg, const float* emb_mask, bool use_cfg) {
    if (!neg.cond && !neg.mask) return 0;
    LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "%s: a negative condition applies to t2i models only", fn);
    LG_REQUIRE(neg.cond, "%s: neg_mask without neg_cond", fn);
    LG_REQUIRE(use_cfg, "%s: a negative condition replaces the unconditional CFG rows and needs CFG (cfg_scale > 1)", fn);
    LG_REQUIRE(!neg.mask || emb_mask, "%s: neg_mask needs emb_mask (all ones for an unmasked condition)", fn);
    return 0;
}

// lg_decode_rows for text-conditional serving: every row is past its condition (lg_prefill_slot wrote positions 0 .. T - 1), so every
// row takes a token embedding; the emb-mask rows follow the rows' slots (row r reads mask row r % B, of neg_mask when set for r >= B)
static int decode_rows_t2i_impl(const char* fn, lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, const float* emb_mask,
                                const float* neg_mask, int B, int use_cfg, float* logits_out, void* stream) {
    const int R = use_cfg ? 2 * B : B;
    LG_REQUIRE(e, "%s: null engine", fn);
    LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "%s: text-conditional models only", fn);
    LG_REQUIRE(tokens && pos_rows && logits_out && B > 0, "%s: bad argument", fn);
    LG_REQUIRE(!neg_mask || use_cfg, "%s: neg_mask masks the unconditional CFG rows and needs use_cfg", fn);
    LG_REQUIRE(!neg_mask || emb_mask, "%s: neg_mask needs emb_mask (all ones for an unmasked condition)", fn);
    auto embed = [&](cudaStream_t st) -> int {
        return launch_embed(e->tok_emb, tokens, B, R, -1, e->cfg.dim, e->cfg.dtype, e->full.h, st);
    };
    return eager_forward(fn, e, R, 1, 1, PosArg{nullptr, 0, pos_rows}, emb_mask, neg_mask, B, logits_out, stream, embed);
}

extern "C" {

int lg_decode_rows_t2i(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, const float* emb_mask, int B, int use_cfg,
                       float* logits_out, void* stream) {
    return decode_rows_t2i_impl("lg_decode_rows_t2i", e, tokens, pos_rows, emb_mask, nullptr, B, use_cfg, logits_out, stream);
}

int lg_decode_rows_t2i_neg(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, const float* emb_mask, const float* neg_mask, int B,
                           int use_cfg, float* logits_out, void* stream) {
    return decode_rows_t2i_impl("lg_decode_rows_t2i_neg", e, tokens, pos_rows, emb_mask, neg_mask, B, use_cfg, logits_out, stream);
}

int lg_score_workspace_bytes(lg_engine* e, int rows, int seq, size_t* bytes) {
    LG_REQUIRE(e && bytes && rows > 0 && seq > 0, "lg_score_workspace_bytes: bad argument");
    LG_REQUIRE(seq >= e->cfg.cls_token_num && seq <= e->cfg.cls_token_num + e->cfg.block_size - 1,
               "lg_score_workspace_bytes: seq %d outside [cls_token_num, cls_token_num + block_size - 1] = [%d, %d]", seq,
               e->cfg.cls_token_num, e->cfg.cls_token_num + e->cfg.block_size - 1);
    Workspace tmp;
    *bytes = e->carve_score(tmp, nullptr, rows, seq);
    return 0;
}

int lg_score(lg_engine* e, const void* cond, const float* emb_mask, const int32_t* idx, const int32_t* targets, int B, int T, int S,
             int use_cfg, float cfg_scale, void* dev_ws, size_t ws_bytes, float* logits_out, float* nll_out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(e && e->finalized, "lg_score: engine not finalized");
    DeviceGuard guard(e->device);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(cond && B > 0, "lg_score: null cond or B=%d", B);
    LG_REQUIRE(T == c.cls_token_num, "lg_score: T=%d must equal cls_token_num=%d", T, c.cls_token_num);
    LG_REQUIRE(S >= 1 && S <= c.block_size, "lg_score: S=%d outside [1, block_size=%d]", S, c.block_size);
    LG_REQUIRE((idx == nullptr) == (S == 1), "lg_score: idx must be NULL exactly when S == 1 (S=%d)", S);
    LG_REQUIRE(logits_out || nll_out, "lg_score: nothing to write (logits_out and nll_out are both NULL)");
    LG_REQUIRE(!nll_out || targets, "lg_score: nll_out needs targets");
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "lg_score: emb_mask only applies to t2i models");
    LG_REQUIRE(!use_cfg || std::isfinite(cfg_scale), "lg_score: cfg_scale %g is not finite", (double)cfg_scale);
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "lg_score: scratch must be non-null and 256-byte aligned");
    const int nh = use_cfg ? 2 : 1, seq = T + S - 1, D = c.dim, V = c.vocab_size, dt = c.dtype;
    // images per chunk: the scratch bounds it, and so does attention_kernel's grid (R * seq <= 65535 query rows) when the sequence
    // is not on a tensor-core path (fp32 models, or LG_ATTN_TMA=0)
    auto fits = [&](int nb) {
        Workspace w;
        return e->carve_score(w, (char*)dev_ws, nh * nb, seq) <= ws_bytes && e->make_maps(w) == 0 &&
               attn_plan(e->attn_args(w, 0, nh * nb, seq)).kernel >= 0;
    };
    {
        Workspace one;
        const size_t need1 = e->carve_score(one, nullptr, nh, seq);
        LG_REQUIRE(ws_bytes >= need1, "lg_score: scratch of %zu bytes is too small for one image (%zu)", ws_bytes, need1);
    }
    int lo = 1, hi = B;   // largest chunk that fits
    while (lo < hi) {
        const int mid = lo + (hi - lo + 1) / 2;
        if (fits(mid)) lo = mid; else hi = mid - 1;
    }
    LG_REQUIRE(fits(lo), "lg_score: no chunk of images fits the scratch (%zu bytes) and the attention grid", ws_bytes);
    const size_t esz = e->esz;
    for (int b0 = 0; b0 < B; b0 += lo) {
        const int nb = std::min(lo, B - b0), R = nh * nb;
        Workspace w;
        e->carve_score(w, (char*)dev_ws, R, seq);
        LG_TRY(e->make_maps(w));
        // K / V rows past the sequence and dims hd..hdp-1 are never written. The tensor-core attentions read them: the hd-64 prefill
        // kernel (seq 121..128) stages keys up to 128 and the windowed kernel (seq > 128) whole 64-key blocks, and both multiply the
        // masked probabilities (exact zeros) by those V rows; the CUDA-core kernel of shorter sequences reads only keys it wrote
        LG_CUDA_OK(cudaMemsetAsync(w.kcache, 0, w.cache_bytes, st));
        const void* cond_c = c.model_type == LG_MODEL_C2I ? (const void*)((const int32_t*)cond + b0)
                                                          : (const void*)((const char*)cond + (size_t)b0 * T * c.caption_dim * esz);
        const float* em = emb_mask ? emb_mask + (size_t)b0 * T : nullptr;
        Workspace wc = w;   // the condition rows [R * T, D] go to ff first, then the sequence embedding assembles h
        wc.h = w.ff;
        LG_TRY(e->embed_cond(wc, cond_c, nullptr, nb, R, T, st));
        LG_TRY(launch_embed_seq(w.ff, e->tok_emb, idx ? idx + (size_t)b0 * (S - 1) : nullptr, nb, R, T, seq, D, dt, w.h, st));
        LG_TRY(e->run_layers(w, R * seq, seq, PosArg{nullptr, 0}, em, nullptr, nb, false, st));
        LG_TRY(launch_gather_scored(w.xn, nb, nh, seq, T, S, D, dt, w.q, st));
        // the head in chunks of at most w.head_rows rows (a CFG pair never splits)
        const int P = nb * S, per = std::max(1, w.head_rows / nh);
        for (int p0 = 0; p0 < P;) {
            int np = std::min(per, P - p0);
            while (np > 1 && gemm_partial_floats(np * nh, V, D, 0, dt) > w.partial_floats) np /= 2;   // the GEMM plan is not monotone in M
            int ks = 1;
            LG_TRY(e->gemm(w, (const char*)w.q + (size_t)p0 * nh * D * esz, np * nh, V, D, e->output, nullptr, 0, &ks, nullptr, st));
            const size_t g0 = (size_t)b0 * S + p0;
            LG_TRY(launch_score_head(w.partial, ks, np, V, nh, cfg_scale, dt, targets ? targets + g0 : nullptr,
                                     logits_out ? logits_out + g0 * V : nullptr, nll_out ? nll_out + g0 : nullptr, st));
            p0 += np;
        }
    }
    return 0;
}

}  // extern "C"

// A caller's lg_logprobs: NULL or every member NULL is off; on, 0 <= top_n <= kMaxTopLogprobs and top_n > 0 needs both top arrays
static int check_logprobs(const char* fn, const lg_logprobs* lp, bool* on) {
    *on = lp && (lp->logprob || lp->rank || (lp->top_n > 0 && (lp->top_ids || lp->top_logprob)));
    if (!lp) return 0;
    LG_REQUIRE(lp->top_n >= 0 && lp->top_n <= kMaxTopLogprobs, "%s: top_n=%d outside [0, %d]", fn, lp->top_n, kMaxTopLogprobs);
    LG_REQUIRE(lp->top_n == 0 || (lp->top_ids && lp->top_logprob), "%s: top_n=%d needs both top_ids and top_logprob", fn, lp->top_n);
    return 0;
}

// The logprob outputs of `lp` (checked by check_logprobs, or NULL) into a, offset by `off` elements of the token row
static void apply_logprobs(SampleArgs& a, const lg_logprobs* lp, size_t off) {
    if (!lp) return;
    a.lp_out = lp->logprob ? lp->logprob + off : nullptr;
    a.rank_out = lp->rank ? lp->rank + off : nullptr;
    if (lp->top_n > 0) {
        a.top_n = lp->top_n;
        a.top_ids = lp->top_ids + off * lp->top_n;
        a.top_lp = lp->top_logprob + off * lp->top_n;
    }
}

// lg_sample_rows (cfg_rows = interval_rows = img_rows = null), lg_sample_rows_guided (img_rows = null), lg_sample_rows_keyed and
// lg_sample_rows_logprobs (lp: NULL for the others), lg_sample_rows_given (given) and lg_sample_rows_composed (mix_rows, mix_weights: a
// gather table, needs mix_cfg); fn names the entry point in messages
static int sample_rows_impl(const char* fn, const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                            const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                            const int32_t* img_rows, const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq, int seq_stride,
                            void* stream, const int32_t* given = nullptr, const int32_t* mix_rows = nullptr,
                            const float* mix_weights = nullptr) {
    LG_REQUIRE(logits && sc && seed_rows && step_rows && (out_idx || out_seq), "%s: null argument", fn);
    LG_REQUIRE(!given || (out_seq && seq_stride > 0), "%s: given tokens are indexed as out_seq and need it", fn);
    LG_REQUIRE(mix_cfg || (!cfg_rows && !interval_rows), "%s: per-row cfg_rows / interval_rows need mix_cfg (2B logits rows)", fn);
    bool lp_on = false;
    LG_TRY(check_logprobs(fn, lp, &lp_on));
    LG_REQUIRE(!lp_on || out_seq, "%s: logprobs are indexed as out_seq and need it", fn);
    SampleArgs a = make_sample_args(*sc, logits, B, V, mix_cfg, round_dtype);
    a.seed_rows = seed_rows; a.step_rows = step_rows;
    a.cfg_rows = cfg_rows; a.interval_rows = interval_rows; a.img_rows = img_rows;
    a.out_idx = out_idx; a.out_seq = out_seq; a.seq_stride = seq_stride; a.given = given;
    a.mix_rows = mix_rows; a.mix_weights = mix_rows ? mix_weights : nullptr;
    if (lp_on) apply_logprobs(a, lp, 0);
    return launch_sample(a, (cudaStream_t)stream);
}

extern "C" {

int lg_sample_rows(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                   const int32_t* step_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream) {
    return sample_rows_impl("lg_sample_rows", logits, B, V, mix_cfg, round_dtype, sc, seed_rows, step_rows, nullptr, nullptr, nullptr,
                            nullptr, out_idx, out_seq, seq_stride, stream);
}

int lg_sample_rows_guided(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                          const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                          int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream) {
    return sample_rows_impl("lg_sample_rows_guided", logits, B, V, mix_cfg, round_dtype, sc, seed_rows, step_rows, cfg_rows,
                            interval_rows, nullptr, nullptr, out_idx, out_seq, seq_stride, stream);
}

int lg_sample_rows_keyed(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                         const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                         const int32_t* img_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream) {
    return sample_rows_impl("lg_sample_rows_keyed", logits, B, V, mix_cfg, round_dtype, sc, seed_rows, step_rows, cfg_rows,
                            interval_rows, img_rows, nullptr, out_idx, out_seq, seq_stride, stream);
}

int lg_sample_rows_logprobs(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                            const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                            const int32_t* img_rows, const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq, int seq_stride,
                            void* stream) {
    return sample_rows_impl("lg_sample_rows_logprobs", logits, B, V, mix_cfg, round_dtype, sc, seed_rows, step_rows, cfg_rows,
                            interval_rows, img_rows, lp, out_idx, out_seq, seq_stride, stream);
}

int lg_sample_rows_given(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                         const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                         const int32_t* img_rows, const int32_t* given, const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq,
                         int seq_stride, void* stream) {
    return sample_rows_impl("lg_sample_rows_given", logits, B, V, mix_cfg, round_dtype, sc, seed_rows, step_rows, cfg_rows,
                            interval_rows, img_rows, lp, out_idx, out_seq, seq_stride, stream, given);
}

int lg_sample_rows_composed(const float* logits, int rows, int B, int V, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                            const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows, const int32_t* img_rows,
                            const int32_t* given, const int32_t* mix_rows, const float* mix_weights, const lg_logprobs* lp,
                            int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream) {
    static const char* fn = "lg_sample_rows_composed";
    // every row may be plain (the roles live on the device), and a plain row reads rows b and B + b
    LG_REQUIRE(B > 0 && V > 0 && rows >= 2 * B, "%s: bad shape rows=%d B=%d V=%d (rows >= 2B)", fn, rows, B, V);
    LG_REQUIRE((mix_rows != nullptr) == (mix_weights != nullptr), "%s: mix_rows and mix_weights go together", fn);
    LG_REQUIRE(round_dtype == LG_DTYPE_F32 || lg_dtype_is16(round_dtype), "%s: unsupported round dtype %d", fn, round_dtype);
    return sample_rows_impl(fn, logits, B, V, 1, round_dtype, sc, seed_rows, step_rows, cfg_rows, interval_rows, img_rows, lp, out_idx,
                            out_seq, seq_stride, stream, given, mix_rows, mix_weights);
}

int lg_sample(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, uint64_t step,
              int32_t* out_idx, float* out_probs, void* stream) {
    LG_REQUIRE(logits && sc && out_idx, "lg_sample: null argument");
    SampleArgs a = make_sample_args(*sc, logits, B, V, mix_cfg, round_dtype);
    a.step = step; a.out_idx = out_idx; a.out_probs = out_probs;
    return launch_sample(a, (cudaStream_t)stream);
}

// The segments generate_impl runs, in token order. A plan starts with one LEAD and draws every token that is not given to all images:
//   LEAD   [0, len): tokens given to every image, prefilled with the condition in one pass (len = 0: the condition alone); its head
//          draws token len
//   DECODE [start, start + len): one decode step per token; images with a given token there take it
//   EXTEND [start, start + len): tokens given to every image between two drawn ones; one window pass over tokens start - 1 ..
//          start + len - 1 writes their K / V, and its last row's head draws token start + len
//   TAIL   [start, S): tokens given to every image after the last drawn one; no forward pass
enum GivenSegKind { kSegLead = 0, kSegDecode = 1, kSegExtend = 2, kSegTail = 3 };
struct GivenSeg {
    int kind, start, len;
};
constexpr int kGivenWindowRows = 64;   // rows of an extend pass's window chunk per image (the windowed tensor-core attention's limit)

// The plan of given [B, S] (host, -1: drawn), or an error when every token is given or a value is below -1
static int given_plan(const char* fn, const int32_t* given, int B, int S, std::vector<GivenSeg>& segs) {
    std::vector<char> all(S, 1);   // token k is given to every image
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < S; ++k) {
            const int32_t v = given[(size_t)b * S + k];
            LG_REQUIRE(v >= -1, "%s: given[%d][%d] = %d (token ids, or -1 for a drawn token)", fn, b, k, v);
            if (v < 0) all[k] = 0;
        }
    int P = 0;
    while (P < S && all[P]) ++P;
    LG_REQUIRE(P < S, "%s: every token is given; nothing to draw", fn);
    segs.clear();
    segs.push_back({kSegLead, 0, P});
    for (int k = P + 1; k < S;) {
        const int a = k;
        const char g = all[k];
        while (k < S && all[k] == g) ++k;
        if (!g) segs.push_back({kSegDecode, a, k - a});
        else if (k == S) segs.push_back({kSegTail, a, k - a});
        else segs.push_back({kSegExtend, a, k++ - a});   // the window draws token k
    }
    return 0;
}

// The rows of the longest extend window of a plan, capped at one chunk (0: no extend)
static int given_window_rows(const std::vector<GivenSeg>& segs) {
    int W = 0;
    for (const GivenSeg& s : segs)
        if (s.kind == kSegExtend) W = std::max(W, std::min(s.len + 1, kGivenWindowRows));
    return W;
}

struct PrefixArgs {              // lg_generate_prefix: prefix [B, P] and the prefill's scratch (P = 0: lg_generate)
    const int32_t* prefix = nullptr;
    int P = 0;
    char* scratch = nullptr;
    size_t scratch_bytes = 0;
    // lg_generate_given: the plan (null: LEAD P, then DECODE to the end), the given tokens dev [B, S] (-1: drawn) and the extend
    // passes' scratch (given_window_bytes) for window chunks of W rows
    const std::vector<GivenSeg>* segs = nullptr;
    const int32_t* given = nullptr;
    char* window = nullptr;
    int W = 0;
};
// lg_generate_composed: every image is K consecutive rows of each half (its K conditions, and K copies of its unconditional row), mixed
// by the sample kernel's grouped mode with weights dev f32 [B / K][K]. Every per-row input (cond, masks, negatives, prefix, given) has
// a row per row; out_tokens and the logprobs have one per image. K = 1 with null weights: one row per image, plain CFG.
struct Compose {
    int K = 1;
    const float* weights = nullptr;
};
static int generate_impl(lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T, int S,
                         const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher,
                         const PrefixArgs& pa, const lg_logprobs* lp, cudaStream_t st, const Compose& cp = Compose{});
// Whether a call runs the unconditional rows: CFG (generate.py:128), or a composed call, which always mixes
static bool uses_cfg(const lg_sample_cfg* sc, const Compose& cp) { return cp.weights || sc->cfg_scale > 1.0f; }

}  // extern "C"

// Bytes of the extend passes' scratch for B images (nh rows each) and window chunks of W rows: the windows of every chain, one after
// the other, for each chain count generate_impl may run (0 without an extend)
static size_t given_window_bytes(const lg_engine* e, int B, int nh, int W) {
    size_t most = 0;
    for (int n = 1; W > 0 && n <= lg_engine::kMaxChains; ++n) {
        if (B % n) continue;
        RowBuffers rb;
        int32_t *win, *pos;
        most = std::max(most, n * e->carve_given_window(rb, &win, &pos, nullptr, B / n, nh, W));
    }
    return most;
}

static int generate_entry(const char* fn, lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T, int S,
                          const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher, void* stream,
                          const lg_logprobs* lp = nullptr, const Compose& cp = Compose{}) {
    LG_REQUIRE(e, "%s: null engine", fn);
    LG_TRY(check_negative(fn, e, neg, emb_mask, sc && uses_cfg(sc, cp)));
    DeviceGuard guard(e->device);
    return e->run_forked((cudaStream_t)stream, lg_engine::kMaxChains, [&](cudaStream_t st) {
        return generate_impl(e, cond, emb_mask, neg, B, T, S, sc, out_tokens, dbg_logits, teacher, PrefixArgs{}, lp, st, cp);
    });
}

extern "C" {

int lg_generate(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc,
                int32_t* out_tokens, float* dbg_logits, const int32_t* teacher, void* stream) {
    return generate_entry("lg_generate", e, cond, emb_mask, Negative{}, B, T, S, sc, out_tokens, dbg_logits, teacher, stream);
}

int lg_generate_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T, int S,
                    const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher, void* stream) {
    return generate_entry("lg_generate_neg", e, cond, emb_mask, Negative{neg_cond, neg_mask}, B, T, S, sc, out_tokens, dbg_logits, teacher,
                          stream);
}

int lg_prefix_workspace_bytes(lg_engine* e, int rows, int seq, size_t* bytes) {
    LG_REQUIRE(e && bytes && rows > 0 && seq > 0, "lg_prefix_workspace_bytes: bad argument");
    RowBuffers tmp;
    *bytes = e->carve_prefix(tmp, nullptr, rows, seq);
    return 0;
}

}  // extern "C"

static int generate_prefix_entry(const char* fn, lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T,
                                 int S, const lg_sample_cfg* sc, const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes,
                                 int32_t* out_tokens, float* dbg_logits, void* stream, const lg_logprobs* lp = nullptr,
                                 const Compose& cp = Compose{}) {
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    DeviceGuard guard(e->device);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(cond && sc && out_tokens && B > 0 && S > 0, "%s: null argument or B=%d S=%d", fn, B, S);
    LG_REQUIRE(prefix, "%s: null prefix", fn);
    LG_REQUIRE(P >= 1 && P <= S - 1, "%s: prefix length P=%d outside [1, S - 1] (S=%d)", fn, P, S);
    LG_REQUIRE(T == c.cls_token_num, "%s: T=%d must equal cls_token_num=%d", fn, T, c.cls_token_num);
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    const int nh = uses_cfg(sc, cp) ? 2 : 1;   // generate.py:128
    LG_TRY(check_negative(fn, e, neg, emb_mask, nh == 2));
    LG_TRY(check_ready(e, nh * B, T + S));
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    RowBuffers one;
    const size_t need1 = e->carve_prefix(one, nullptr, nh, T + P);
    LG_REQUIRE(ws_bytes >= need1, "%s: scratch of %zu bytes is too small for one image (%zu)", fn, ws_bytes, need1);
    const PrefixArgs pa{prefix, P, (char*)dev_ws, ws_bytes};
    return e->run_forked((cudaStream_t)stream, lg_engine::kMaxChains, [&](cudaStream_t st) {
        return generate_impl(e, cond, emb_mask, neg, B, T, S, sc, out_tokens, dbg_logits, nullptr, pa, lp, st, cp);
    });
}

extern "C" {

int lg_generate_prefix(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc,
                       const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, float* dbg_logits, void* stream) {
    return generate_prefix_entry("lg_generate_prefix", e, cond, emb_mask, Negative{}, B, T, S, sc, prefix, P, dev_ws, ws_bytes, out_tokens,
                                 dbg_logits, stream);
}

int lg_generate_prefix_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                           int S, const lg_sample_cfg* sc, const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes, int32_t* out_tokens,
                           float* dbg_logits, void* stream) {
    return generate_prefix_entry("lg_generate_prefix_neg", e, cond, emb_mask, Negative{neg_cond, neg_mask}, B, T, S, sc, prefix, P, dev_ws,
                                 ws_bytes, out_tokens, dbg_logits, stream);
}

int lg_generate_logprobs(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                         int S, const lg_sample_cfg* sc, const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes,
                         const lg_logprobs* lp, int32_t* out_tokens, void* stream) {
    const char* fn = "lg_generate_logprobs";
    bool lp_on = false;
    LG_TRY(check_logprobs(fn, lp, &lp_on));
    const Negative neg{neg_cond, neg_mask};
    if (P == 0) return generate_entry(fn, e, cond, emb_mask, neg, B, T, S, sc, out_tokens, nullptr, nullptr, stream, lp_on ? lp : nullptr);
    return generate_prefix_entry(fn, e, cond, emb_mask, neg, B, T, S, sc, prefix, P, dev_ws, ws_bytes, out_tokens, nullptr, stream,
                                 lp_on ? lp : nullptr);
}

int lg_test_prefix_chunks(lg_engine* e, int* chains) {
    if (!e) return -1;
    if (chains) *chains = e->prefix_chains;
    return e->prefix_chunks;
}

}  // extern "C"

// lg_generate_given's scratch before the prefill's: the given tokens [B, S], the leading run [B, P] and the extend passes' windows
static size_t given_fixed_bytes(const lg_engine* e, int B, int S, int nh, int P, int W) {
    return align_up((size_t)B * S * sizeof(int32_t)) + align_up((size_t)B * P * sizeof(int32_t)) + given_window_bytes(e, B, nh, W);
}

// The checks lg_generate_given and lg_given_workspace_bytes (fn) make of given [B, S] (host) before any launch, then its plan and the
// bytes of its scratch: fixed (given_fixed_bytes) and the prefill's (lg_prefix_workspace_bytes of every row, 0 without a LEAD)
static int given_layout(const char* fn, const lg_engine* e, const int32_t* given, int B, int S, int nh, std::vector<GivenSeg>& segs,
                        size_t* fixed, size_t* prefill) {
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(given, "%s: null given", fn);
    LG_REQUIRE(B > 0 && S >= 1 && S <= c.block_size, "%s: B=%d, or S=%d outside [1, block_size=%d]", fn, B, S, c.block_size);
    for (size_t i = 0; i < (size_t)B * S; ++i)
        LG_REQUIRE(given[i] < c.vocab_size, "%s: given[%zu][%zu] = %d is not below vocab_size=%d", fn, i / S, i % S, given[i],
                   c.vocab_size);
    LG_TRY(given_plan(fn, given, B, S, segs));
    const int P = segs[0].len, W = given_window_rows(segs);
    LG_REQUIRE((long long)nh * B * W <= 65535, "%s: %d rows x window %d exceed 65535 query rows", fn, nh * B, W);
    *fixed = given_fixed_bytes(e, B, S, nh, P, W);
    RowBuffers rb;
    *prefill = P > 0 ? e->carve_prefix(rb, nullptr, nh * B, c.cls_token_num + P) : 0;
    return 0;
}

extern "C" {

int lg_given_workspace_bytes(lg_engine* e, const int32_t* given, int B, int S, int use_cfg, size_t* bytes) {
    LG_REQUIRE(e && bytes, "lg_given_workspace_bytes: null argument");
    std::vector<GivenSeg> segs;
    size_t fixed = 0, prefill = 0;
    LG_TRY(given_layout("lg_given_workspace_bytes", e, given, B, S, use_cfg ? 2 : 1, segs, &fixed, &prefill));
    *bytes = fixed + prefill;
    return 0;
}

}  // extern "C"

// lg_generate_given, and lg_generate_composed with given tokens (B: rows per half, given [B, S] per row, out_tokens [B / K, S])
static int generate_given_impl(const char* fn, lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T,
                               int S, const lg_sample_cfg* sc, const int32_t* given, void* dev_ws, size_t ws_bytes, int32_t* out_tokens,
                               void* stream, const Compose& cp = Compose{}) {
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(cond && sc && out_tokens, "%s: null cond, sc or out_tokens", fn);
    LG_REQUIRE(T == c.cls_token_num, "%s: T=%d must equal cls_token_num=%d", fn, T, c.cls_token_num);
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    const int nh = uses_cfg(sc, cp) ? 2 : 1;   // generate.py:128
    LG_TRY(check_negative(fn, e, neg, emb_mask, nh == 2));
    std::vector<GivenSeg> segs;
    size_t fixed = 0, prefill = 0;
    LG_TRY(given_layout(fn, e, given, B, S, nh, segs, &fixed, &prefill));
    const int P = segs[0].len, W = given_window_rows(segs);
    LG_TRY(check_ready(e, nh * B, T + S));
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    RowBuffers one;
    const size_t need1 = fixed + (P > 0 ? e->carve_prefix(one, nullptr, nh, T + P) : 0);
    LG_REQUIRE(ws_bytes >= need1, "%s: scratch of %zu bytes is too small (%zu with the prefill of one image)", fn, ws_bytes, need1);
    // the scratch: given [B, S], the leading run [B, P], the extend windows, then the prefill's activations
    char* base = (char*)dev_ws;
    int32_t* given_dev = (int32_t*)base;
    int32_t* lead_dev = (int32_t*)(base + align_up((size_t)B * S * sizeof(int32_t)));
    PrefixArgs pa{P > 0 ? lead_dev : nullptr, P, base + fixed, ws_bytes - fixed};
    pa.segs = &segs; pa.given = given_dev; pa.W = W;
    pa.window = (char*)lead_dev + align_up((size_t)B * P * sizeof(int32_t));
    DeviceGuard guard(e->device);
    // given [B, S] and the leading run [B, P] go up in one copy from the engine's pinned staging buffer (laid out as the scratch's head,
    // so the host never waits for earlier work on the stream), then out_tokens starts as given: every drawn token overwrites its -1.
    // The copies run on the caller's stream before the fork, so every chain's stream is ordered after them.
    const cudaStream_t caller = (cudaStream_t)stream;
    const size_t up = (char*)lead_dev - base + (size_t)B * P * sizeof(int32_t);
    LG_TRY(e->stage_given(up));
    std::copy(given, given + (size_t)B * S, e->given_host);
    int32_t* lead_host = e->given_host + ((char*)lead_dev - base) / sizeof(int32_t);
    for (int b = 0; b < B; ++b) std::copy(given + (size_t)b * S, given + (size_t)b * S + P, lead_host + (size_t)b * P);
    LG_CUDA_OK(cudaMemcpyAsync(base, e->given_host, up, cudaMemcpyHostToDevice, caller));
    LG_CUDA_OK(cudaEventRecord(e->ev_given, caller));
    if (cp.K == 1)
        LG_CUDA_OK(cudaMemcpyAsync(out_tokens, given_dev, (size_t)B * S * sizeof(int32_t), cudaMemcpyDeviceToDevice, caller));
    else   // an image's K rows hold the same given tokens: row j K of each image
        LG_CUDA_OK(cudaMemcpy2DAsync(out_tokens, (size_t)S * sizeof(int32_t), given_dev, (size_t)cp.K * S * sizeof(int32_t),
                                     (size_t)S * sizeof(int32_t), B / cp.K, cudaMemcpyDeviceToDevice, caller));
    return e->run_forked(caller, lg_engine::kMaxChains, [&](cudaStream_t st) {
        return generate_impl(e, cond, emb_mask, neg, B, T, S, sc, out_tokens, nullptr, nullptr, pa, nullptr, st, cp);
    });
}

extern "C" {

int lg_generate_given(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T, int S,
                      const lg_sample_cfg* sc, const int32_t* given, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, void* stream) {
    return generate_given_impl("lg_generate_given", e, cond, emb_mask, Negative{neg_cond, neg_mask}, B, T, S, sc, given, dev_ws, ws_bytes,
                               out_tokens, stream);
}

int lg_test_given_plan(const int32_t* given, int B, int S, int32_t* segs_out, int max_segs) {
    static const char* fn = "lg_test_given_plan";
    LG_REQUIRE(given && B > 0 && S > 0 && (segs_out || max_segs == 0) && max_segs >= 0, "%s: bad argument", fn);
    std::vector<GivenSeg> segs;
    LG_TRY(given_plan(fn, given, B, S, segs));
    for (int i = 0; i < (int)segs.size() && i < max_segs; ++i) {
        segs_out[3 * i] = segs[i].kind; segs_out[3 * i + 1] = segs[i].start; segs_out[3 * i + 2] = segs[i].len;
    }
    return (int)segs.size();
}

int lg_generate_composed(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int K,
                         int T, int S, const lg_sample_cfg* sc, const float* weights, const int32_t* prefix, int P, const int32_t* given,
                         void* dev_ws, size_t ws_bytes, const lg_logprobs* lp, int32_t* out_tokens, void* stream) {
    static const char* fn = "lg_generate_composed";
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    LG_REQUIRE(cond && sc && weights && out_tokens, "%s: null cond, sc, weights or out_tokens", fn);
    LG_REQUIRE(B > 0 && K >= 1 && K <= kMaxMixGroups && (long long)B * K <= 65535 && S > 0,
               "%s: B=%d, K=%d outside [1, %d], or S=%d", fn, B, K, kMaxMixGroups, S);
    LG_REQUIRE(K == 1 || sc->cfg_interval < 0, "%s: cfg_interval=%d needs K = 1 (got K=%d)", fn, sc->cfg_interval, K);
    LG_REQUIRE(P >= 0 && P <= S - 1 && (P > 0) == (prefix != nullptr), "%s: prefix length P=%d outside [0, S - 1], or prefix %s", fn, P,
               prefix ? "given with P = 0" : "null");
    bool lp_on = false;
    LG_TRY(check_logprobs(fn, lp, &lp_on));
    LG_REQUIRE(!given || (P == 0 && !lp_on), "%s: given tokens take no prefix and no logprobs", fn);
    const int R = B * K;   // rows per half
    const Compose cp{K, weights};
    const Negative neg{neg_cond, neg_mask};
    if (given) {
        // the rows of an image carry one token row: refuse rows that disagree before the upload
        for (int j = 0; j < B; ++j)
            for (int i = 1; i < K; ++i)
                LG_REQUIRE(std::equal(given + (size_t)j * K * S, given + ((size_t)j * K + 1) * S, given + ((size_t)j * K + i) * S),
                           "%s: given row %d of image %d differs from its row 0", fn, i, j);
        return generate_given_impl(fn, e, cond, emb_mask, neg, R, T, S, sc, given, dev_ws, ws_bytes, out_tokens, stream, cp);
    }
    LG_REQUIRE(T == e->cfg.cls_token_num, "%s: T=%d must equal cls_token_num=%d", fn, T, e->cfg.cls_token_num);
    LG_REQUIRE(!emb_mask || e->cfg.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    LG_TRY(check_negative(fn, e, neg, emb_mask, true));
    LG_TRY(check_ready(e, 2 * R, T + S));
    if (P == 0) return generate_entry(fn, e, cond, emb_mask, neg, R, T, S, sc, out_tokens, nullptr, nullptr, stream, lp_on ? lp : nullptr, cp);
    return generate_prefix_entry(fn, e, cond, emb_mask, neg, R, T, S, sc, prefix, P, dev_ws, ws_bytes, out_tokens, nullptr, stream,
                                 lp_on ? lp : nullptr, cp);
}

namespace {
// One independent decode chain (a contiguous group of images with its own workspace view, stream and graph).
struct Chain {
    Workspace w;
    cudaStream_t st = nullptr;
    const void* cond = nullptr;
    const float* emb_mask = nullptr;
    Negative neg;                      // this chain's images' negatives (null: the null condition)
    const int32_t* prefix = nullptr;   // [B, P] of this chain's images (lg_generate_prefix)
    int B = 0, R = 0;
    SampleArgs sa{};
    Graph graph;
    RowBuffers win;                    // the extend passes' row buffers (lg_generate_given)
    int32_t* win_tokens = nullptr;     // [B, W]
    int32_t* win_pos = nullptr;        // [R]
};
}  // namespace

// One chunk of a condition (+ prefix) prefill: positions 0 .. T + P - 1 of n contiguous cache rows of `kv` from row r0 on, in one
// forward over the row buffers of `scratch`. The rows are n images embedded with their condition (cond: the chunk's first image's),
// or, when `uncond`, with their negatives (neg_cond [n, T, C], the chunk's first image's) or without one the null condition, then
// their prefix embeddings (prefix [n, P], unread when P = 0); emb_mask [n, T] (the mask of the rows' half) or null.
// The attention runs at first_row = r0 over the maps of the whole view, so only rows r0 .. r0 + n - 1 of the cache are written. The
// last position of every row is gathered to `last` [n, D].
static int prefill_chunk(lg_engine* e, const KvCache& kv, int r0, int n, const void* cond, bool uncond, const void* neg_cond,
                         const int32_t* prefix, const float* emb_mask, int T, int P, char* scratch, size_t scratch_bytes, void* last,
                         const char* fn, cudaStream_t st) {
    const int D = e->cfg.dim, dt = e->cfg.dtype, seq = T + P;
    Workspace w;
    static_cast<KvCache&>(w) = kv;
    w.first_row = r0;
    LG_REQUIRE(e->carve_prefix(w, scratch, n, seq) <= scratch_bytes, "%s: a chunk of %d rows outgrows the scratch", fn, n);
    Workspace wc = w;   // the condition rows [n * T, D] go to ff first, then the sequence embedding assembles h
    wc.h = w.ff;
    LG_TRY(e->embed_cond(wc, cond, neg_cond, uncond ? 0 : n, n, T, st));   // B = 0: every row takes the negative or null condition
    LG_TRY(launch_embed_seq(w.ff, e->tok_emb, prefix, n, n, T, seq, D, dt, w.h, st));
    LG_TRY(e->run_layers(w, n * seq, seq, PosArg{nullptr, 0}, emb_mask, nullptr, n, false, st));
    return launch_gather_last(w.xn, n, seq, D, dt, last, st);
}

// lg_generate_prefix's prefill of chain k: positions 0 .. T + P - 1 (the condition, then the prefix embeddings) of every row in one
// forward, its K / V written into the chain's cache. The rows go in chunks of at most `nr` contiguous cache rows of the chain's view
// that stay inside its conditional rows [0, B) or its unconditional rows [B, 2B): a chunk is then images img0 .. img0 + n - 1 of one
// half, embedded with the condition of those images or their negatives (the null condition without), and its attention runs at first_row = its first cache
// row over the maps of the whole view. Chunks also never cross a block of `blk` images (the images of one chain under the largest
// split), so one and two chains run the same chunks with the same GEMM plans: the results are bit-identical. The chunk's last
// positions are gathered into k.w.q rows, and one head GEMM over the R rows leaves the logits of token P in k.w.logits.
static int prefix_prefill(lg_engine* e, Chain& k, int nh, int T, int P, int nr, int blk, const PrefixArgs& pa, cudaStream_t st) {
    const lg_model_cfg& c = e->cfg;
    const int D = c.dim;
    const size_t esz = e->esz;
    for (int half = 0; half < nh; ++half)
        for (int b0 = 0; b0 < k.B; b0 += blk)
        for (int img0 = b0, b1 = std::min(b0 + blk, k.B); img0 < b1; img0 += nr) {
            const int n = std::min(nr, b1 - img0), r0 = half * k.B + img0;
            const void* cond_c = c.model_type == LG_MODEL_C2I ? (const void*)((const int32_t*)k.cond + img0)
                                                              : (const void*)((const char*)k.cond + (size_t)img0 * T * c.caption_dim * esz);
            const float* mask = half != 0 && k.neg.mask ? k.neg.mask : k.emb_mask;
            const float* em = mask ? mask + (size_t)img0 * T : nullptr;
            const void* neg_c = k.neg.cond ? (const char*)k.neg.cond + (size_t)img0 * T * c.caption_dim * esz : nullptr;
            LG_TRY(prefill_chunk(e, k.w, r0, n, cond_c, half != 0, neg_c, k.prefix + (size_t)img0 * P, em, T, P, pa.scratch,
                                 pa.scratch_bytes, k.w.q + (size_t)r0 * D * esz, "lg_generate_prefix", st));
            ++e->prefix_chunks;
        }
    GemmNext nx_first{e->layers[0].wqkv.p, e->layers[0].wqkv.bytes(3 * D, D, esz), nullptr, 0};
    return e->head(k.w, k.w.q, k.R, k.w.logits, &nx_first, st);
}

int lg_slot_workspace_bytes(lg_engine* e, int use_cfg, size_t* bytes) {
    LG_REQUIRE(e && bytes, "lg_slot_workspace_bytes: null argument");
    LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "lg_slot_workspace_bytes: text-conditional models only");
    RowBuffers tmp;
    *bytes = e->carve_slot(tmp, nullptr, use_cfg ? 2 : 1, e->cfg.cls_token_num);
    return 0;
}

int lg_slot_prefix_workspace_bytes(lg_engine* e, int use_cfg, int P, size_t* bytes) {
    LG_REQUIRE(e && bytes, "lg_slot_prefix_workspace_bytes: null argument");
    LG_REQUIRE(P >= 0 && P <= e->cfg.block_size - 1, "lg_slot_prefix_workspace_bytes: prefix length P=%d outside [0, block_size - 1 = %d]",
               P, e->cfg.block_size - 1);
    RowBuffers tmp;
    *bytes = e->carve_slot(tmp, nullptr, use_cfg ? 2 : 1, e->cfg.cls_token_num + P);
    return 0;
}

// A join of serving: lg_generate_prefix's prefill chunk over one request, once for its conditional row `slot` and once, under CFG,
// for its unconditional row B + slot, each one row of T + P positions (the condition, then the prefix embeddings). Every call runs the
// same chunks at the same shapes (one row of T + P positions, then a head GEMM over the request's nh rows), whatever the slot, B or
// the other requests, so a request's logits do not depend on which requests join in the same step or are running. lg_prefill_slot
// is the P = 0 case; fn names the entry point in the messages.
static int prefill_slot_impl(const char* fn, lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int T,
                             const int32_t* prefix, int P, int slot, int B, int use_cfg, void* dev_ws, size_t ws_bytes, float* logits_out,
                             void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(e, "%s: null engine", fn);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(cond && logits_out, "%s: null cond or logits_out", fn);
    LG_REQUIRE(T == c.cls_token_num, "%s: T=%d must equal cls_token_num=%d", fn, T, c.cls_token_num);
    LG_REQUIRE(P == 0 || prefix, "%s: null prefix with P=%d", fn, P);
    LG_REQUIRE(P >= 0 && P <= c.block_size - 1, "%s: prefix length P=%d outside [0, block_size - 1 = %d]", fn, P, c.block_size - 1);
    LG_REQUIRE(B > 0 && slot >= 0 && slot < B, "%s: slot %d outside [0, B=%d)", fn, slot, B);
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    LG_TRY(check_negative(fn, e, neg, emb_mask, use_cfg != 0));
    const int nh = use_cfg ? 2 : 1, D = c.dim, V = c.vocab_size, seq = T + P;
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    LG_TRY(check_ready(e, nh * B, seq));
    RowBuffers hb;
    const size_t need = e->carve_slot(hb, (char*)dev_ws, nh, seq);
    LG_REQUIRE(ws_bytes >= need, "%s: scratch of %zu bytes is too small (%zu)", fn, ws_bytes, need);
    LG_REQUIRE(attn_plan(e->attn_args(e->full, 0, 1, seq)).kernel >= 0, "%s: %s", fn, attn_plan(e->attn_args(e->full, 0, 1, seq)).error);
    DeviceGuard guard(e->device);
    LG_TRY(e->zero_fill_if_needed(st));
    // a c2i join without a prefix is one position per row: where lg_prefill of one image takes the small-row decode path, the join
    // takes it too, one row at a time, so that a one-slot server draws token 0 from the logits generate() draws it from at B = 1
    if (seq == 1 && c.model_type == LG_MODEL_C2I && e->small_row_path(1, e->attn_args(e->full, 0, 1, 1))) {
        for (int half = 0; half < nh; ++half) {
            Workspace w;
            static_cast<KvCache&>(w) = e->full;
            w.first_row = half * B + slot;
            e->carve_prefix(w, (char*)dev_ws, 1, 1);
            LG_TRY(e->embed_cond(w, cond, nullptr, half != 0 ? 0 : 1, 1, T, st));
            LG_TRY(e->forward(w, 1, 1, PosArg{nullptr, 0}, nullptr, nullptr, 1, logits_out + (size_t)half * V, false, st));
        }
        return round_logits_inplace(logits_out, (size_t)nh * V, c.dtype, st);
    }
    for (int half = 0; half < nh; ++half)
        LG_TRY(prefill_chunk(e, e->full, half * B + slot, 1, cond, half != 0, neg.cond, prefix, half != 0 && neg.mask ? neg.mask : emb_mask,
                             T, P, (char*)dev_ws, ws_bytes, hb.q + (size_t)half * D * e->esz, fn, st));
    Workspace w;
    static_cast<RowBuffers&>(w) = hb;
    GemmNext nx_first{e->layers[0].wqkv.p, e->layers[0].wqkv.bytes(3 * D, D, e->esz), nullptr, 0};
    LG_TRY(e->head(w, hb.q, nh, logits_out, &nx_first, st));
    return round_logits_inplace(logits_out, (size_t)nh * V, c.dtype, st);
}

int lg_prefill_slot_prefix(lg_engine* e, const void* cond, const float* emb_mask, int T, const int32_t* prefix, int P, int slot, int B,
                           int use_cfg, void* dev_ws, size_t ws_bytes, float* logits_out, void* stream) {
    return prefill_slot_impl("lg_prefill_slot_prefix", e, cond, emb_mask, Negative{}, T, prefix, P, slot, B, use_cfg, dev_ws, ws_bytes,
                             logits_out, stream);
}

int lg_prefill_slot_prefix_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int T,
                               const int32_t* prefix, int P, int slot, int B, int use_cfg, void* dev_ws, size_t ws_bytes, float* logits_out,
                               void* stream) {
    return prefill_slot_impl("lg_prefill_slot_prefix_neg", e, cond, emb_mask, Negative{neg_cond, neg_mask}, T, prefix, P, slot, B, use_cfg,
                             dev_ws, ws_bytes, logits_out, stream);
}

int lg_prefill_slot(lg_engine* e, const void* cond, const float* emb_mask, int T, int slot, int B, int use_cfg, void* dev_ws,
                    size_t ws_bytes, float* logits_out, void* stream) {
    LG_REQUIRE(e, "lg_prefill_slot: null engine");
    LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "lg_prefill_slot: text-conditional models only");
    return prefill_slot_impl("lg_prefill_slot", e, cond, emb_mask, Negative{}, T, nullptr, 0, slot, B, use_cfg, dev_ws, ws_bytes, logits_out,
                             stream);
}

// The chunk loop of an extend pass: tokens a - 1 .. a + K - 1 of nb images (nh cache rows each, from w.first_row on) at positions
// T + a - 1 .., through the layers in window chunks of at most W rows; their K / V go to w's cache, the activations to w's row buffers.
// Token a - 1 is tokens[b] when tokens is set (the token the previous draw fed forward), every other token given[b][k] ([nb, S]). Rows
// r < nb attend with emb_mask, the others with neg_mask when set. The last row of every cache row's window is gathered to `last`
// [nh * nb, D]. lg_generate_given's extend (every chain's images) and lg_extend_slot (one row of one slot per call) share it, so one
// image at nh = 1 runs the same chunks and GEMM plans in both.
static int extend_window(lg_engine* e, const Workspace& w, int32_t* win_tokens, int32_t* win_pos, const int32_t* tokens,
                         const int32_t* given, int nb, int nh, int S, int T, int a, int K, int W, const float* emb_mask,
                         const float* neg_mask, void* last, cudaStream_t st) {
    const int D = e->cfg.dim, dt = e->cfg.dtype, R = nh * nb;
    int n = 0;
    for (int c0 = 0; c0 < K + 1; c0 += n) {
        n = std::min(W, K + 1 - c0);
        const int j0 = a - 1 + c0;
        LG_TRY(launch_given_window(tokens, given, nb, nh, S, j0, n, tokens && c0 == 0, T + j0, win_tokens, win_pos, st));
        LG_PROF(PC_EMBED_MISC, st, launch_embed(e->tok_emb, win_tokens, nb * n, R * n, -1, D, dt, w.h, st));
        LG_TRY(e->run_layers(w, R * n, n, PosArg{nullptr, 0, win_pos}, emb_mask, neg_mask, nb, false, st));
    }
    return launch_gather_last(w.xn, R, n, D, dt, last, st);
}

// lg_extend_slot's scratch for a request of nh rows and window chunks of W rows, from `base` (null: sizes only): the rows of one cache
// row's window (carve_given_window of one image, one row), then the request's nh last rows (head.q) and the partials of the head GEMM
// over them.
static size_t carve_slot_extend(const lg_engine* e, RowBuffers& win, int32_t** win_tokens, int32_t** win_pos, RowBuffers& head, char* base,
                                int nh, int W) {
    const int D = e->cfg.dim, V = e->cfg.vocab_size, dt = e->cfg.dtype;
    Carver c{base, 0, 1, e->carve_given_window(win, win_tokens, win_pos, base, 1, 1, W)};
    head.q = c.split((size_t)nh * D * e->esz);
    head.partial_floats = std::max(gemm_partial_floats(nh, V, D, 0, dt), gemm_partial_floats(nh, V, D, 0, dt, e->output.scale != nullptr));
    head.partial = (float*)c.split(head.partial_floats * sizeof(float));
    return c.off;
}

int lg_slot_extend_workspace_bytes(lg_engine* e, int use_cfg, int K, size_t* bytes) {
    static const char* fn = "lg_slot_extend_workspace_bytes";
    LG_REQUIRE(e && bytes, "%s: null argument", fn);
    LG_REQUIRE(K >= 1 && K <= e->cfg.block_size - 2, "%s: K=%d outside [1, block_size - 2 = %d]", fn, K, e->cfg.block_size - 2);
    RowBuffers win, head;
    int32_t *t, *p;
    *bytes = carve_slot_extend(e, win, &t, &p, head, nullptr, use_cfg ? 2 : 1, std::min(K + 1, kGivenWindowRows));
    return 0;
}

// An extend of serving: lg_generate_given's extend pass over one request, once for its conditional row `slot` and once, under CFG, for
// its unconditional row B + slot, each one cache row in chunks of at most kGivenWindowRows positions, then one head GEMM over the
// request's nh rows. Every call runs the same chunks at the same shapes whatever the slot, B or the other requests.
int lg_extend_slot(lg_engine* e, const int32_t* tokens, int S, int a, int K, int slot, int B, int use_cfg, const float* emb_mask,
                   const float* neg_mask, void* dev_ws, size_t ws_bytes, float* logits_out, void* stream) {
    static const char* fn = "lg_extend_slot";
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(e, "%s: null engine", fn);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(tokens && logits_out, "%s: null tokens or logits_out", fn);
    LG_REQUIRE(S >= 3 && S <= c.block_size, "%s: S=%d outside [3, block_size=%d]", fn, S, c.block_size);
    LG_REQUIRE(a >= 1 && K >= 1 && a + K <= S - 1, "%s: extend [a=%d, a + K=%d) must lie in [1, S - 1 = %d)", fn, a, a + K, S - 1);
    LG_REQUIRE(B > 0 && slot >= 0 && slot < B, "%s: slot %d outside [0, B=%d)", fn, slot, B);
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    LG_REQUIRE(!neg_mask || use_cfg, "%s: neg_mask masks the unconditional CFG row and needs use_cfg", fn);
    LG_REQUIRE(!neg_mask || emb_mask, "%s: neg_mask needs emb_mask (all ones for an unmasked condition)", fn);
    const int nh = use_cfg ? 2 : 1, D = c.dim, V = c.vocab_size, T = c.cls_token_num, W = std::min(K + 1, kGivenWindowRows);
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    LG_REQUIRE(e->finalized, "%s: engine not finalized", fn);
    LG_TRY(check_ready(e, nh * B, T + a + K));
    RowBuffers win, hb;
    int32_t *win_tokens, *win_pos;
    const size_t need = carve_slot_extend(e, win, &win_tokens, &win_pos, hb, (char*)dev_ws, nh, W);
    LG_REQUIRE(ws_bytes >= need, "%s: scratch of %zu bytes is too small (%zu)", fn, ws_bytes, need);
    // every chunk's attention at first_row = the slot's row: the window kernel (16-bit cache), the CUDA-core kernel (fp32 or fp8 cache)
    // and, for a chunk of one row, the decode kernel all address the cache from first_row through make_attn_args
    for (int c0 = 0, n = 0; c0 < K + 1; c0 += n) {
        n = std::min(W, K + 1 - c0);
        KvCache kv = e->full;
        kv.first_row = slot;
        AttnArgs aa = e->attn_args(kv, 0, 1, n);
        aa.pos = PosArg{nullptr, 0, win_pos};
        const AttnPlan p = attn_plan(aa);
        LG_REQUIRE(p.kernel >= 0, "%s: %s", fn, p.error);
    }
    DeviceGuard guard(e->device);
    LG_TRY(e->zero_fill_if_needed(st));
    for (int half = 0; half < nh; ++half) {
        Workspace w;
        static_cast<KvCache&>(w) = e->full;
        static_cast<RowBuffers&>(w) = win;
        w.first_row = half * B + slot;
        LG_TRY(extend_window(e, w, win_tokens, win_pos, nullptr, tokens, 1, 1, S, T, a, K, W, half != 0 && neg_mask ? neg_mask : emb_mask,
                             nullptr, hb.q + (size_t)half * D * e->esz, st));
    }
    Workspace w;
    static_cast<RowBuffers&>(w) = hb;
    GemmNext nx_first{e->layers[0].wqkv.p, e->layers[0].wqkv.bytes(3 * D, D, e->esz), nullptr, 0};
    LG_TRY(e->head(w, hb.q, nh, logits_out, &nx_first, st));
    return round_logits_inplace(logits_out, (size_t)nh * V, c.dtype, st);
}

static int generate_impl(lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T, int S,
                         const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher,
                         const PrefixArgs& pa, const lg_logprobs* lp, cudaStream_t st0, const Compose& cp) {
    LG_REQUIRE(cond && sc && out_tokens && B > 0 && S > 0 && cp.K >= 1 && B % cp.K == 0, "lg_generate: bad argument");
    const bool use_cfg = uses_cfg(sc, cp);  // generate.py:128
    const int K = cp.K;   // rows per image and half; B rows per half are B / K images
    const int R = use_cfg ? 2 * B : B;
    LG_TRY(check_ready(e, R, T + S));
    LG_REQUIRE(T == e->cfg.cls_token_num, "lg_generate: T=%d must equal cls_token_num=%d", T, e->cfg.cls_token_num);
    if (emb_mask) LG_REQUIRE(e->cfg.model_type == LG_MODEL_T2I, "emb_masks only apply to t2i models");
    const lg_model_cfg& c = e->cfg;

    // Multi-chain decode: at large batch every kernel of a decode step is latency-bound (a few microseconds of
    // dependent load -> compute -> store), so the batch is cut into n_sub independent chains (the chain-count policy of
    // lg_engine_set_workspace, which LG_SPLIT overrides; each chain has its own KV-cache slice, stream and CUDA graph) whose kernels interleave on the GPU. Each image's arithmetic is unchanged, so the result
    // is bit-identical to the single-chain run. A chain never splits an image's K rows.
    const bool split = e->n_sub >= 2 && lg_env_flag("LG_SPLIT", 2) >= 2 && R == e->full.rows && (B / K) % e->n_sub == 0 &&
                       !prof_enabled() && !lg_debug_sync();
    const int nchains = split ? e->n_sub : 1;
    Chain ch[lg_engine::kMaxChains];
    for (int g = 0; g < nchains; ++g) {
        Chain& k = ch[g];
        k.w = split ? e->sub[g] : e->full;
        k.st = g == 0 ? st0 : e->works[g];
        k.B = B / nchains;
        k.R = R / nchains;
        const size_t boff = (size_t)g * k.B, ioff = boff / K;   // the chain's first row and first image
        k.cond = c.model_type == LG_MODEL_C2I ? (const void*)((const int32_t*)cond + boff)
                                              : (const void*)((const char*)cond + boff * T * c.caption_dim * e->esz);
        k.emb_mask = emb_mask ? emb_mask + boff * T : nullptr;
        k.neg.cond = neg.cond ? (const void*)((const char*)neg.cond + boff * T * c.caption_dim * e->esz) : nullptr;
        k.neg.mask = neg.mask ? neg.mask + boff * T : nullptr;
        k.prefix = pa.prefix ? pa.prefix + boff * pa.P : nullptr;
        k.sa = make_sample_args(*sc, k.w.logits, k.B, c.vocab_size, use_cfg, c.dtype);
        SampleArgs& sa = k.sa;
        sa.row_offset = (int)boff;
        sa.out_seq = out_tokens + ioff * S; sa.seq_stride = S; sa.next_tokens = k.w.tokens;
        sa.teacher = teacher ? teacher + ioff * S : nullptr;
        sa.given = pa.given ? pa.given + boff * S : nullptr;
        sa.dbg_logits = dbg_logits; sa.dbg_batch = B;
        if (cp.weights) { sa.mix_groups = K; sa.mix_weights = cp.weights + boff; }
        // the chain's image b is image ioff + b of the call
        if (sa.temp_rows) sa.temp_rows += ioff;
        if (sa.topk_rows) sa.topk_rows += ioff;
        if (sa.topp_rows) sa.topp_rows += ioff;
        if (sa.greedy_rows) sa.greedy_rows += ioff;
        apply_logprobs(sa, lp, ioff * S);
    }
    std::vector<GivenSeg> lead_decode;   // lg_generate and lg_generate_prefix: LEAD P, then one DECODE run to the end
    if (!pa.segs) {
        lead_decode.push_back({kSegLead, 0, pa.P});
        if (S > pa.P + 1) lead_decode.push_back({kSegDecode, pa.P + 1, S - pa.P - 1});
    }
    const std::vector<GivenSeg>& segs = pa.segs ? *pa.segs : lead_decode;
    for (int g = 0, off = 0; pa.W > 0 && g < nchains; ++g) {
        Chain& k = ch[g];
        off += (int)e->carve_given_window(k.win, &k.win_tokens, &k.win_pos, pa.window + off, k.B, use_cfg ? 2 : 1, pa.W);
    }

    // Fused tail (bf16 / fp16): the sample kernel writes the next step's input rows (token embedding, and on the batched path the layer-0
    // RMSNorm) and advances the device-resident counters, so a decode iteration loses its embed / rmsnorm / advance kernels.
    const bool fuse_tail = lg_dtype_is16(c.dtype) && lg_env_flag("LG_FUSE_TAIL", 1) && c.dim % 2 == 0;
    auto arm_tail = [&](Chain& k, bool advance) {
        SampleArgs& sa = k.sa;
        const bool small = e->small_row_path(k.R, e->attn_args(k.w, 0, k.R, 1));
        sa.emb_table = e->tok_emb; sa.emb_h = k.w.h; sa.emb_D = c.dim; sa.emb_rows = k.R;
        sa.emb_xn = small ? nullptr : k.w.xn;
        sa.emb_norm_w = e->layers[0].attn_norm; sa.emb_eps = c.norm_eps;
        sa.adv_pos = advance ? k.w.counters : nullptr;
        sa.adv_step = advance ? k.w.counters + 1 : nullptr;
        sa.adv_ticket = advance ? reinterpret_cast<unsigned int*>(k.w.counters + 64) : nullptr;
    };
    // eager: the step is launched outside graph capture. Its first kernel is then launched without PDL, so it starts only after the
    // previous kernel (the sample kernel, whose fused tail advances the position counter at its very end, or set_counters) has
    // completed; the fused decode attention reads that counter before its dependency wait (DESIGN §4, "Reads before the dependency
    // wait"). In a captured step the graph orders its first node after everything launched before the graph.
    auto body = [&](Chain& k, bool eager) -> int {
        int* d_pos = k.w.counters;
        int* d_step = k.w.counters + 1;
        // with the fused tail the previous iteration's sample kernel left h (and xn) in place
        if (!fuse_tail)
            LG_PROF(PC_EMBED_MISC, k.st, launch_embed(e->tok_emb, k.w.tokens, k.B, k.R, -1, c.dim, c.dtype, k.w.h, k.st, !eager));
        const bool xn_ready = fuse_tail && k.sa.emb_xn != nullptr;
        LG_TRY(e->forward(k.w, k.R, 1, PosArg{d_pos, 0}, k.emb_mask, k.neg.mask, k.B, k.w.logits, xn_ready, k.st, !eager || !fuse_tail));
        LG_PROF(PC_SAMPLE, k.st, launch_sample(k.sa, k.st));
        if (!fuse_tail) LG_PROF(PC_EMBED_MISC, k.st, launch_advance(d_pos, d_step, k.st));
        return 0;
    };
    // An extend pass (lg_generate_given): tokens a - 1 .. a + K - 1 of every row, at positions T + a - 1 .., through the layers in
    // window chunks of at most pa.W rows (their K / V go to the chain's cache); the head over the last row of every image's window
    // gives the logits of token a + K, which is drawn (or taken as given) with its own step, and the counters move past it
    auto extend = [&](Chain& k, int a, int K) -> int {
        const int D = c.dim;
        Workspace w;
        static_cast<KvCache&>(w) = k.w;
        static_cast<RowBuffers&>(w) = k.win;
        LG_TRY(extend_window(e, w, k.win_tokens, k.win_pos, k.w.tokens, k.sa.given, k.B, use_cfg ? 2 : 1, S, T, a, K, pa.W, k.emb_mask,
                             k.neg.mask, w.q, k.st));
        GemmNext nx_first{e->layers[0].wqkv.p, e->layers[0].wqkv.bytes(3 * D, D, e->esz), nullptr, 0};
        LG_TRY(e->head(w, w.q, k.R, k.w.logits, &nx_first, k.st));
        SampleArgs sa = k.sa;   // the decode step's draw at a fixed step; the counters are set, not advanced
        sa.step = a + K; sa.step_dev = nullptr; sa.adv_pos = nullptr; sa.adv_step = nullptr; sa.adv_ticket = nullptr;
        LG_PROF(PC_SAMPLE, k.st, launch_sample(sa, k.st));
        return launch_set_counters(k.w.counters, T + a + K, k.w.counters + 1, a + K + 1, k.st);
    };

    // ---- prefix prefill (lg_generate_prefix): tokens 0 .. P - 1 are the prefix; every chain's prefill shares the one scratch, so all
    // of them run on the caller's stream, in chunks of the most rows that fit the scratch and the attention kernel's grid
    const int P = pa.P;
    if (P > 0) {
        const int nh = use_cfg ? 2 : 1, seq = T + P;
        auto fits = [&](int n) {
            RowBuffers rb;
            if (e->carve_prefix(rb, nullptr, n, seq) > pa.scratch_bytes) return false;
            return attn_plan(e->attn_args(ch[0].w, 0, n, seq)).kernel >= 0;
        };
        const int blk = (B / K) % lg_engine::kMaxChains == 0 ? B / lg_engine::kMaxChains : B;   // one chain's rows under the largest split
        int lo = 1, hi = blk;       // largest chunk that fits
        while (lo < hi) {
            const int mid = lo + (hi - lo + 1) / 2;
            if (fits(mid)) lo = mid; else hi = mid - 1;
        }
        LG_REQUIRE(fits(lo), "lg_generate_prefix: no chunk of rows fits the scratch (%zu bytes) and the attention grid", pa.scratch_bytes);
        LG_CUDA_OK(cudaMemcpy2DAsync(out_tokens, (size_t)S * sizeof(int32_t), pa.prefix, (size_t)K * P * sizeof(int32_t),
                                     (size_t)P * sizeof(int32_t), B / K, cudaMemcpyDeviceToDevice, st0));   // row j K of image j
        if (lp) LG_TRY(launch_given_logprobs(lp->logprob, lp->rank, lp->top_n > 0 ? lp->top_ids : nullptr,
                                             lp->top_n > 0 ? lp->top_logprob : nullptr, lp->top_n, B / K, S, P, st0));
        e->prefix_chunks = 0;
        e->prefix_chains = nchains;
        for (int g = 0; g < nchains; ++g) LG_TRY(prefix_prefill(e, ch[g], nh, T, P, lo, blk, pa, st0));
        if (nchains > 1) {
            LG_CUDA_OK(cudaEventRecord(e->ev_prefill, st0));
            for (int g = 1; g < nchains; ++g) LG_CUDA_OK(cudaStreamWaitEvent(ch[g].st, e->ev_prefill, 0));
        }
    }
    // ---- prefill (generate.py:167-169) + first decode step, eagerly, per chain; token P is sampled first (0 without a prefix)
    for (int g = 0; g < nchains; ++g) {
        Chain& k = ch[g];
        if (P == 0) {
            LG_TRY(e->embed_cond(k.w, k.cond, k.neg.cond, k.B, k.R, T, k.st));
            LG_TRY(e->forward(k.w, k.R * T, T, PosArg{nullptr, 0}, k.emb_mask, k.neg.mask, k.B, k.w.logits, false, k.st));
        }
        k.sa.step = P; k.sa.step_dev = nullptr;
        const bool tail = S > P + 1 && fuse_tail;
        if (tail) arm_tail(k, false);            // the prefill's sample prepares the first decode step's rows; counters are set below
        LG_TRY(launch_sample(k.sa, k.st));
        if (S == P + 1) continue;
        LG_TRY(launch_set_counters(k.w.counters, T + P, k.w.counters + 1, P + 1, k.st));
        k.sa.step_dev = k.w.counters + 1;
        if (tail) arm_tail(k, true);
    }
    // ---- the plan's other segments, every chain in turn. The first decode step runs eagerly (it also sets every kernel attribute
    // outside capture); the later ones replay, per chain, one captured graph of one decode step (generate.py:105-123; the loop state is
    // device-resident, so every step has identical kernel arguments), chains interleaved: with two chains the gap between graph
    // launches of one chain is covered by the other chain's kernels.
    int remaining = -1;   // decode steps after the first
    for (const GivenSeg& sg : segs)
        if (sg.kind == kSegDecode) remaining += sg.len;
    const bool graph = e->use_graph && remaining >= 3 && !prof_enabled() && !lg_debug_sync();
    bool eager_done = false, captured = false;
    for (const GivenSeg& sg : segs) {
        if (sg.kind == kSegExtend)
            for (int g = 0; g < nchains; ++g) LG_TRY(extend(ch[g], sg.start, sg.len));
        if (sg.kind != kSegDecode) continue;
        for (int i = 0; i < sg.len; ++i) {
            if (!eager_done || !graph) {
                for (int g = 0; g < nchains; ++g) LG_TRY(body(ch[g], true));
                eager_done = true;
                continue;
            }
            if (!captured)
                for (int g = 0; g < nchains; ++g) LG_TRY(ch[g].graph.capture(ch[g].st, [&] { return body(ch[g], false); }));
            captured = true;
            for (int g = 0; g < nchains; ++g) LG_TRY(ch[g].graph.launch(ch[g].st));
        }
    }
    return 0;
}

int lg_sjd_workspace_bytes(lg_engine* e, int B, int use_cfg, int L, size_t* bytes) {
    LG_REQUIRE(e && bytes && B > 0 && L >= 2 && L <= 64, "lg_sjd_workspace_bytes: bad argument (B=%d L=%d)", B, L);
    Workspace w;
    SjdArgs sa{};
    *bytes = e->carve_sjd(w, sa, nullptr, B, use_cfg ? 2 : 1, L);
    return 0;
}

static int generate_sjd_impl(lg_engine* e, const Workspace& w, SjdArgs& sa, const void* cond, const float* emb_mask, const Negative& neg,
                             const lg_sample_cfg& sc, bool use_cfg, int32_t* iters_out, cudaStream_t st) {
    const lg_model_cfg& c = e->cfg;
    const int B = sa.B, S = sa.S, L = sa.L, T = sa.T, V = c.vocab_size, D = c.dim, dt = c.dtype, R = sa.nh * B, M = R * L;
    static int calls = 0;
    sa.done_token = ++calls;   // a pass still in flight from an earlier call cannot end this one
    LG_CUDA_OK(cudaMemsetAsync(sa.state, 0, kSjdStateInts * sizeof(int32_t), st));
    // prefill and token 0, drawn as lg_generate draws it
    LG_TRY(e->embed_cond(e->full, cond, neg.cond, B, R, T, st));
    LG_TRY(e->forward(e->full, R * T, T, PosArg{nullptr, 0}, emb_mask, neg.mask, B, e->full.logits, false, st));
    SampleArgs s0 = make_sample_args(sc, e->full.logits, B, V, use_cfg, dt);
    s0.step = 0; s0.out_seq = sa.out; s0.seq_stride = S;
    LG_TRY(launch_sample(s0, st));
    LG_TRY(launch_sjd_refresh(sa, 1, st));
    // one pass: window embedding, the layers over R * L rows at per-row positions, the head over every row, p and x for every slot
    // (B * L images, CFG twins at rows b * L + i and (B + b) * L + i), acceptance, next window
    SampleArgs sp = make_sample_args(sc, w.logits, B * L, V, use_cfg, dt);
    sp.param_div = L;   // window rows b * L .. b * L + L - 1 are image b's
    sp.seed_rows = sa.seed_rows; sp.step_rows = sa.step_rows;
    sp.out_idx = const_cast<int32_t*>(sa.x); sp.out_probs = const_cast<float*>(sa.p);
    auto pass = [&]() -> int {
        LG_PROF(PC_EMBED_MISC, st, launch_embed(e->tok_emb, sa.win, B * L, M, -1, D, dt, w.h, st));
        LG_TRY(e->run_layers(w, M, L, PosArg{nullptr, 0, sa.pos_rows}, emb_mask, neg.mask, B, false, st));
        LG_TRY(e->head(w, w.xn, M, w.logits, nullptr, st));
        LG_PROF(PC_SAMPLE, st, launch_sample(sp, st));
        LG_PROF(PC_SAMPLE, st, launch_sjd_verify(sa, st));
        LG_PROF(PC_SAMPLE, st, launch_sjd_refresh(sa, 0, st));
        LG_CUDA_OK(cudaMemcpyAsync(e->sjd_done_host, sa.state + kSjdDone, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        return 0;
    };
    // Every pass has the same kernel arguments (the loop state is on the device), so one captured graph is replayed. The host reads
    // pass j - 1's done flag after it has enqueued pass j: the GPU never waits for the host, and at most one pass runs after the last
    // image finished (a no-op: finished images are frozen). At most S - 1 passes: each one makes at least one token final.
    LG_TRY(pass());   // eagerly first: sets every kernel attribute outside capture
    LG_CUDA_OK(cudaEventRecord(e->ev_pass[0], st));
    const bool use_graph = e->use_graph && !prof_enabled() && !lg_debug_sync() && S - 1 > 2;
    Graph graph;
    if (use_graph) LG_TRY(graph.capture(st, pass));
    for (int launched = 1; launched < S - 1; ++launched) {
        LG_TRY(use_graph ? graph.launch(st) : pass());
        cudaError_t ce = cudaEventRecord(e->ev_pass[launched & 1], st);
        if (ce == cudaSuccess) ce = cudaEventSynchronize(e->ev_pass[(launched - 1) & 1]);
        if (ce != cudaSuccess) return lg_fail("lg_generate_sjd: waiting for a pass failed: %s", cudaGetErrorString(ce));
        if (*(volatile int*)e->sjd_done_host == sa.done_token) break;
    }
    LG_CUDA_OK(cudaMemcpyAsync(iters_out, sa.state + kSjdIters, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // extern "C"

static int generate_sjd_entry(const char* fn, lg_engine* e, const void* cond, const float* emb_mask, const Negative& neg, int B, int T, int S,
                              const lg_sample_cfg* sc, int L, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* iters_out,
                              float* dbg_probs, void* stream) {
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    DeviceGuard guard(e->device);
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(cond && sc && out_tokens && iters_out && B > 0, "%s: null argument or B=%d", fn, B);
    LG_REQUIRE(L >= 2 && L <= 64, "%s: window L=%d outside [2, 64]", fn, L);
    LG_REQUIRE(S > L && S <= c.block_size, "%s: S=%d must lie in [L + 1, block_size=%d] (L=%d)", fn, S, c.block_size, L);
    LG_REQUIRE(T == c.cls_token_num, "%s: T=%d must equal cls_token_num=%d", fn, T, c.cls_token_num);
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    LG_REQUIRE((size_t)c.vocab_size * sizeof(float) <= 200 * 1024, "%s: vocab %d too large for the sampler", fn, c.vocab_size);
    const bool use_cfg = sc->cfg_scale > 1.0f;   // generate.py:128
    LG_TRY(check_negative(fn, e, neg, emb_mask, use_cfg));
    const int nh = use_cfg ? 2 : 1, R = nh * B;
    LG_TRY(check_ready(e, R, T + S));
    LG_REQUIRE((long long)R * L <= 65535, "%s: %d rows x window %d exceed 65535 query rows", fn, R, L);
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    Workspace w;   // the KV cache and its maps of the workspace, the row buffers of the scratch
    SjdArgs sa{};
    const size_t need = e->carve_sjd(w, sa, (char*)dev_ws, B, nh, L);
    LG_REQUIRE(ws_bytes >= need, "%s: scratch of %zu bytes is too small (%zu)", fn, ws_bytes, need);
    static_cast<KvCache&>(w) = e->full;
    sa.B = B; sa.S = S; sa.L = L; sa.V = c.vocab_size; sa.T = T; sa.nh = nh;
    sa.greedy = sc->greedy; sa.greedy_rows = sc->greedy_rows; sa.seed = sc->seed; sa.row_offset = 0;
    sa.out = out_tokens; sa.dbg = dbg_probs;
    if (!e->sjd_done_host) {
        LG_CUDA_OK(cudaHostAlloc((void**)&e->sjd_done_host, sizeof(int), cudaHostAllocDefault));
        *e->sjd_done_host = 0;
        for (cudaEvent_t& ev : e->ev_pass) LG_CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    return e->run_forked((cudaStream_t)stream, 1, [&](cudaStream_t st) {
        return generate_sjd_impl(e, w, sa, cond, emb_mask, neg, *sc, use_cfg, iters_out, st);
    });
}

extern "C" {

int lg_generate_sjd(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc, int L,
                    void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* iters_out, float* dbg_probs, void* stream) {
    return generate_sjd_entry("lg_generate_sjd", e, cond, emb_mask, Negative{}, B, T, S, sc, L, dev_ws, ws_bytes, out_tokens, iters_out,
                              dbg_probs, stream);
}

int lg_generate_sjd_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                        int S, const lg_sample_cfg* sc, int L, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* iters_out,
                        float* dbg_probs, void* stream) {
    return generate_sjd_entry("lg_generate_sjd_neg", e, cond, emb_mask, Negative{neg_cond, neg_mask}, B, T, S, sc, L, dev_ws, ws_bytes,
                              out_tokens, iters_out, dbg_probs, stream);
}

}  // extern "C"

// The checks every per-slot SJD entry fn makes of its shape (S: 0 when the entry takes none) and scratch, then sa and w over dev_ws:
// the slot state and row buffers of the scratch, the KV cache of the workspace
static int sjd_slots_view(const char* fn, lg_engine* e, int B, int use_cfg, int L, int S, void* dev_ws, size_t ws_bytes, Workspace& w,
                          SjdArgs& sa) {
    LG_REQUIRE(B > 0, "%s: B=%d", fn, B);
    LG_REQUIRE(L >= 2 && L <= 64, "%s: window L=%d outside [2, 64]", fn, L);
    LG_REQUIRE(S == 0 || S > L, "%s: S=%d must exceed the window L=%d", fn, S, L);
    LG_REQUIRE(dev_ws && ((uintptr_t)dev_ws & 255) == 0, "%s: scratch must be non-null and 256-byte aligned", fn);
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    const lg_model_cfg& c = e->cfg;
    const int nh = use_cfg ? 2 : 1;
    LG_REQUIRE(S <= c.block_size, "%s: S=%d exceeds block_size=%d", fn, S, c.block_size);
    LG_REQUIRE((size_t)c.vocab_size * sizeof(float) <= 200 * 1024, "%s: vocab %d too large for the sampler", fn, c.vocab_size);
    LG_REQUIRE((long long)nh * B * L <= 65535, "%s: %d rows x window %d exceed 65535 query rows", fn, nh * B, L);
    LG_TRY(check_ready(e, nh * B, c.cls_token_num + std::max(S, L + 1)));
    const size_t need = e->carve_sjd_slots(w, sa, (char*)dev_ws, B, nh, L);
    LG_REQUIRE(ws_bytes >= need, "%s: scratch of %zu bytes is too small (%zu)", fn, ws_bytes, need);
    static_cast<KvCache&>(w) = e->full;
    sa.B = B; sa.S = S; sa.L = L; sa.V = c.vocab_size; sa.T = c.cls_token_num; sa.nh = nh; sa.row_offset = 0;
    if (!use_cfg) { sa.cfg_rows = nullptr; sa.interval_rows = nullptr; }
    return 0;
}

extern "C" {

int lg_sjd_slots_workspace_bytes(lg_engine* e, int B, int use_cfg, int L, size_t* bytes) {
    LG_REQUIRE(e && bytes && B > 0 && L >= 2 && L <= 64, "lg_sjd_slots_workspace_bytes: bad argument (B=%d L=%d)", B, L);
    Workspace w;
    SjdArgs sa{};
    *bytes = e->carve_sjd_slots(w, sa, nullptr, B, use_cfg ? 2 : 1, L);
    return 0;
}

int lg_sjd_slots_reset(lg_engine* e, int B, int use_cfg, int L, void* dev_ws, size_t ws_bytes, void* stream) {
    Workspace w;
    SjdArgs sa{};
    LG_TRY(sjd_slots_view("lg_sjd_slots_reset", e, B, use_cfg, L, 0, dev_ws, ws_bytes, w, sa));
    cudaStream_t st = (cudaStream_t)stream;
    DeviceGuard guard(e->device);
    // zeros everywhere (valid window tokens and positions for the rows of free slots), then nfin = 0x7f7f7f7f: every slot frozen
    RowBuffers rb;
    SjdArgs sizes{};
    LG_CUDA_OK(cudaMemsetAsync(dev_ws, 0, e->carve_sjd_slots(rb, sizes, nullptr, B, sa.nh, L), st));
    LG_CUDA_OK(cudaMemsetAsync(sa.nfin, 0x7f, (size_t)B * sizeof(int32_t), st));
    return 0;
}

int lg_test_scratch_regions(lg_engine* e, int kind, const int64_t* args, int nargs, const int32_t* given, int64_t* out, int cap) {
    static const char* fn = "lg_test_scratch_regions";
    static const int kArgs[] = {2, 2, 2, 1, 2, 2, 4, 3, 3};   // arguments of each kind (the workspace also takes 4: its chain view)
    LG_REQUIRE(e && args && (out || cap == 0) && cap >= 0, "%s: bad argument", fn);
    LG_REQUIRE(kind >= 0 && kind <= 8 && (nargs == kArgs[kind] || (kind == 0 && nargs == 4)), "%s: kind %d with %d arguments", fn, kind,
               nargs);
    int a[4] = {0, 0, 0, 0};
    for (int i = 0; i < nargs; ++i) {
        LG_REQUIRE(args[i] >= 0 && args[i] <= INT32_MAX, "%s: argument %d = %lld", fn, i, (long long)args[i]);
        a[i] = (int)args[i];
    }
    // the same checks as the kind's *_workspace_bytes, before anything is logged
    size_t bytes = 0;
    std::vector<GivenSeg> segs;
    size_t fixed = 0, prefill = 0;
    switch (kind) {
        case 0: LG_TRY(lg_engine_workspace_bytes(e, a[0], a[1], &bytes));
                LG_REQUIRE(nargs == 2 || (a[3] >= 1 && a[3] <= lg_engine::kMaxChains && a[2] < a[3] && a[0] % a[3] == 0),
                           "%s: chain %d of %d over %d rows", fn, a[2], a[3], a[0]);
                break;
        case 1: LG_TRY(lg_score_workspace_bytes(e, a[0], a[1], &bytes)); break;
        case 2: LG_TRY(lg_prefix_workspace_bytes(e, a[0], a[1], &bytes)); break;
        case 3: LG_TRY(lg_slot_workspace_bytes(e, a[0], &bytes)); break;
        case 4: LG_TRY(lg_slot_prefix_workspace_bytes(e, a[0], a[1], &bytes)); break;
        case 5: LG_TRY(lg_slot_extend_workspace_bytes(e, a[0], a[1], &bytes)); break;
        case 6: LG_TRY(given_layout(fn, e, given, a[0], a[1], a[2] ? 2 : 1, segs, &fixed, &prefill));
                LG_REQUIRE(a[3] >= 1 && a[3] <= lg_engine::kMaxChains && a[0] % a[3] == 0, "%s: %d chains over B=%d", fn, a[3], a[0]);
                break;
        case 7: LG_TRY(lg_sjd_workspace_bytes(e, a[0], a[1], a[2], &bytes)); break;
        case 8: LG_TRY(lg_sjd_slots_workspace_bytes(e, a[0], a[1], a[2], &bytes)); break;
    }
    RegionLog log;
    t_region_log = &log;
    Workspace w;
    SjdArgs sa{};
    RowBuffers rb, head;
    int32_t *win = nullptr, *pos = nullptr;
    switch (kind) {
        case 0: e->carve(w, nullptr, a[0], a[1], a[2], nargs == 4 ? a[3] : 1); break;
        case 1: e->carve_score(w, nullptr, a[0], a[1]); break;
        case 2: e->carve_prefix(rb, nullptr, a[0], a[1]); break;
        case 3: e->carve_slot(rb, nullptr, a[0] ? 2 : 1, e->cfg.cls_token_num); break;
        case 4: e->carve_slot(rb, nullptr, a[0] ? 2 : 1, e->cfg.cls_token_num + a[1]); break;
        case 5: carve_slot_extend(e, rb, &win, &pos, head, nullptr, a[0] ? 2 : 1, std::min(a[1] + 1, kGivenWindowRows)); break;
        case 6: {   // generate_given_impl's scratch: given [B, S], the leading run [B, P], the windows of a[3] chains, the prefill
            const int B = a[0], S = a[1], nh = a[2] ? 2 : 1, n = a[3], P = segs[0].len, W = given_window_rows(segs);
            Carver c{nullptr};
            c.split((size_t)B * S * sizeof(int32_t), kRegionInt);
            c.split((size_t)B * P * sizeof(int32_t), kRegionInt);
            for (int g = 0; W > 0 && g < n; ++g) {
                log.shift = c.off;
                log.chain = g;
                c.off += e->carve_given_window(rb, &win, &pos, nullptr, B / n, nh, W);
            }
            log.shift = fixed;
            log.chain = -1;
            if (P > 0) e->carve_prefix(rb, nullptr, nh * B, e->cfg.cls_token_num + P);
            break;
        }
        case 7: e->carve_sjd(rb, sa, nullptr, a[0], a[1] ? 2 : 1, a[2]); break;
        case 8: e->carve_sjd_slots(rb, sa, nullptr, a[0], a[1] ? 2 : 1, a[2]); break;
    }
    t_region_log = nullptr;
    const int count = (int)(log.rows.size() / 4);
    std::copy(log.rows.begin(), log.rows.begin() + 4 * std::min(count, cap), out);
    return count;
}

}  // extern "C"

// lg_sjd_slot_start (image 0) and lg_sjd_slot_start_image; fn names the entry point in messages
static int sjd_slot_start_impl(const char* fn, lg_engine* e, int slot, int B, int use_cfg, int L, int S, uint64_t seed, float cfg_scale,
                               int cfg_interval, int image, const int32_t* out_tokens, void* dev_ws, size_t ws_bytes, void* stream) {
    LG_REQUIRE(out_tokens, "%s: null out_tokens", fn);
    LG_REQUIRE(slot >= 0 && slot < B, "%s: slot %d outside [0, B=%d)", fn, slot, B);
    LG_REQUIRE(image >= 0 && image < 0x7fffffff, "%s: image %d outside [0, 2^31 - 1)", fn, image);
    LG_REQUIRE(S > 0, "%s: S=%d", fn, S);
    LG_REQUIRE(std::isfinite(cfg_scale) && cfg_interval >= -1, "%s: cfg_scale %g must be finite and cfg_interval %d >= -1", fn,
               (double)cfg_scale, cfg_interval);
    Workspace w;
    SjdArgs sa{};
    LG_TRY(sjd_slots_view(fn, e, B, use_cfg, L, S, dev_ws, ws_bytes, w, sa));
    DeviceGuard guard(e->device);
    sa.seed = seed; sa.start_cfg = cfg_scale; sa.start_interval = cfg_interval; sa.start_img = image;
    sa.out = const_cast<int32_t*>(out_tokens);   // read only: token 0 of the slot's row
    return launch_sjd_refresh(sa, 1, (cudaStream_t)stream, slot);
}

extern "C" {

int lg_sjd_slot_start(lg_engine* e, int slot, int B, int use_cfg, int L, int S, uint64_t seed, float cfg_scale, int cfg_interval,
                      const int32_t* out_tokens, void* dev_ws, size_t ws_bytes, void* stream) {
    return sjd_slot_start_impl("lg_sjd_slot_start", e, slot, B, use_cfg, L, S, seed, cfg_scale, cfg_interval, 0, out_tokens, dev_ws,
                               ws_bytes, stream);
}

int lg_sjd_slot_start_image(lg_engine* e, int slot, int B, int use_cfg, int L, int S, uint64_t seed, float cfg_scale, int cfg_interval,
                            int image, const int32_t* out_tokens, void* dev_ws, size_t ws_bytes, void* stream) {
    return sjd_slot_start_impl("lg_sjd_slot_start_image", e, slot, B, use_cfg, L, S, seed, cfg_scale, cfg_interval, image, out_tokens,
                               dev_ws, ws_bytes, stream);
}

int lg_copy_slot_kv(lg_engine* e, int src_slot, const int32_t* dst_slots, int n_dst, int B, int use_cfg, int len, void* stream) {
    static const char* fn = "lg_copy_slot_kv";
    LG_REQUIRE(n_dst >= 0 && (n_dst == 0 || dst_slots), "%s: n_dst=%d with %s dst_slots", fn, n_dst, dst_slots ? "non-null" : "null");
    LG_REQUIRE(B > 0 && src_slot >= 0 && src_slot < B, "%s: source slot %d outside [0, B=%d)", fn, src_slot, B);
    for (int i = 0; i < n_dst; ++i) {
        const int d = dst_slots[i];
        LG_REQUIRE(d >= 0 && d < B, "%s: destination slot %d outside [0, B=%d)", fn, d, B);
        LG_REQUIRE(d != src_slot, "%s: destination slot %d is the source", fn, d);
        for (int j = 0; j < i; ++j) LG_REQUIRE(dst_slots[j] != d, "%s: destination slot %d repeated", fn, d);
    }
    LG_REQUIRE(len >= 0, "%s: len %d < 0", fn, len);
    LG_REQUIRE(e && e->finalized, "%s: engine not finalized", fn);
    LG_REQUIRE(e->full.base, "%s: workspace not set", fn);
    const int nh = use_cfg ? 2 : 1;
    LG_REQUIRE(nh * B <= e->full.rows, "%s: %d rows (nh=%d, B=%d) exceed the workspace's %d", fn, nh * B, nh, B, e->full.rows);
    LG_REQUIRE(len <= e->full.max_seq, "%s: len %d exceeds the workspace's max_seq %d", fn, len, e->full.max_seq);
    cudaStream_t st = (cudaStream_t)stream;
    DeviceGuard guard(e->device);
    LG_TRY(e->zero_fill_if_needed(st));
    // fp8 scales are per layer, shared by every row: the codes alone are copied
    KvCopyArgs a{};
    a.kcache = e->full.kcache; a.vcache = e->full.vcache;
    a.layers = e->full.layers; a.rows = e->full.rows; a.H = e->cfg.n_head; a.max_seq = e->full.max_seq;
    a.row_bytes = e->hdp * (e->full.kv_f8 ? 1 : (int)e->esz);
    a.B = B; a.nh = nh; a.len = len; a.src = src_slot;
    for (int d0 = 0; d0 < n_dst; d0 += kKvCopyMaxDst) {
        a.n_dst = std::min(kKvCopyMaxDst, n_dst - d0);
        for (int i = 0; i < a.n_dst; ++i) a.dst[i] = dst_slots[d0 + i];
        LG_TRY(launch_copy_slot_kv(a, st));
    }
    return 0;
}

}  // extern "C"

extern "C" {

int lg_sjd_pass_slots(lg_engine* e, const lg_sample_cfg* sc, const float* emb_mask, const float* neg_mask, int B, int use_cfg, int S, int L,
                      void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* nfin_out, float* dbg_p, void* stream) {
    static const char* fn = "lg_sjd_pass_slots";
    LG_REQUIRE(sc && out_tokens && nfin_out, "%s: null argument", fn);
    LG_REQUIRE(S > 0, "%s: S=%d", fn, S);
    LG_REQUIRE(!neg_mask || use_cfg, "%s: neg_mask masks the unconditional CFG rows and needs use_cfg", fn);
    LG_REQUIRE(!neg_mask || emb_mask, "%s: neg_mask needs emb_mask (all ones for an unmasked condition)", fn);
    Workspace w;
    SjdArgs sa{};
    LG_TRY(sjd_slots_view(fn, e, B, use_cfg, L, S, dev_ws, ws_bytes, w, sa));
    const lg_model_cfg& c = e->cfg;
    LG_REQUIRE(!emb_mask || c.model_type == LG_MODEL_T2I, "%s: emb_mask only applies to t2i models", fn);
    const int V = c.vocab_size, D = c.dim, dt = c.dtype, M = sa.nh * B * L;
    cudaStream_t st = (cudaStream_t)stream;
    DeviceGuard guard(e->device);
    LG_TRY(e->zero_fill_if_needed(st));
    sa.greedy = sc->greedy; sa.greedy_rows = sc->greedy_rows; sa.out = out_tokens;
    // generate_sjd_impl's pass over the slots: window embedding, the layers over nh * B * L rows at the slots' positions, the head, p and
    // x of every row with the row's seed, token index and guidance, acceptance, next window
    LG_PROF(PC_EMBED_MISC, st, launch_embed(e->tok_emb, sa.win, B * L, M, -1, D, dt, w.h, st));
    LG_TRY(e->run_layers(w, M, L, PosArg{nullptr, 0, sa.pos_rows}, emb_mask, neg_mask, B, false, st));
    LG_TRY(e->head(w, w.xn, M, w.logits, nullptr, st));
    SampleArgs sp = make_sample_args(*sc, w.logits, B * L, V, use_cfg, dt);
    sp.param_div = L;   // window rows b * L .. b * L + L - 1 are slot b's
    sp.seed_rows = sa.seed_rows; sp.step_rows = sa.step_rows;
    sp.cfg_rows = sa.cfg_rows; sp.interval_rows = sa.interval_rows;
    sp.out_idx = const_cast<int32_t*>(sa.x); sp.out_probs = const_cast<float*>(sa.p);
    LG_PROF(PC_SAMPLE, st, launch_sample(sp, st));
    if (dbg_p) LG_CUDA_OK(cudaMemcpyAsync(dbg_p, sa.p, (size_t)B * L * V * sizeof(float), cudaMemcpyDeviceToDevice, st));
    LG_PROF(PC_SAMPLE, st, launch_sjd_verify(sa, st));
    LG_PROF(PC_SAMPLE, st, launch_sjd_refresh(sa, 0, st));
    LG_CUDA_OK(cudaMemcpyAsync(nfin_out, sa.nfin, (size_t)B * sizeof(int32_t), cudaMemcpyDefault, st));
    return 0;
}

int lg_test_sjd_verify(int B, int S, int L, int V, int greedy, uint64_t seed, const float* p, const float* q, const int32_t* qflag,
                       const int32_t* x, const int32_t* win, int32_t* nfin, int32_t* start, int32_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(p && q && qflag && x && win && nfin && start && out, "lg_test_sjd_verify: null argument");
    LG_REQUIRE(B > 0 && V > 0 && L >= 2 && L <= 64 && S > L, "lg_test_sjd_verify: bad shape B=%d S=%d L=%d V=%d", B, S, L, V);
    SjdArgs sa{};
    sa.B = B; sa.S = S; sa.L = L; sa.V = V; sa.T = 0; sa.nh = 1; sa.greedy = greedy; sa.seed = seed;
    sa.p = p; sa.q = const_cast<float*>(q); sa.qflag = const_cast<int32_t*>(qflag); sa.x = x; sa.win = const_cast<int32_t*>(win);
    sa.nfin = nfin; sa.start = start; sa.out = out; sa.done_token = 1;
    int32_t* tmp = nullptr;   // shift [B], pos_rows [B], loop state
    LG_CUDA_OK(cudaMallocAsync((void**)&tmp, (2 * (size_t)B + kSjdStateInts) * sizeof(int32_t), st));
    LG_CUDA_OK(cudaMemsetAsync(tmp, 0, (2 * (size_t)B + kSjdStateInts) * sizeof(int32_t), st));
    sa.shift = tmp; sa.pos_rows = tmp + B; sa.state = tmp + 2 * B;
    const int rc = launch_sjd_verify(sa, st);
    cudaFreeAsync(tmp, st);
    return rc;
}

int lg_test_sjd_slots(int B, int S, int L, int V, int greedy, const float* p, const int32_t* x, float* q, int32_t* qflag, int32_t* win,
                      int32_t* nfin, int32_t* start, uint64_t* seed_slots, int32_t* pass_slots, uint64_t* seed_rows, int32_t* step_rows,
                      int32_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(p && x && q && qflag && win && nfin && start && seed_slots && pass_slots && seed_rows && step_rows && out,
               "lg_test_sjd_slots: null argument");
    LG_REQUIRE(B > 0 && V > 0 && L >= 2 && L <= 64 && S > L, "lg_test_sjd_slots: bad shape B=%d S=%d L=%d V=%d", B, S, L, V);
    SjdArgs sa{};
    sa.B = B; sa.S = S; sa.L = L; sa.V = V; sa.T = 0; sa.nh = 1; sa.greedy = greedy;
    sa.p = p; sa.q = q; sa.qflag = qflag; sa.x = x; sa.win = win; sa.nfin = nfin; sa.start = start; sa.out = out; sa.done_token = 1;
    sa.seed_slots = seed_slots; sa.pass_slots = pass_slots; sa.seed_rows = seed_rows; sa.step_rows = step_rows;
    int32_t* tmp = nullptr;   // shift [B], pos_rows [B], loop state
    LG_CUDA_OK(cudaMallocAsync((void**)&tmp, (2 * (size_t)B + kSjdStateInts) * sizeof(int32_t), st));
    LG_CUDA_OK(cudaMemsetAsync(tmp, 0, (2 * (size_t)B + kSjdStateInts) * sizeof(int32_t), st));
    sa.shift = tmp; sa.pos_rows = tmp + B; sa.state = tmp + 2 * B;
    int rc = launch_sjd_verify(sa, st);
    if (rc == 0) rc = launch_sjd_refresh(sa, 0, st);
    cudaFreeAsync(tmp, st);
    return rc;
}

int lg_test_sample(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, uint64_t step,
                   const int32_t* step_dev, int row_offset, const uint64_t* seed_rows, const int32_t* step_rows, int32_t* out_idx,
                   float* out_probs, int32_t* out_seq, int seq_stride, const int32_t* teacher, int32_t* next_tokens, float* dbg_logits,
                   int dbg_batch, const void* emb_table, void* emb_h, void* emb_xn, const void* emb_norm_w, float emb_eps, int D,
                   int emb_rows, int32_t* adv_pos, int32_t* adv_step, int32_t* path, int* vec_loads, void* stream) {
    static const char* fn = "lg_test_sample";
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(logits && sc, "%s: null logits or config", fn);
    LG_REQUIRE(B > 0 && V > 0, "%s: bad shape B=%d V=%d", fn, B, V);
    LG_REQUIRE((size_t)V * sizeof(float) <= 200 * 1024, "lg_sample: vocab %d too large for the shared-memory row stage", V);
    LG_REQUIRE(round_dtype == LG_DTYPE_F32 || lg_dtype_is16(round_dtype), "%s: unsupported round dtype %d", fn, round_dtype);
    LG_REQUIRE(((uintptr_t)logits & 3) == 0 && ((uintptr_t)out_probs & 3) == 0 && ((uintptr_t)dbg_logits & 3) == 0,
               "%s: misaligned (4 bytes) f32 buffer", fn);
    LG_REQUIRE(!(step_dev && seed_rows), "%s: step_dev and step_rows both give the step", fn);
    LG_REQUIRE((seed_rows != nullptr) == (step_rows != nullptr), "%s: seed_rows and step_rows go together", fn);
    LG_REQUIRE(row_offset >= 0, "%s: row_offset %d < 0", fn, row_offset);
    LG_REQUIRE(!(out_seq || teacher) || seq_stride > 0, "%s: out_seq / teacher need seq_stride > 0", fn);
    LG_REQUIRE(!teacher || next_tokens || emb_table, "%s: teacher only changes next_tokens and the fused tail", fn);
    LG_REQUIRE(!dbg_logits || (dbg_batch >= 0 && (dbg_batch == 0 ? row_offset == 0 : row_offset + B <= dbg_batch)),
               "%s: dbg rows row_offset + b must lie in dbg_batch (%d)", fn, dbg_batch);
    if (emb_table) {
        LG_REQUIRE(lg_dtype_is16(round_dtype), "lg_sample: the fused tail needs a 16-bit round dtype");
        LG_REQUIRE(emb_h && D > 0 && D % 2 == 0 && emb_rows >= B && (!emb_xn || emb_norm_w),
                   "%s: the fused tail needs emb_h, an even D > 0, emb_rows >= B and emb_norm_w with emb_xn", fn);
        LG_REQUIRE(((uintptr_t)emb_table & 3) == 0 && ((uintptr_t)emb_h & 3) == 0 && ((uintptr_t)emb_xn & 3) == 0 &&
                   ((uintptr_t)emb_norm_w & 3) == 0, "%s: misaligned (4 bytes) fused-tail buffer", fn);
    } else {
        LG_REQUIRE(!emb_h && !emb_xn && !emb_norm_w, "%s: emb_h / emb_xn / emb_norm_w without emb_table", fn);
    }
    SampleArgs a = make_sample_args(*sc, logits, B, V, mix_cfg, round_dtype);
    a.step = step; a.step_dev = step_dev; a.row_offset = row_offset; a.seed_rows = seed_rows; a.step_rows = step_rows;
    a.out_idx = out_idx; a.out_probs = out_probs; a.out_seq = out_seq; a.seq_stride = seq_stride; a.teacher = teacher;
    a.next_tokens = next_tokens; a.dbg_logits = dbg_logits; a.dbg_batch = dbg_batch;
    a.emb_table = emb_table; a.emb_h = emb_h; a.emb_xn = emb_xn; a.emb_norm_w = emb_norm_w; a.emb_eps = emb_eps; a.emb_D = D;
    a.emb_rows = emb_rows; a.adv_pos = adv_pos; a.adv_step = adv_step; a.dbg_path = path;
    if (vec_loads) *vec_loads = sample_vec_loads(a);
    if (!adv_pos && !adv_step) return launch_sample(a, st);
    // the arrival ticket: zeroed here, and it must be back at zero once the launch is done (synchronises)
    unsigned int* ticket = nullptr;
    LG_CUDA_OK(cudaMallocAsync((void**)&ticket, sizeof(unsigned int), st));
    LG_CUDA_OK(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    a.adv_ticket = ticket;
    const int rc = launch_sample(a, st);
    unsigned int left = 0;
    const cudaError_t ce = cudaMemcpyAsync(&left, ticket, sizeof(left), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(ticket, st);
    LG_TRY(rc);
    LG_CUDA_OK(ce);
    LG_CUDA_OK(cudaStreamSynchronize(st));
    LG_REQUIRE(left == 0, "%s: the counter ticket was left at %u", fn, left);
    return 0;
}

int lg_test_sample_given(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                         const int32_t* step_rows, const int32_t* given, int32_t* out_idx, int32_t* out_seq, int seq_stride,
                         int32_t* next_tokens, void* stream) {
    static const char* fn = "lg_test_sample_given";
    LG_REQUIRE(logits && sc && seed_rows && step_rows && given && out_seq && seq_stride > 0, "%s: null argument or seq_stride=%d", fn,
               seq_stride);
    SampleArgs a = make_sample_args(*sc, logits, B, V, mix_cfg, round_dtype);
    a.seed_rows = seed_rows; a.step_rows = step_rows; a.given = given;
    a.out_idx = out_idx; a.out_seq = out_seq; a.seq_stride = seq_stride; a.next_tokens = next_tokens;
    return launch_sample(a, (cudaStream_t)stream);
}

int lg_test_sample_groups(const float* logits, int B, int K, int V, int round_dtype, const lg_sample_cfg* sc, const float* weights,
                          const uint64_t* seed_rows, const int32_t* step_rows, int32_t* out_idx, int32_t* next_tokens, void* stream) {
    static const char* fn = "lg_test_sample_groups";
    LG_REQUIRE(logits && sc && weights && out_idx, "%s: null logits, sc, weights or out_idx", fn);
    LG_REQUIRE(B > 0 && K >= 1 && K <= kMaxMixGroups && V > 0, "%s: bad shape B=%d K=%d V=%d", fn, B, K, V);
    LG_REQUIRE((seed_rows != nullptr) == (step_rows != nullptr), "%s: seed_rows and step_rows go together", fn);
    LG_REQUIRE(round_dtype == LG_DTYPE_F32 || lg_dtype_is16(round_dtype), "%s: unsupported round dtype %d", fn, round_dtype);
    SampleArgs a = make_sample_args(*sc, logits, B * K, V, 1, round_dtype);
    a.mix_groups = K; a.mix_weights = weights;
    a.seed_rows = seed_rows; a.step_rows = step_rows;
    a.out_idx = out_idx; a.next_tokens = next_tokens;
    return launch_sample(a, (cudaStream_t)stream);
}

int lg_test_score_head(const float* partial, int ks, int P, int V, int nh, float cfg_scale, int dtype, const int32_t* targets,
                       float* logits, float* nll, void* stream) {
    static const char* fn = "lg_test_score_head";
    LG_REQUIRE(partial && (logits || nll), "%s: null slabs, or neither logits nor nll", fn);
    LG_REQUIRE(!nll || targets, "%s: nll needs targets", fn);
    LG_REQUIRE(ks >= 1 && P > 0 && V > 0 && (nh == 1 || nh == 2), "%s: bad shape ks=%d P=%d V=%d nh=%d", fn, ks, P, V, nh);
    LG_REQUIRE(dtype == LG_DTYPE_F32 || lg_dtype_is16(dtype), "%s: unsupported dtype %d", fn, dtype);
    return launch_score_head(partial, ks, P, V, nh, cfg_scale, dtype, targets, logits, nll, (cudaStream_t)stream);
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
    const size_t needf = gemm_partial_floats(M, N, K, 0, dtype);
    LG_REQUIRE(scratch_bytes >= needf * sizeof(float), "lg_test_gemm: scratch %zu < %zu", scratch_bytes, needf * sizeof(float));
    GemmPlan plan;
    LG_TRY(gemm_partial(x, K, w, nullptr, 0, M, N, K, dtype, (float*)dev_scratch, &plan, st));
    return launch_reduce_f32((const float*)dev_scratch, plan.ksplit, M, N, y, st);
}

// What lg_test_linear and lg_test_linear_plan (fn) check of the shape-only arguments, then the call's path {kernel (3: gemv_small),
// tile, ksplit, row blocks or PF}
static int test_linear_args(const char* fn, int dtype, int M, int N, int K, bool paired, bool small, int epi, bool norm_out, bool w8,
                            int* path) {
    LG_REQUIRE((epi >= 0 && epi <= 4) || epi == 6, "%s: epilogue %d outside 0..4 and 6", fn, epi);
    const bool gated = epi == 2 || epi == 6;
    LG_REQUIRE(paired == gated, "%s: wb goes with the SwiGLU epilogue (2) and the gated-GELU epilogue (6) alone, epilogue %d", fn, epi);
    LG_REQUIRE(!norm_out || (epi == 1 && !small), "%s: norm_out goes with the batched residual epilogue alone", fn);
    if (small) {
        LG_REQUIRE(epi <= 2, "%s: the small path has no store or gelu epilogue (%d)", fn, epi);
        const GemvSmallPlan p = gemv_small_plan(M, N, K, dtype, paired, w8);
        LG_REQUIRE(p.rows != 0, "%s: %s", fn, p.error);
        path[0] = 3; path[1] = p.rows; path[2] = 1; path[3] = p.pf;
        return 0;
    }
    const GemmPlan p = gemm_plan(M, paired ? 2 * N : N, K, paired ? N : 0, dtype, w8);
    LG_REQUIRE(p.kernel >= 0, "%s: %s", fn, p.error);
    LG_REQUIRE(epi != 1 || (N % 4 == 0 && N <= 4096), "%s: the residual epilogue needs N %% 4 == 0 and N <= 4096 (N=%d)", fn, N);
    LG_REQUIRE(!gated || N % 4 == 0, "%s: the SwiGLU and gated-GELU epilogues need N %% 4 == 0 (N=%d)", fn, N);
    path[0] = p.kernel; path[1] = p.tile; path[2] = p.ksplit; path[3] = p.row_blocks;
    return 0;
}

// lg_test_linear / lg_test_linear_w8 (fn) over weights in the model dtype / fp8 weights (w8: wa.scale and, with wb, wb.scale set)
static int test_linear_run(const char* fn, bool w8, int dtype, int M, int N, int K, const void* x, const void* norm_in, float eps,
                           const GemmWeight& wa, const GemmWeight& wb, int epi, const void* norm_out, void* h, void* out, float* out_f32,
                           float* acc_out, int small, void* dev_scratch, size_t scratch_bytes, int* path, cudaStream_t st) {
    auto a16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    int pl[4];
    LG_TRY(test_linear_args(fn, dtype, M, N, K, wb.p != nullptr, small != 0, epi, norm_out != nullptr, w8, pl));
    LG_REQUIRE(x && wa.p && a16(x) && a16(wa.p) && a16(wb.p) && a16(norm_in) && a16(norm_out) && a16(h) && a16(out) && a16(out_f32) && a16(acc_out),
               "%s: null or misaligned (16 bytes) operand", fn);
    LG_REQUIRE((out_f32 != nullptr) == (epi == 0) && (h != nullptr) == (epi == 1) && (out != nullptr) == (epi >= 2 || norm_out != nullptr),
               "%s: epilogue %d writes out_f32 (0), h (1), out (1 with norm_out, 2-4) and no other buffer", fn, epi);
    LG_REQUIRE(!small || !acc_out, "%s: the small path keeps its accumulator on chip (acc_out)", fn);
    if (w8) {
        LG_REQUIRE(wa.scale && (wb.p == nullptr) == (wb.scale == nullptr), "%s: every fp8 weight comes with its row scales", fn);
        LG_TRY(w8_check_scales("wa_scale", wa.scale, N, dtype));
        if (wb.p) LG_TRY(w8_check_scales("wb_scale", wb.scale, N, dtype));
    }
    const int NN = wb.p ? 2 * N : N;
    const size_t pbytes = small ? 0 : align_up(gemm_partial_floats(M, NN, K, wb.p ? N : 0, dtype, w8) * sizeof(float));
    const size_t need = pbytes + (!small && norm_in ? (size_t)M * K * lg_dtype_info(dtype).esz : 0);
    LG_REQUIRE(need == 0 || (dev_scratch && ((uintptr_t)dev_scratch & 255) == 0 && scratch_bytes >= need),
               "%s: scratch %zu < %zu (256-byte aligned)", fn, scratch_bytes, need);
    if (path) std::copy(pl, pl + 4, path);
    if (small) {
        GemvSmall g{wa, wb, N, K, M, x, norm_in, eps, epi == 0 ? out_f32 : nullptr, epi == 1 ? h : nullptr, epi == 2 ? out : nullptr, dtype};
        return launch_gemv_small(g, st);
    }
    float* partial = (float*)dev_scratch;
    const void* xin = x;
    if (norm_in) {   // layer 0's attention norm (run_layers)
        xin = (char*)dev_scratch + pbytes;
        LG_TRY(launch_rmsnorm(x, norm_in, (void*)xin, M, K, eps, dtype, st));
    }
    GemmPlan p;
    LG_TRY(gemm_partial(xin, K, wa, wb, wb.p ? N : 0, M, NN, K, dtype, partial, &p, st));
    if (acc_out) LG_TRY(launch_reduce_f32(partial, p.ksplit, M, NN, acc_out, st));
    switch (epi) {
        case 0: return launch_reduce_f32(partial, p.ksplit, M, N, out_f32, st);
        case 1: return launch_residual_norm(partial, p.ksplit, M, N, h, norm_out, norm_out ? out : nullptr, eps, dtype, st);
        case 2: return launch_silu_mul(partial, p.ksplit, M, N, out, dtype, st);
        case 6: return launch_gelu_mul(partial, p.ksplit, M, N, out, dtype, st);
        default: return launch_store_act(partial, p.ksplit, M, N, out, epi == 4, dtype, st);
    }
}

int lg_test_linear(int dtype, int M, int N, int K, const void* x, const void* norm_in, float eps, const void* wa, const void* wb, int epi,
                   const void* norm_out, void* h, void* out, float* out_f32, float* acc_out, int small, void* dev_scratch,
                   size_t scratch_bytes, int* path, void* stream) {
    return test_linear_run("lg_test_linear", false, dtype, M, N, K, x, norm_in, eps, GemmWeight(wa), GemmWeight(wb), epi, norm_out, h, out,
                           out_f32, acc_out, small, dev_scratch, scratch_bytes, path, (cudaStream_t)stream);
}

int lg_test_linear_w8(int dtype, int M, int N, int K, const void* x, const void* norm_in, float eps, const uint8_t* wa, const float* wa_scale,
                      const uint8_t* wb, const float* wb_scale, int epi, const void* norm_out, void* h, void* out, float* out_f32,
                      float* acc_out, int small, void* dev_scratch, size_t scratch_bytes, int* path, void* stream) {
    return test_linear_run("lg_test_linear_w8", true, dtype, M, N, K, x, norm_in, eps, GemmWeight(wa, wa_scale), GemmWeight(wb, wb_scale), epi,
                           norm_out, h, out, out_f32, acc_out, small, dev_scratch, scratch_bytes, path, (cudaStream_t)stream);
}

int lg_test_linear_plan(int dtype, int M, int N, int K, int paired, int small, int epi, int has_norm_in, int* plan) {
    (void)has_norm_in;   // no dispatch rule depends on the RMSNorm prologue
    LG_REQUIRE(plan, "lg_test_linear_plan: null plan");
    return test_linear_args("lg_test_linear_plan", dtype, M, N, K, paired != 0, small != 0, epi, false, false, plan);
}

int lg_test_linear_w8_plan(int dtype, int M, int N, int K, int paired, int small, int epi, int has_norm_in, int* plan) {
    (void)has_norm_in;
    LG_REQUIRE(plan, "lg_test_linear_w8_plan: null plan");
    return test_linear_args("lg_test_linear_w8_plan", dtype, M, N, K, paired != 0, small != 0, epi, false, true, plan);
}

int lg_quantize_rows_e4m3(const void* w, int N, int K, int dtype, uint8_t* codes_out, float* scales_out, void* stream) {
    return launch_quantize_rows_e4m3(w, N, K, dtype, codes_out, scales_out, (cudaStream_t)stream);
}
int lg_weight_fp8_stored_index(int k) { return k < 0 ? -1 : w8_stored_index(k); }

// What lg_test_attention and lg_test_attention_plan (fn) check of the shape-only arguments, then the call's AttnArgs (no QKV slabs
// attached yet) over a K / V buffer of n_layer layers, with `maps` as the engine builds them (without a buffer: only whether it would),
// held to the dispatch rules: more than 65535 query rows only on kernel 2, slabs fused into the attention (`fused`) only on kernel 1
static int test_attention_args(const char* fn, KvMaps& maps, AttnArgs& aa, int dtype, int kv_dtype, const float* kv_scales, int R, int Tq,
                               int H, int hd, int hdp, int max_seq, void* kcache, void* vcache, int n_layer, int layer, PosArg pos,
                               bool fused) {
    LG_REQUIRE(dtype == LG_DTYPE_F32 || lg_dtype_is16(dtype), "%s: unsupported model dtype %d", fn, dtype);
    LG_REQUIRE(kv_dtype == dtype || (kv_dtype == LG_DTYPE_E4M3 && lg_dtype_is16(dtype)),
               "%s: KV dtype %d with model dtype %d (the model dtype, or LG_DTYPE_E4M3 for a bf16 / fp16 model)", fn, kv_dtype, dtype);
    LG_REQUIRE(R > 0 && Tq > 0 && H > 0 && max_seq > 0 && n_layer > 0 && layer >= 0 && layer < n_layer,
               "%s: bad shape R=%d Tq=%d H=%d max_seq=%d layer %d of %d", fn, R, Tq, H, max_seq, layer, n_layer);
    LG_REQUIRE(hd == 64 || hd == 100 || hd == 128, "%s: unsupported head_dim %d (64, 100, 128)", fn, hd);
    LG_REQUIRE(hdp == attn_kv_row_width(dtype, hd), "%s: row width %d for head_dim %d", fn, hdp, hd);
    if (pos.rows) {
        LG_REQUIRE(pos.dev == nullptr && pos.value == 0, "%s: per-row positions take no counter and no value", fn);
    } else {
        LG_REQUIRE(pos.value >= 0 && (pos.dev || pos.value + Tq <= max_seq), "%s: position %d + Tq %d exceeds max_seq %d", fn,
                   pos.value, Tq, max_seq);
    }
    const long long rows = (long long)n_layer * R * H * max_seq;
    if (kcache) LG_TRY(make_kv_maps(maps, dtype, hd, hdp, kv_dtype, kcache, vcache, rows));
    else maps.usable = attn_tma_maps_usable(dtype, hd, hdp, rows);
    aa = make_attn_args(dtype, H, hd, hdp, R, max_seq, (char*)kcache, (char*)vcache, maps, kv_dtype == LG_DTYPE_E4M3 ? kv_scales : nullptr,
                        layer, R, Tq);
    aa.pos = pos;
    const AttnPlan p = attn_plan(aa);
    LG_REQUIRE((long long)R * Tq <= 65535 || p.kernel == 2,
               "%s: bad shape R=%d Tq=%d: more than 65535 query rows need the causal tensor-core kernel", fn, R, Tq);
    LG_REQUIRE(!fused || p.kernel == 1, "%s: the fused QKV epilogue needs the TMA decode kernel", fn);
    return 0;
}

}  // extern "C"

// lg_test_attention (fn) with emb_mask_uncond, the mask rows r >= B read (null: emb_mask's)
static int test_attention_impl(const char* fn, int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp,
                               int max_seq, void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                               const int32_t* pos_rows, const float* emb_mask, const float* emb_mask_uncond, int B, int Tc, const void* q,
                               const float* qkv_partial, int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path,
                               void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    auto a16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    LG_REQUIRE(kv_dtype == LG_DTYPE_E4M3 ? kv_scale_ok(k_scale) && kv_scale_ok(v_scale) : k_scale == 1.f && v_scale == 1.f,
               "%s: K / V scales %g / %g (fp8: powers of two in [2^-8, 2^7], otherwise 1)", fn, (double)k_scale, (double)v_scale);
    LG_REQUIRE(kcache && vcache && out && a16(kcache) && a16(vcache) && a16(out) && a16(q) && a16(q_out) && a16(qkv_partial) && a16(freqs),
               "%s: null or misaligned (16 bytes) buffer", fn);
    LG_REQUIRE(!emb_mask || (B > 0 && Tc > 0 && Tc <= max_seq), "%s: emb_mask needs B > 0 and 0 < Tc <= max_seq (B=%d Tc=%d)", fn,
               B, Tc);
    LG_REQUIRE((q != nullptr) != (qkv_partial != nullptr), "%s: pass exactly one of q and qkv_partial", fn);
    LG_REQUIRE(q ? fuse == 0 : (ksplit > 0 && freqs && (fuse == 1 || (fuse == 0 && q_out))),
               "%s: q takes fuse = 0; qkv_partial needs ksplit > 0, freqs and fuse = 1 or q_out", fn);
    KvMaps maps;
    AttnArgs aa;
    const float scales[2] = {k_scale, v_scale};
    LG_REQUIRE(!emb_mask_uncond || emb_mask, "%s: emb_mask_uncond needs emb_mask", fn);
    LG_TRY(test_attention_args(fn, maps, aa, dtype, kv_dtype, scales, R, Tq, H, hd, hdp, max_seq, kcache, vcache, n_layer,
                               layer, PosArg{pos_dev, pos_value, pos_rows}, qkv_partial && fuse));
    aa.q = q ? q : q_out; aa.out = out;
    aa.emb_mask = emb_mask; aa.B = emb_mask ? B : 1; aa.Tc = emb_mask ? Tc : 0; aa.emb_mask_uncond = emb_mask_uncond;
    if (qkv_partial) {
        if (fuse) {
            aa.qkv_partial = qkv_partial; aa.qkv_ksplit = ksplit; aa.freqs = freqs;
        } else {
            LG_TRY(launch_qkv_epilogue(make_qkv_epi_args(aa, qkv_partial, ksplit, freqs), st));
        }
    }
    return launch_attention(aa, st, path);
}

extern "C" {

int lg_test_attention(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                      void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                      const int32_t* pos_rows, const float* emb_mask, int B, int Tc, const void* q, const float* qkv_partial,
                      int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path, void* stream) {
    return test_attention_impl("lg_test_attention", dtype, kv_dtype, k_scale, v_scale, R, Tq, H, hd, hdp, max_seq, kcache, vcache, n_layer,
                               layer, pos_value, pos_dev, pos_rows, emb_mask, nullptr, B, Tc, q, qkv_partial, ksplit, freqs, fuse, q_out, out,
                               path, stream);
}

int lg_test_attention_neg(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                          void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                          const int32_t* pos_rows, const float* emb_mask, const float* emb_mask_uncond, int B, int Tc, const void* q,
                          const float* qkv_partial, int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path,
                          void* stream) {
    return test_attention_impl("lg_test_attention_neg", dtype, kv_dtype, k_scale, v_scale, R, Tq, H, hd, hdp, max_seq, kcache, vcache,
                               n_layer, layer, pos_value, pos_dev, pos_rows, emb_mask, emb_mask_uncond, B, Tc, q, qkv_partial, ksplit, freqs,
                               fuse, q_out, out, path, stream);
}

int lg_test_attention_plan(int dtype, int kv_dtype, int R, int Tq, int H, int hd, int hdp, int max_seq, int n_layer, int pos_kind,
                           int pos_value, int input, int* plan) {
    // stand-ins for the call's device buffers: the checks and attn_plan only test them for null
    static const int32_t pos_buf = 0;
    static const float slab_buf = 0.f;
    LG_REQUIRE(pos_kind >= 0 && pos_kind <= 2 && input >= 0 && input <= 2 && plan,
               "lg_test_attention_plan: pos_kind %d or input %d outside 0..2, or null plan", pos_kind, input);
    KvMaps maps;
    AttnArgs aa;
    const float scales[2] = {1.f, 1.f};
    LG_TRY(test_attention_args("lg_test_attention_plan", maps, aa, dtype, kv_dtype, scales, R, Tq, H, hd, hdp, max_seq, nullptr, nullptr,
                               n_layer, 0, PosArg{pos_kind == 1 ? &pos_buf : nullptr, pos_value, pos_kind == 2 ? &pos_buf : nullptr},
                               input == 2));
    if (input == 2) aa.qkv_partial = &slab_buf;
    const AttnPlan p = attn_plan(aa);
    plan[0] = p.kernel; plan[1] = p.stages; plan[2] = p.fused;
    return 0;
}

}  // extern "C"

namespace {
// the 16-bit head's logits as the reference materialises them (gpt.py:368: `.float()` of a bf16 / fp16 tensor); past +-65504 an fp16
// logit becomes +-inf, like torch's fp16 head
template <typename T>
__global__ void round_logits_kernel(float* p, size_t n) {
    lg_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        p[i] = ElemTraits<T>::round(p[i]);
}
}  // namespace
static int round_logits_inplace(float* logits, size_t n, int dtype, cudaStream_t st) {
    if (!lg_dtype_is16(dtype)) return 0;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 132 * 8);
    (void)lg_launch(dtype == LG_DTYPE_F16 ? round_logits_kernel<f16> : round_logits_kernel<bf16>, dim3(blocks), dim3(256), 0, st, logits, n);
    LG_LAUNCH_CHECK();
    return 0;
}
