// Internal launch API shared by the translation units of libllamagen_b200.so.
#pragma once
#include "common.cuh"

// ------------------------------------------------------------------------------------------------
// sampling.cu
// ------------------------------------------------------------------------------------------------
struct SampleArgs {
    const float* logits;   // [rows, V], cond rows first
    int B, V;
    int mix_cfg;           // rows == 2B and CFG mixing requested
    int round_dtype;       // LG_DTYPE_BF16 / LG_DTYPE_F16: round raw logits to that type before use (16-bit head output,
                           // gpt.py:368); LG_DTYPE_F32 (0): use them as they are
    float cfg_scale;
    int cfg_interval;
    float temperature;
    int top_k;
    float top_p;
    int greedy;
    uint64_t seed;
    uint64_t step;         // index of the token being produced (0 = prefill sample)
    const int* step_dev;   // when non-null the step is read from device memory (graph replay)
    int row_offset;        // added to the image index in the RNG stream (multi-rank decorrelation)
    int32_t* out_idx;      // [B] or null
    float* out_probs;      // [B, V] or null
    int32_t* out_seq;      // [B, seq_stride] or null: out_seq[b, step] = idx
    int seq_stride;
    int32_t* next_tokens;  // [B] or null: token fed to the next decode step
    const int32_t* teacher;// [B, seq_stride] or null: teacher-forced next token
    float* dbg_logits;     // [S, dbg_batch, V] or null: mixed logits before temperature (row = row_offset + b)
    int dbg_batch;         // total images in the dbg buffer (0 -> B)
    // continuous batching (lg_sample_rows): every image is its own request with its own RNG seed and token index
    const uint64_t* seed_rows = nullptr;   // [B] or null
    const int* step_rows = nullptr;        // [B] or null
    // fused tail of a decode iteration (16-bit models; rows in round_dtype): the CTA that picked image b's token also writes the next step's input rows b and
    // B + b (token embedding, gpt.py:352; optionally its RMSNorm for layer 0, gpt.py:143-148) and the last CTA to finish advances the
    // device-resident position / step counters - three dependent kernels (embed, rmsnorm, advance) fewer per token
    const void* emb_table = nullptr;       // tok_embeddings [V][D] (null: no fused tail)
    void* emb_h = nullptr;                 // [R][D] next step's residual stream
    void* emb_xn = nullptr;                // [R][D] RMSNorm(h) * norm_w, or null
    const void* emb_norm_w = nullptr;      // [D]
    float emb_eps = 0.f;
    int emb_D = 0;
    int emb_rows = 0;                      // R (2B with CFG twins, else B)
    int* adv_pos = nullptr;                // incremented once per launch by the last CTA (null: no advance)
    int* adv_step = nullptr;
    unsigned int* adv_ticket = nullptr;    // zero-initialised arrival counter, left at zero
};
int launch_sample(const SampleArgs& a, cudaStream_t st);

// ------------------------------------------------------------------------------------------------
// gemm.cu — y_partial[ks][M][N] (f32) = x[M,K] * W[N,K]^T ; W may be two row segments (w1 | w3).
// ------------------------------------------------------------------------------------------------
struct GemmPlan {
    int ksplit;            // number of fp32 partial slabs written
};
// Weights the NEXT GEMM of the decode chain will stream: the current GEMM's CTAs ask the L2 to fetch them
// (cp.async.bulk.prefetch.L2) so the next kernel's TMA loads hit L2 instead of paying the HBM latency.
struct GemmNext {
    const void* p0 = nullptr; size_t b0 = 0;
    const void* p1 = nullptr; size_t b1 = 0;
};
// Returns the plan used; partial must hold ksplit_max(M,N,K) * M * N floats (see gemm_partial_floats).
size_t gemm_partial_floats(int M, int N, int K, int dtype);
int gemm_partial(const void* X, int ldx, const void* Wa, const void* Wb, int n_split, int M, int N, int K,
                 int dtype, float* partial, GemmPlan* plan, cudaStream_t st, const GemmNext* next = nullptr);

// ------------------------------------------------------------------------------------------------
// xf_kernels.cu — transformer glue kernels (all templated on the activation dtype internally)
// ------------------------------------------------------------------------------------------------
struct PosArg {            // position of row-block: pos = (rows ? rows[r] : (dev ? *dev : 0) + value) + t
    const int* dev;
    int value;
    const int* rows = nullptr;   // per-row positions [R] (continuous batching: sequences at different depths share one step)
};

// out[r,:] = table[idx(r),:]; idx(r) = r < B ? src[r] : (null_idx >= 0 ? null_idx : src[r-B])
int launch_embed(const void* table, const int32_t* src, int B, int R, int null_idx, int D, int dtype,
                 void* out, cudaStream_t st);
// continuous batching, c2i: row r at position 0 takes the class embedding (cond rows: label src[r], uncond rows: null_idx),
// at any other position the token embedding of src[r % B]
int launch_embed_rows(const void* cls_table, const void* tok_table, const int32_t* src, const int* pos_rows, int B, int R, int null_idx,
                      int D, int dtype, void* out, cudaStream_t st);
// t2i cond rows: out[(r*T+t),:] = r < B ? cond[r,t,:] : uncond[t,:]   (generate.py:137)
int launch_build_caption_rows(const void* cond, const void* uncond, int B, int R, int T, int C, int dtype,
                              void* out, cudaStream_t st);
// xn = rmsnorm(x) * w   (gpt.py:143-148)
int launch_rmsnorm(const void* x, const void* w, void* xn, int M, int D, float eps, int dtype, cudaStream_t st);

struct QkvEpiArgs {
    const float* partial; int ksplit;   // [ks][M][3D]
    int M, Tq, D, H, hd;
    PosArg pos;
    const float* freqs;                 // [P, hd/2, 2]
    void* q;                            // [M, D]
    void* kcache; void* vcache;         // [R, H, maxS, hd] for this layer
    int maxS;
    int dtype;
    int hdp = 0;                        // elements between consecutive cache rows (0: hd). GPT-3B's hd = 100 is stored in 112-wide rows
    // fp8 KV cache (lg_engine_set_kv_cache): K / V are stored as e4m3(x * inv) with inv = 1 / (this layer's power-of-two scale)
    int kv_f8 = 0;
    float k_inv = 1.f, v_inv = 1.f;
};
int launch_qkv_epilogue(const QkvEpiArgs& a, cudaStream_t st);

// h += T(sum partial); optionally xn = rmsnorm(h) * norm_w  (fused residual + next norm)
int launch_residual_norm(const float* partial, int ksplit, int M, int D, void* h, const void* norm_w, void* xn,
                         float eps, int dtype, cudaStream_t st);
// out[m, j] = silu(T(p[m, j])) * T(p[m, F + j])   (gpt.py:167)
int launch_silu_mul(const float* partial, int ksplit, int M, int F, void* out, int dtype, cudaStream_t st);
// out = gelu_tanh(T(p))  (gpt.py:122-131)   /   out = T(p)
int launch_store_act(const float* partial, int ksplit, int M, int N, void* out, int gelu, int dtype, cudaStream_t st);
// logits f32 [R, V] = sum partial rows (only needed when ksplit > 1 or rows are strided)
int launch_reduce_f32(const float* partial, int ksplit, int M, int N, float* out, cudaStream_t st);
// gather last-position rows: out[r,:] = in[(r*T + T-1),:]
int launch_gather_last(const void* in, int R, int T, int D, int dtype, void* out, cudaStream_t st);

struct AttnArgs {
    const void* q;          // [M, D] post-RoPE
    const void* kcache; const void* vcache;   // [R, H, maxS, hd]
    void* out;              // [M, D]
    int R, Tq, H, hd, maxS;
    PosArg pos;             // query t attends keys [0, pos+t]
    const float* emb_mask;  // [B, Tc] or null  (generate.py:154-163)
    int B, Tc;
    float scale;
    int dtype;
    int hdp = 0;            // elements between consecutive cache rows (0: hd); q / out stay [M, H*hd]
    // TMA path (attn_tma.cu): tensor maps over the whole K / V cache regions + this layer's first row
    const void* kmap = nullptr; const void* vmap = nullptr;        // kKC-row boxes
    const void* kmap16 = nullptr; const void* vmap16 = nullptr;    // 16-row boxes for the tail chunk
    long long cache_row_base = 0;
    // fused QKV epilogue (TMA path, Tq == 1): the attention kernel reduces the QKV GEMM's split-K slabs itself
    const float* qkv_partial = nullptr; int qkv_ksplit = 0; const float* freqs = nullptr;
    // fp8 KV cache: the caches hold e4m3 codes; `scale` already includes the K scale, the output is multiplied by v_scale, and the
    // fused writer stores e4m3(k * k_inv), e4m3(v * v_inv)
    int kv_f8 = 0;
    float k_inv = 1.f, v_inv = 1.f, v_scale = 1.f;
};
// KV-cache row width in elements: head_dim 100 of a bf16 / fp16 model (GPT-3B) is stored in 112-wide rows, 16-byte multiples that
// the TMA attention kernels can stream (dims 100..111 stay zero); every other cache row is hd wide
inline int attn_kv_row_width(int dtype, int hd) { return hd == 100 && lg_dtype_is16(dtype) ? 112 : hd; }
// path (optional, int[3]): the kernel that was launched (0 = attention_kernel, 1 = attn_tma_kernel,
// 3 = attn_prefill_tc_kernel), its TMA ring depth (0 for attention_kernel, 1 for the single-stage prefill) and whether it fused the
// QKV epilogue
int launch_attention(const AttnArgs& a, cudaStream_t st, int* path = nullptr);
inline void set_attn_path(int* path, int kernel, int stages, int fused) {
    if (path) { path[0] = kernel; path[1] = stages; path[2] = fused; }
}
// attn_tma.cu — TMA + tensor-core decode attention for bf16 / fp16 caches (dtype: LG_DTYPE_BF16 or LG_DTYPE_F16) and fp8 caches of
// those models (map dtype LG_DTYPE_E4M3: 64- or 128-byte boxes)
int attn_tma_make_map(void* map_out /*CUtensorMap, 128 B*/, const void* cache_base, long long total_rows, int hdp, int dtype,
                      int tail16 = 0);
// whether KV-cache tensor maps are built for a workspace (and the TMA attention kernels can run): 16-bit model, hd 64 / 128 or
// hd 100 in 112-wide rows, fewer than 2^31 cache rows over all layers
bool attn_tma_maps_usable(int dtype, int hd, int hdp, long long total_rows);
bool attn_tma_supported(const AttnArgs& a);
bool attn_tma_enabled();
int launch_attention_tma(const AttnArgs& a, cudaStream_t st, int* path = nullptr);
// t2i condition prefill (1 < Tq <= 128, hd 64, bf16 / fp16): TMA-staged Q/K/V, mma.sync QK^T and PV, one CTA per (row, head)
bool attn_prefill_tc_supported(const AttnArgs& a);
int launch_attention_prefill_tc(const AttnArgs& a, cudaStream_t st, int* path = nullptr);
// conv_tc.cu — wgmma implicit-GEMM convolution over bf16 NHWC activations (TMA 4-D boxes, register accumulators)
bool conv_tc_supported(int Hin, int Win, int Cin, int Cout, int ksize, int up, bool nchw_out);
void conv_tc_set_cta_budget(int ctas);   // > 0: persistent conv CTAs (at most `ctas`), 0: one CTA per tile (default)
int conv_tc_make_phase_weights(const float* w_f32, bf16* out, int cout, int cin, cudaStream_t st);
int launch_conv_tc(const bf16* in, int B, int Hin, int Win, int Cin, const bf16* weights, const float* bias, int Cout,
                   int ksize, int up, const bf16* residual, bf16* out_bf, float* out_nchw, cudaStream_t st, uint8_t* out_u8 = nullptr,
                   float* gn_partial = nullptr, size_t gn_floats = 0, int* gn_splits = nullptr,    // *gn_splits > 0: the drain also wrote the
                   int* path = nullptr);   // output's GroupNorm(32) partial statistics [B][*gn_splits][32][2] into gn_partial;
                                           // *path: 1 = conv_tc_kernel, 2 = conv_tcw_kernel was launched
// gemm_tc.cu — wgmma/TMA weight-streaming GEMM (bf16 or fp16, row blocks of <= 256)
int gemm_tc_ksplit(int M, int N, int K);
bool gemm_tc_supported(int M, int N, int K, int dtype);
int gemm_tc_partial(const void* X, int ldx, const void* Wa, const void* Wb, int n_split, int M, int N, int K, int dtype,
                    float* partial, int* ksplit_out, cudaStream_t st, const GemmNext* next = nullptr);

// gemv_small.cu — decode GEMMs for R <= 8 rows: CTA-owned output columns (no split-K), RMSNorm in the prologue (normw != null),
// epilogue by destination: out_f32 [R][N] | h (in-place residual add) | ff (SwiGLU gate of the Wa/Wb row pair)
struct GemvSmall {
    const void* Wa; const void* Wb;   // [N][K]; Wb only for the paired (w1 | w3) form
    int N, K, R;
    const void* in;                   // [R][K]
    const void* normw; float eps;     // RMSNorm weight [K] or null
    float* out_f32; void* h; void* ff;
    int dtype;                        // LG_DTYPE_BF16 or LG_DTYPE_F16: every 16-bit tensor above
};
bool gemv_small_supported(int R, int N, int K, int dtype, bool paired);
int launch_gemv_small(const GemvSmall& g, cudaStream_t st);

// *pos += 1; *step += 1  (device-side loop counters for graph replay)
int launch_advance(int* pos, int* step, cudaStream_t st);
int launch_set_counters(int* pos, int pos_v, int* step, int step_v, cudaStream_t st);

// ------------------------------------------------------------------------------------------------
// per-kernel-class device timing (bench.py's roofline leg): when enabled every launch site wrapped in
// LG_PROF is bracketed by cudaEvents on the launching stream; graphs are bypassed while it is on.
// ------------------------------------------------------------------------------------------------
enum ProfClass {
    PC_GEMM_QKV = 0, PC_QKV_EPI, PC_ATTENTION, PC_GEMM_WO, PC_RESNORM, PC_GEMM_W13, PC_SILU, PC_GEMM_W2,
    PC_GEMM_HEAD, PC_SAMPLE, PC_EMBED_MISC, PC_VQ_CONV, PC_VQ_GN_STATS, PC_VQ_GN_APPLY, PC_VQ_ATTN, PC_VQ_MISC,
    PC_COUNT
};
bool prof_enabled();
void prof_begin(int cls, cudaStream_t st);
void prof_end(cudaStream_t st);
#define LG_PROF(cls, st, expr)                                                                   \
    do {                                                                                         \
        prof_begin((cls), (st));                                                                 \
        int _pr = (expr);                                                                        \
        prof_end((st));                                                                          \
        if (_pr < 0) return _pr;                                                                 \
    } while (0)
