// Internal launch API shared by the translation units of libllamagen_b200.so.
#pragma once
#include "common.cuh"
#include <algorithm>

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
    // per-request guidance (lg_sample_rows_guided; needs mix_cfg): image b takes cfg_rows[b] / interval_rows[b] in place of
    // cfg_scale / cfg_interval, and mixes only when its scale is > 1 (generate.py's `if cfg_scale > 1.0`)
    const float* cfg_rows = nullptr;       // [B] or null
    const int32_t* interval_rows = nullptr;// [B] or null
    // parallel sampling (lg_sample_rows_keyed; needs seed_rows): image b keys its draw as image img_rows[b] of a call with seed
    // seed_rows[b], where null keys every row as image 0
    const int32_t* img_rows = nullptr;     // [B] or null
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
    // lg_test_sample only: [B][3] per image, written by thread 0 of its CTA: top-k select (0 none, 1 histogram, 2 radix fallback),
    // nucleus tie trim (0 / 1), draw ending (0 greedy, 1 claimed by a segment, 2 the past-the-end fallback). Null in production.
    int32_t* dbg_path = nullptr;
    // token log-probabilities (lg_sample_rows_logprobs, lg_generate_logprobs), each null or indexed as out_seq: element
    // b * seq_stride + step (top_ids / top_lp: that element's row of top_n). Any of them non-null selects the logprob instantiation.
    float* lp_out = nullptr;               // logprob of the drawn token: (x_pick - m) - log(Z) on the processed row x
    int32_t* rank_out = nullptr;           // 1 + #{v : x_v > x_pick}
    int32_t* top_ids = nullptr;            // the top_n kept tokens by (x desc, id asc); -1 past the kept ones
    float* top_lp = nullptr;               // their logprobs; -inf past the kept ones
    int top_n = 0;                         // 0 .. kMaxTopLogprobs
    // inpainting (lg_generate_given): [B, seq_stride] or null; a value >= 0 at element b * seq_stride + step is image b's given token
    // there: it goes to out_idx, out_seq, next_tokens and the fused tail in place of the draw (-1: the draw)
    const int32_t* given = nullptr;
    // composable guidance (lg_generate_composed): mix_groups = K > 0 makes the B rows of each half B / K images of K rows, image j's
    // rows j K .. j K + K - 1; one CTA per image mixes x = u + w_1 (c_1 - u) + ... + w_K (c_K - u) (left to right, in fp32) from its
    // conditional rows and the unconditional row B + j K, with mix_weights [B / K][K]. Image j's draw keys as image j + row_offset / K;
    // out_idx, out_probs, out_seq, the logprobs, teacher, seed_rows, step_rows and img_rows are per image, given is read at row j K
    // ([B][seq_stride]), and the token goes to next_tokens and the fused tail's rows of all 2K rows. 0: one row per image, as above
    int mix_groups = 0;
    const float* mix_weights = nullptr;
    // composed draws inside a mixed batch (lg_sample_rows_composed; mix_groups = 0, needs mix_cfg and seed_rows): int32
    // [B][1 + kMaxMixGroups], one CTA per row, and mix_weights becomes per row, [B][kMaxMixGroups]. Entry 0 of row b is its role:
    // -2, a condition row: the CTA writes nothing; -1, a plain row: conditional row b, unconditional row B + b, cfg_rows / interval_rows
    // as in lg_sample_rows_guided; u >= 0, a lead row: unconditional row u, conditional rows in entries 1 .. K (then -1), always mixed
    // (interval_rows still drops the mix). Keys, given, logprobs and outputs are row b's. No fused tail, no dbg_logits
    const int32_t* mix_rows = nullptr;
    // per-image sampling filters (lg_sample_cfg's *_rows): each null (the scalar above) or one entry per image; CTA b reads entry
    // b / param_div and uses it in place of temperature, top_k, top_p and greedy, with the scalar semantics. param_div = L for the
    // B * L window rows of a speculative-decoding pass, so that every window row of image b reads entry b; 1 otherwise (the grouped
    // instantiation's CTA is the image without a gather table and the row with one)
    const float* temp_rows = nullptr;      // [images] or null
    const int32_t* topk_rows = nullptr;    // [images] or null
    const float* topp_rows = nullptr;      // [images] or null
    const int32_t* greedy_rows = nullptr;  // [images] or null
    int param_div = 1;
};
constexpr int kMaxTopLogprobs = 20;
constexpr int kMaxMixGroups = 8;
inline bool sample_wants_logprobs(const SampleArgs& a) { return a.lp_out || a.rank_out || a.top_ids || a.top_lp; }
// The sample kernel stages the row with 16-byte loads (and dbg_logits with 16-byte stores) iff this holds, else element by element
__host__ __device__ inline bool sample_vec_loads(const SampleArgs& a) {
    return (a.V & 3) == 0 && ((uintptr_t)a.logits & 15) == 0 && ((uintptr_t)a.dbg_logits & 15) == 0;
}
int launch_sample(const SampleArgs& a, cudaStream_t st);
// Logprob rows of given tokens (lg_generate_logprobs' prefix): element b * S + k, k < P, of every non-null array gets logprob 0, rank 0,
// top ids -1 and top logprobs -inf
int launch_given_logprobs(float* lp, int32_t* rank, int32_t* top_ids, float* top_lp, int top_n, int B, int S, int P, cudaStream_t st);
// One chunk of an inpainting window (lg_generate_given's extend pass): image b's rows feed tokens j0 .. j0 + n - 1, token j0 from
// tokens[b] when `from_tokens` (the token the previous sample fed forward), the others from given [B, S]; win [B, n] gets them and
// pos_rows [nh * B] the position T + j0 of the chunk's first row (CFG twins included)
int launch_given_window(const int32_t* tokens, const int32_t* given, int B, int nh, int S, int j0, int n, int from_tokens, int pos0,
                        int32_t* win, int32_t* pos_rows, cudaStream_t st);

// Speculative Jacobi decoding (lg_generate_sjd). Image b's window has L slots; slot i feeds token start[b] + i - 1 (win) and its
// output p (the sample kernel's out_probs) is the distribution of token start[b] + i. Rows of image b are b * L + i.
enum SjdState { kSjdIters = 0, kSjdDone, kSjdTicket, kSjdActive, kSjdFinished, kSjdLive, kSjdStateInts };
struct SjdArgs {
    int B, S, L, V, T, nh;       // nh: 2 with CFG twins (rows b and B + b), else 1
    int greedy;
    uint64_t seed;
    int row_offset;              // added to the image index in every uniform's key
    const float* p;              // [B * L][V] this pass's p rows
    float* q;                    // [B * L][V] q of the draft for token start + i (slot i), unless qflag says uniform
    int32_t* qflag;              // [B * L] 1: that q is uniform, 1 / V
    const int32_t* x;            // [B * L] the sample kernel's draw from p of slot i
    int32_t* win;                // [B * L] window input tokens
    int32_t* nfin;               // [B] tokens final so far
    int32_t* start;              // [B] first token index the window predicts
    int32_t* shift;              // [B] start after the pass minus start before it
    int32_t* pos_rows;           // [nh * B] T + start - 1 (the position of slot 0)
    uint64_t* seed_rows;         // [B * L] the sample kernel's per-row seeds (redraws)
    int32_t* step_rows;          // [B * L] token index of each slot
    int32_t* out;                // [B][S]
    int32_t* state;              // [kSjdStateInts], zero-initialised
    float* dbg;                  // [passes][B][L][V] copy of every pass's p rows, or null
    int done_token;              // written to state[kSjdDone] once every image has S tokens (unique per call)
    // Per-slot mode (serving, lg_sjd_pass_slots): every image b is a slot with its own seed and pass counter, keyed as image
    // img_slots[b] (0 when img_slots is null) of a call with that seed (seed and row_offset unused). A slot with nfin >= S is frozen:
    // verify and refresh write nothing of it.
    uint64_t* seed_slots = nullptr;   // [B] or null (per-call mode)
    int32_t* pass_slots = nullptr;    // [B] passes the slot has run since its start; verify advances it, refresh keys with it
    int32_t* img_slots = nullptr;     // [B] or null: the image index every slot keys as, written by its start (start_img)
    int start_img = 0;
    float* cfg_rows = nullptr;        // [B * L] per-row guidance of the window rows (a start writes its slot's L rows), or null
    int32_t* interval_rows = nullptr; // [B * L]
    float start_cfg = 1.f;            // a start's (first = 1, one slot) seed is `seed`; its guidance scale and cfg_interval
    int start_interval = -1;
    const int32_t* greedy_rows = nullptr;   // [B] or null (greedy): image (slot) b's greedy flag, for acceptance and the residual draw
};
int launch_sjd_verify(const SjdArgs& a, cudaStream_t st);
// slot >= 0: only image `slot` (a per-slot start, with first = 1)
int launch_sjd_refresh(const SjdArgs& a, int first, cudaStream_t st, int slot = -1);

// ------------------------------------------------------------------------------------------------
// gemm.cu — y_partial[ks][M][N] (f32) = x[M,K] * W[N,K]^T ; W may be two row segments (w1 | w3).
// ------------------------------------------------------------------------------------------------
// The kernel a GEMM call runs on; n_split: weight rows [0, n_split) come from Wa, the rest from Wb (0 or N: Wa alone).
//   2 gemm_tc_kernel (gemm_tc.cu): bf16 / fp16, N % 128 == 0 and a segment boundary on a 128-row tile, unless LG_GEMM_TC=0.
//     tile: the row pad of a row block (16 ... 256), row_blocks: blocks of min(M, 256) rows.
//   0 gemm_skinny_kernel: fp32 at any M, and 16-bit at M <= 8 that kernel 2 does not take. tile 8 rows.
//   1 gemm_mma_kernel: every other 16-bit call. tile: 32, 64 or 128 rows (bm).
// ksplit: fp32 slabs [ksplit][M][N] written (<= 16). kernel -1: the call is not valid, `error` says why. The only reader of
// LG_GEMM_TC.
// w8: the weight is fp8 (GemmWeight::scale set). Kernel 2 is the only batched kernel that reads e4m3 codes, so such a call needs a
// bf16 / fp16 model, N % 128 == 0, a segment boundary on a 128-row tile, K % 64 == 0 and LG_GEMM_TC other than 0; anything else is
// kernel -1 (there is no 16-bit copy to fall back to). Where both are valid, the fp8 plan equals the 16-bit plan of the shape.
struct GemmPlan { int kernel = -1; int tile = 0; int ksplit = 0; int row_blocks = 0; char error[96] = {}; };
GemmPlan gemm_plan(int M, int N, int K, int n_split, int dtype, bool w8 = false);
// One GEMM weight [N][K] as the engine holds it: rows in the model dtype (scale null), or fp8 e4m3 codes in the stored K order of
// include/llamagen_b200.h (LG_DTYPE_E4M3) with one fp32 power-of-two scale per row
struct GemmWeight {
    const void* p = nullptr;
    const float* scale = nullptr;
    GemmWeight() = default;
    GemmWeight(const void* w, const float* s = nullptr) : p(w), scale(s) {}
    size_t bytes(size_t N, size_t K, size_t esz) const { return N * K * (scale ? 1 : esz); }
};
// Weights the NEXT GEMM of the decode chain will stream: the current GEMM's CTAs ask the L2 to fetch them
// (cp.async.bulk.prefetch.L2) so the next kernel's TMA loads hit L2 instead of paying the HBM latency.
struct GemmNext {
    const void* p0 = nullptr; size_t b0 = 0;
    const void* p1 = nullptr; size_t b1 = 0;
};
// floats of fp32 slabs the call's plan writes (0 for an invalid call); partial must hold that many
size_t gemm_partial_floats(int M, int N, int K, int n_split, int dtype, bool w8 = false);
// runs the call on the kernel gemm_plan picks; *plan (optional) receives that plan. wb.p null: wa alone
// pdl false: launched without PDL (lg_launch_pdl), so it starts after the stream's previous kernel completed
int gemm_partial(const void* X, int ldx, const GemmWeight& wa, const GemmWeight& wb, int n_split, int M, int N, int K,
                 int dtype, float* partial, GemmPlan* plan, cudaStream_t st, const GemmNext* next = nullptr, bool pdl = true);

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
                 void* out, cudaStream_t st, bool pdl = true);
// continuous batching, c2i: row r at position 0 takes the class embedding (cond rows: label src[r], uncond rows: null_idx),
// at any other position the token embedding of src[r % B]
int launch_embed_rows(const void* cls_table, const void* tok_table, const int32_t* src, const int* pos_rows, int B, int R, int null_idx,
                      int D, int dtype, void* out, cudaStream_t st);
// t2i cond rows: out[(r*T+t),:] = r < B ? cond[r,t,:] : uncond[(r-B)*uncond_stride + t*C + :]   (generate.py:137). uncond_stride 0:
// every unconditional row is uncond_embedding [T, C]; T * C: uncond holds one negative condition [T, C] per image
int launch_build_caption_rows(const void* cond, const void* uncond, size_t uncond_stride, int B, int R, int T, int C, int dtype,
                              void* out, cudaStream_t st);
// xn = rmsnorm(x) * w   (gpt.py:143-148)
int launch_rmsnorm(const void* x, const void* w, void* xn, int M, int D, float eps, int dtype, cudaStream_t st, bool pdl = true);

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
// out[m, j] = T(gelu_tanh(T(p[m, j]))) * T(p[m, F + j])   (T5's gated-GELU feed-forward; the rounding points of launch_silu_mul)
int launch_gelu_mul(const float* partial, int ksplit, int M, int F, void* out, int dtype, cudaStream_t st);
// out = gelu_tanh(T(p))  (gpt.py:122-131)   /   out = T(p)
int launch_store_act(const float* partial, int ksplit, int M, int N, void* out, int gelu, int dtype, cudaStream_t st);
// logits f32 [R, V] = sum partial rows (only needed when ksplit > 1 or rows are strided)
int launch_reduce_f32(const float* partial, int ksplit, int M, int N, float* out, cudaStream_t st);
// gather last-position rows: out[r,:] = in[(r*T + T-1),:]
int launch_gather_last(const void* in, int R, int T, int D, int dtype, void* out, cudaStream_t st);
// KV fan-out of serving (lg_copy_slot_kv): in a cache laid out [layers][rows, H, max_seq, row_bytes] (K at kcache, V at vcache),
// positions [0, len) of row half * B + src (half < nh) are copied to row half * B + dst[d] for every destination d, in every layer, K
// and V. One launch for up to kKvCopyMaxDst destinations, 16-byte copies when every segment allows them.
constexpr int kKvCopyMaxDst = 64;
struct KvCopyArgs {
    char *kcache, *vcache;
    int layers, rows, H, max_seq, row_bytes;   // row_bytes: bytes per position of one head (hdp elements of the stored type)
    int B, nh, len, src, n_dst;
    int dst[kKvCopyMaxDst];
};
int launch_copy_slot_kv(const KvCopyArgs& a, cudaStream_t st);

// lg_score: h[r, t] = t < T ? cond_rows[r * T + t] : table[idx[r % B][t - T]] over R * seq rows (idx [B][seq - T])
int launch_embed_seq(const void* cond_rows, const void* table, const int32_t* idx, int B, int R, int T, int seq, int D, int dtype, void* out,
                     cudaStream_t st);
// out row (b * S + s) * nh + half = in row (b + half * B) * seq + T - 1 + s (the scored positions of B images, CFG twins adjacent)
int launch_gather_scored(const void* in, int B, int nh, int seq, int T, int S, int D, int dtype, void* out, cudaStream_t st);
// P scored positions from the head's split-K slabs [ksplit][P * nh][V]: logits (dtype-rounded, CFG-mixed when nh == 2) -> logits
// [P][V] (or null), nll[p] = logsumexp - logit[targets[p]] (or null; NaN for a target outside [0, V))
int launch_score_head(const float* partial, int ksplit, int P, int V, int nh, float cfg_scale, int dtype, const int32_t* targets,
                      float* logits, float* nll, cudaStream_t st);

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
    const float* emb_mask_uncond = nullptr;   // [B, Tc]: the mask rows r >= B read (a negative prompt's); null: emb_mask's
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
// The emb-mask row attention row r reads (AttnArgs or attn_tma.cu's AttnTmaArgs): row r % B of emb_mask for the conditional rows
// r < B, and of emb_mask_uncond, when it is set, for the rows r >= B; null without a mask
template <class A>
__device__ __forceinline__ const float* attn_mask_row(const A& a, int r) {
    if (!a.emb_mask) return nullptr;
    return (r >= a.B && a.emb_mask_uncond ? a.emb_mask_uncond : a.emb_mask) + (size_t)(r % a.B) * a.Tc;
}
// KV-cache row width in elements: head_dim 100 of a bf16 / fp16 model (GPT-3B) is stored in 112-wide rows, 16-byte multiples that
// the TMA attention kernels can stream (dims 100..111 stay zero); every other cache row is hd wide
inline int attn_kv_row_width(int dtype, int hd) { return hd == 100 && lg_dtype_is16(dtype) ? 112 : hd; }
// The kernel an attention call runs on (attn_tma.cu), in this order of preference; the TMA kernels (1-4) need a 16-bit model with
// tensor maps over its cache (attn_tma_maps_usable), R <= 65535 and LG_ATTN_TMA other than 0.
//   1 attn_tma_kernel: decode (Tq = 1). fused = 1 when the call brings the QKV GEMM's split-K slabs: the kernel is also their
//     epilogue. stages: its TMA ring, 8 for fused hd 64 with R * H <= 264 (LG_ATTN_DEEP), 3 for other fused hd 64 under
//     LG_ATTN_NST=3, 2 otherwise.
//   3 attn_prefill_tc_kernel: the t2i condition prefill, 1 < Tq <= 128 from position 0, hd 64, fp8 caches too (LG_ATTN_PREFILL_TC).
//     TMA-staged Q/K/V, mma.sync QK^T and PV, one CTA per (row, head); stages 1.
//   2 attn_causal_tc_kernel (attn_causal_tc_f8_kernel for an fp8 cache): teacher-forced sequences and prefix prefills, Tq > 128 from
//     position 0, on a cache in the model dtype or fp8: a CTA per (head, row, 64-query block), K / V blocks through a 2-stage TMA ring, mma.sync QK^T and PV with an online
//     softmax; no R * Tq limit.
//   4 attn_window_tc_kernel: speculative-decoding windows, 2 <= Tq <= 64 queries per row at pos.rows[r] + t, caches in the model
//     dtype only, through kernel 2's ring.
//   0 attention_kernel (xf_kernels.cu): CUDA cores, no fused slabs, R * Tq <= 65535, rows attn_kv_row_width wide; stages 0.
// kernel -1: no kernel takes the call, `error` says why. The only reader of LG_ATTN_TMA, LG_ATTN_PREFILL_TC, LG_ATTN_DEEP and
// LG_ATTN_NST.
struct AttnPlan { int kernel = -1; int stages = 0; int fused = 0; char error[96] = {}; };
AttnPlan attn_plan(const AttnArgs& a);
// runs `a` on the kernel attn_plan picks; path (optional, int[3]) receives the plan's {kernel, stages, fused}
int launch_attention(const AttnArgs& a, cudaStream_t st, int* path = nullptr);
int launch_attention_tma(const AttnArgs& a, const AttnPlan& p, cudaStream_t st);   // p.kernel 1-4
// KV-cache tensor maps for bf16 / fp16 caches (dtype: LG_DTYPE_BF16 or LG_DTYPE_F16) and fp8 caches of those models (map dtype
// LG_DTYPE_E4M3: 64- or 128-byte boxes)
int attn_tma_make_map(void* map_out /*CUtensorMap, 128 B*/, const void* cache_base, long long total_rows, int hdp, int dtype,
                      int tail16 = 0);
// whether KV-cache tensor maps are built for a workspace (and the TMA attention kernels can run): 16-bit model, hd 64 / 128 or
// hd 100 in 112-wide rows, fewer than 2^31 cache rows over all layers
bool attn_tma_maps_usable(int dtype, int hd, int hdp, long long total_rows);
// VQ convolutions: vq.cu runs them; conv_tc.cu holds the wgmma kernels and chooses the kernel of each call.
// GroupNorm(32) partial statistics are [B][splits][32 groups][sum, sum of squares] floats. gn_stats_kernel writes at most
// kGnStatsMaxSplits splits per image; the drain of conv_tcw_kernel writes one per 16x16-pixel tile (and upsample phase) of its input.
constexpr int kGnStatsMaxSplits = 64;
// partials capacity that serves every GroupNorm of B images whose convolutions read inputs of at most H x W pixels
inline size_t gn_partial_capacity(int B, int H, int W) {
    return (size_t)B * std::max(kGnStatsMaxSplits, cdiv(H, 16) * cdiv(W, 16) * 4) * 32 * 2;
}
// up: 0 = same resolution, 1 = nearest-2x upsample folded in, 2 = Downsample (pad right/bottom, stride 2)
inline int conv_out_extent(int n, int up) { return up == 1 ? 2 * n : (up == 2 ? n / 2 : n); }
// an upsample conv has pre-summed 2x2 phase weights (conv_tc_make_phase_weights), which the wgmma path needs, exactly when this holds
inline bool conv_has_phase_weights(int up, int cin) { return up == 1 && cin % 64 == 0; }
// One convolution: bf16 NHWC input, weights repacked to bf16 [cout][k*k][cin], exactly one output
struct ConvCall {
    const bf16* in = nullptr;        // [B][Hin][Win][cin]
    int B = 0, Hin = 0, Win = 0, cin = 0, cout = 0, k = 0;
    int up = 0;
    const bf16* w = nullptr;
    const bf16* w_phase = nullptr;   // [4 phases][cout][4 taps][cin] when conv_has_phase_weights(up, cin)
    const float* bias = nullptr;
    const bf16* residual = nullptr;  // bf16 NHWC like the output, may alias out_bf
    bf16* out_bf = nullptr;          // bf16 NHWC
    float* out_nchw = nullptr;       // fp32 NCHW
    uint8_t* out_u8 = nullptr;       // clamp(127.5 y + 128, 0, 255) as uint8 NHWC
    float* gn_partial = nullptr;     // non-null: the drain may write the output's GroupNorm partials here (gn_floats capacity)
    size_t gn_floats = 0;
};
// The kernel a call runs on: 0 = mma.sync gather (vq.cu), 1 = conv_tc_kernel, 2 = conv_tcw_kernel; gn_splits > 0: its drain writes
// that many splits of the output's GroupNorm partials into gn_partial. The only reader of LG_CONV_TC, LG_CONV_SWAP and LG_GN_FUSE.
struct ConvPlan { int kernel = 0; int gn_splits = 0; };
ConvPlan conv_plan(const ConvCall& c);
int launch_conv_tc(const ConvCall& c, const ConvPlan& p, cudaStream_t st);   // p.kernel 1 or 2
void conv_tc_set_cta_budget(int ctas);   // > 0: persistent conv CTAs (at most `ctas`), 0: one CTA per tile (default)
int conv_tc_make_phase_weights(const float* w_f32, bf16* out, int cout, int cin, cudaStream_t st);
// gemm_tc.cu — wgmma/TMA weight-streaming GEMM (bf16 or fp16 activations, 16-bit or fp8 weights, row blocks of <= 256)
int gemm_tc_ksplit(int M, int N, int K);
int gemm_tc_partial(const void* X, int ldx, const GemmWeight& wa, const GemmWeight& wb, int n_split, int M, int N, int K, int dtype,
                    const GemmPlan& p, float* partial, cudaStream_t st, const GemmNext* next = nullptr, bool pdl = true);   // p.kernel 2

// gemv_small.cu — decode GEMMs for R <= 8 rows: CTA-owned output columns (no split-K), RMSNorm in the prologue (normw != null),
// epilogue by destination: out_f32 [R][N] | h (in-place residual add) | ff (SwiGLU gate of the Wa/Wb row pair)
struct GemvSmall {
    GemmWeight Wa, Wb;                // [N][K]; Wb only for the paired (w1 | w3) form; both fp8 or both 16-bit
    int N, K, R;
    const void* in;                   // [R][K]
    const void* normw; float eps;     // RMSNorm weight [K] or null
    float* out_f32; void* h; void* ff;
    int dtype;                        // LG_DTYPE_BF16 or LG_DTYPE_F16: every 16-bit tensor above
    bool pdl = true;                  // false: launched without PDL, it starts after the stream's previous kernel completed
};
// The instantiation a call runs on: rows = weight rows per CTA (8, 16 or 32; the paired form is 32: 16 rows of Wa and of Wb), pf =
// 32-wide k chunks in flight per warp. rows 0: the call is not supported (bf16 / fp16, 1 <= R <= 8, K % 32 == 0, K >= 256,
// R * (2K + 16) bytes <= 90 KiB, N > 0 a multiple of 32, or of 16 when paired), `error` says why. w8 (fp8 weights): a lane's 16-byte
// weight load spans a 64-wide k chunk, so K % 64 == 0 as well; rows as for 16-bit weights, pf counts 64-wide chunks.
struct GemvSmallPlan { int rows = 0; int pf = 0; char error[96] = {}; };
GemvSmallPlan gemv_small_plan(int R, int N, int K, int dtype, bool paired, bool w8 = false);
inline bool gemv_small_supported(int R, int N, int K, int dtype, bool paired, bool w8 = false) {
    return gemv_small_plan(R, N, K, dtype, paired, w8).rows != 0;
}
int launch_gemv_small(const GemvSmall& g, cudaStream_t st);

// weight_fp8.cu — fp8 (e4m3) GEMM weights: W [N][K] in bf16 / fp16 -> codes [N][K] in the stored K order + power-of-two row scales [N]
int launch_quantize_rows_e4m3(const void* w, int N, int K, int dtype, uint8_t* codes, float* scales, cudaStream_t st);
int w8_stored_index(int k);                                     // byte of a row that holds column k's code
void w8_scale_exponents(int dtype, int* emin, int* emax);      // allowed scale exponents of a bf16 / fp16 model
// copies N device scales to the host (synchronises) and fails unless each is 2^e with e in that range
int w8_check_scales(const char* name, const float* dev_scales, int N, int dtype);

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
