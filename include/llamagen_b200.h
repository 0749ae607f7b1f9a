/*
 * llamagen_b200 — C-ABI of the H100-native (sm_90a) autoregressive image-sampling engine.
 *
 * Drop-in boundary for ONE hot path of FoundationVision/LlamaGen (reference paths are
 * relative to the reference checkout):
 *   - autoregressive/models/generate.py:126-176   generate()  (prefill, KV-cached decode, CFG, sampling)
 *   - autoregressive/models/gpt.py:332-382        Transformer.forward (inference branches)
 *   - tokenizer/tokenizer_image/vq_model.py:52-55 VQModel.decode_code (lookup + conv/attn decoder)
 *   - tokenizer/tokenizer_image/vq_model.py:215-233 VectorQuantizer.forward (argmin-L2, encode side)
 *
 * The reference has no FFI layer (it is pure PyTorch); the Python shim in llamagen_b200/ mirrors its
 * Python API (GPT_models / VQ_models / generate / decode_code) and calls these entry points through
 * ctypes.  Conventions:
 *   - every pointer marked "dev" is a CUDA device pointer owned by the CALLER (PyTorch); the library
 *     never frees caller memory.  Engine-owned memory is only small repacked weights / tables.
 *   - every call returns 0 on success, <0 on error; lg_last_error() returns a thread-local message.
 *     Nothing throws or aborts.
 *   - all work is enqueued asynchronously on the given cudaStream_t (passed as void*); no hidden
 *     device synchronisation except where stated.
 *   - one engine per device per process; an engine is not re-entrant.
 */
#ifndef LLAMAGEN_B200_H
#define LLAMAGEN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LG_ABI_VERSION 1

/* LG_DTYPE_F16 (IEEE half) runs the same tensor-core kernels as LG_DTYPE_BF16; values past +-65504 become +-inf, as in torch. */
/* LG_DTYPE_E4M3 (fp8 e4m3, finite, max +-448) is a storage type of a bf16 / fp16 model, never a model dtype: of the KV cache
 * (lg_engine_set_kv_cache) and of the GEMM weights (lg_engine_bind_weight, "fp8 weights" below). */
enum { LG_DTYPE_F32 = 0, LG_DTYPE_BF16 = 1, LG_DTYPE_F16 = 2, LG_DTYPE_E4M3 = 3 };
enum { LG_MODEL_C2I = 0, LG_MODEL_T2I = 1 };

/* Mirrors autoregressive/models/gpt.py:23-50 (ModelArgs) — only the fields the inference path reads. */
typedef struct lg_model_cfg {
    int32_t n_layer;
    int32_t n_head;
    int32_t dim;
    int32_t ffn_dim;       /* FeedForward hidden size, gpt.py:154-159 */
    int32_t vocab_size;
    int32_t cls_token_num; /* 1 (c2i) or 120 (t2i) */
    int32_t block_size;    /* image tokens = grid*grid */
    int32_t num_classes;   /* c2i null class index == num_classes (generate.py:130) */
    int32_t caption_dim;   /* t2i feature width (2048) */
    int32_t model_type;    /* LG_MODEL_* */
    int32_t dtype;         /* LG_DTYPE_F32, _BF16 or _F16: weights, activations and KV cache */
    float   norm_eps;      /* RMSNorm eps, gpt.py:31 */
} lg_model_cfg;

/* Sampling parameters; mirrors generate()'s **sampling_kwargs + cfg args (generate.py:57,126). */
typedef struct lg_sample_cfg {
    float    cfg_scale;     /* >1 enables classifier-free guidance (rows doubled) */
    int32_t  cfg_interval;  /* generate.py:113: after decode iteration i > cfg_interval use cond logits only; -1 = never */
    float    temperature;
    int32_t  top_k;         /* 0 = off */
    float    top_p;         /* 1.0 = off */
    int32_t  greedy;        /* 1 == sample_logits=False (argmax) */
    uint64_t seed;          /* counter-based RNG seed for the multinomial draw */
    /* Per-image filters: device arrays, each NULL (every image takes the scalar above) or one entry per image of the call, entry b
     * replacing temperature, top_k, top_p or greedy for image b with the same semantics (temperature: divide by max(t, 1e-5); top_k:
     * k <= 0 off, clamped to V; top_p: p >= 1 off, p <= 0 keeps the maximum; greedy: nonzero is argmax). Image b is image b of the call
     * (c2i with CFG: conditional image b; a composed call: image b, not its K rows), or slot b for lg_sample_rows* and lg_sjd_pass_slots,
     * whose window rows of slot b all read entry b. The values are not checked on the device: the caller checks them. */
    const float*   temperature_rows;
    const int32_t* top_k_rows;
    const float*   top_p_rows;
    const int32_t* greedy_rows;
} lg_sample_cfg;

typedef struct lg_engine lg_engine;
typedef struct lg_vq lg_vq;

int         lg_version(void);
const char* lg_last_error(void);
/* Number of kernels this library has launched since load (or since lg_reset_launch_count). */
uint64_t    lg_launch_count(void);
void        lg_reset_launch_count(void);

/* ---- AR transformer engine: replaces Transformer.setup_caches/forward (gpt.py:316-382) ---------- */
int  lg_engine_create(const lg_model_cfg* cfg, int device, lg_engine** out);
void lg_engine_destroy(lg_engine* e);
/* Borrow a checkpoint tensor by its reference state_dict name (SURVEY §5), plus "freqs_cis"
 * (fp32 [cls_token_num+block_size, head_dim/2, 2], gpt.py:404-417).  dtype must equal cfg.dtype
 * except freqs_cis (always f32) and fp8 weights with their scales (below).  The caller keeps the tensor alive. */
int  lg_engine_bind_weight(lg_engine* e, const char* name, const void* dev_ptr,
                           const int64_t* shape, int ndim, int dtype);
/* fp8 weights (weight-only, "W8A16") of a bf16 / fp16 model. The six GEMM weights "layers.{i}.attention.wqkv.weight",
 * "...attention.wo.weight", "...feed_forward.w1.weight", "...w3.weight", "...w2.weight" and "output.weight" may each be bound with
 * dtype LG_DTYPE_E4M3 as dev uint8 codes [N, K], together with a companion tensor "<name>_scale", dev f32 [N] (LG_DTYPE_F32):
 *   - scale[n] = 2^e, one per output row; allowed e: [-15, 7] for an fp16 model (every code * scale is then an fp16 value, the
 *     smallest e4m3 subnormal being 2^-9), [-64, 64] for a bf16 model;
 *   - the layer computes y[r, n] = scale[n] * sum_k x[r, k] * code[n, k]: codes widened exactly to the model dtype, products and sum
 *     in fp32 on the tensor cores, the scale applied to the fp32 sum before its first rounding. Activations, KV cache, norms,
 *     embeddings and every rounding point are those of the 16-bit model, so the engine computes what it computes for the 16-bit
 *     weight code * scale (up to the order of the fp32 sum);
 *   - stored K order: the code of column k is byte lg_weight_fp8_stored_index(k) of its row. With k = 64 c + 16 s + 8 h + 2 q + b
 *     (s, q in 0..3; h, b in 0..1) that is 64 c + 16 q + 4 s + 2 h + b: a permutation inside every 64-wide k-block that makes the
 *     tensor-core A fragments of one thread contiguous. Hence K % 64 == 0, and the batched kernel needs N % 128 == 0.
 * Any subset of the six may be fp8, except that w1 and w3 of a layer (one GEMM) go together. lg_quantize_rows_e4m3 produces codes
 * and scales from a 16-bit weight. An fp8 weight has no 16-bit copy inside the engine: a call no fp8 kernel takes is an error. */
/* Validate that every tensor the configured model needs is bound. An fp8 weight is refused on an fp32 model, without its scales,
 * with a scale outside the allowed powers of two (the scales are copied to the host: synchronises), and with a shape the fp8 GEMM
 * kernel does not take (N % 128, K % 64). */
int  lg_engine_finalize(lg_engine* e);
/* w dev [N, K] in dtype (LG_DTYPE_BF16 or _F16, K % 64 == 0) -> codes_out dev uint8 [N, K] in the stored K order and scales_out dev
 * f32 [N]: scale[n] = 2^e with max_k |w[n, k]| / 2^e in (224, 448], e clamped to the allowed range above, 1 for an all-zero row;
 * code = e4m3_satfinite_rne(float(w[n, k]) / scale[n]) (cvt.rn.satfinite.e4m3x2.f32, the KV-cache writers' conversion). */
int  lg_quantize_rows_e4m3(const void* w, int N, int K, int dtype, uint8_t* codes_out, float* scales_out, void* stream);
/* Byte of a stored row that holds column k's code (k >= 0; no GPU needed). */
int  lg_weight_fp8_stored_index(int k);
/* Bytes of caller-provided scratch (KV cache + activations) for `rows` sequences (rows = 2*B under CFG)
 * of up to max_seq positions (cls_token_num + new tokens). Replaces setup_caches (gpt.py:316-330). */
int  lg_engine_workspace_bytes(lg_engine* e, int rows, int max_seq, size_t* bytes);
int  lg_engine_set_workspace(lg_engine* e, void* dev_ws, size_t bytes, int rows, int max_seq);
/* KV-cache storage of a bf16 / fp16 model. kv_dtype = LG_DTYPE_E4M3 stores K and V as fp8 e4m3 (one byte per element, half
 * the cache bytes): the stored byte is e4m3_satfinite_rne(x / s) of the model-dtype value x (K after RoPE), and every read,
 * including the current step's own key and value, sees e4m3 * s. scales: host float [n_layer][2] = (k, v) per layer, each a
 * power of two in [2^-8, 2^7], or NULL for all 1.0. kv_dtype = the model's dtype restores the default 16-bit cache.
 * Call after lg_engine_create / lg_engine_finalize and before lg_engine_workspace_bytes / lg_engine_set_workspace: the call
 * drops the workspace, so compute calls fail until lg_engine_set_workspace runs again. fp32 models are refused. */
int  lg_engine_set_kv_cache(lg_engine* e, int kv_dtype, const float* scales);

/* Prefill over the condition (generate.py:77-86 / gpt.py:348-349).
 *  c2i: cond = dev int32 [B] class labels.      t2i: cond = dev [B, T, caption_dim] features (cfg.dtype),
 *  emb_mask = dev f32 [B, T] or NULL.  With use_cfg the engine appends the null-condition rows itself
 *  (generate.py:129-137).  Writes last-position logits f32 [rows, V] to logits_out (dev), rows = B or 2B. */
int  lg_prefill(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int use_cfg,
                float* logits_out, void* stream);
/* One decode step at absolute position `pos` (generate.py:89-102 model call): tokens dev int32 [B];
 * under CFG both halves consume the same token (torch.cat([x, x])). logits_out f32 [rows, V]. */
int  lg_decode_step(lg_engine* e, const int32_t* tokens, int B, int pos, int use_cfg,
                    float* logits_out, void* stream);
/* Iteration-level scheduling for class-conditional serving (autoregressive/serve/llm_engine.py:511 `step()`, serve/llm.py:238-266):
 * ONE decode step for sequences at DIFFERENT depths. pos_rows dev int32 [R]: position of every row (R = 2B under CFG, cond rows
 * first); a row at position 0 has just joined and takes its class embedding (cond rows: tokens[b] is the label, uncond rows: the
 * null class), any other row the embedding of tokens[b]. Writes row r's K/V at pos_rows[r] and attends over [0, pos_rows[r]].
 * logits_out dev f32 [R, V]. */
int  lg_decode_rows(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, int B, int use_cfg, float* logits_out, void* stream);
/* Text-conditional serving. The lg_engine_set_workspace workspace holds B request slots: slot s owns cache row s and, with use_cfg,
 * row B + s. Bytes of caller-provided scratch for lg_prefill_slot (t2i models only). */
int  lg_slot_workspace_bytes(lg_engine* e, int use_cfg, size_t* bytes);
/* Start one request in slot `slot`: cond dev [T, caption_dim] in the model dtype (left-padded, padding zeroed, as
 * cond.prepare_condition makes it), T == cls_token_num; emb_mask dev f32 [T] or NULL. Writes the K / V of positions 0 .. T - 1 of
 * the slot's rows (the CFG row with the null condition, uncond_embedding, and the same emb_mask, as lg_generate does) and nothing
 * else of the workspace. logits_out dev f32 [nh, V] (nh = 2 with use_cfg, cond row first): the head output at position T - 1, rounded
 * as lg_prefill rounds it. The arithmetic depends on neither slot, B, nor the contents of any other row, including the rows' own
 * stale K / V from an earlier request: each row is prefilled alone (lg_generate_prefix's prefill chunk of one row, P = 0), then one
 * head GEMM runs over the request's nh rows. dev_ws: 256-byte aligned, at least lg_slot_workspace_bytes. Every argument is checked
 * before any launch; the workspace needs rows >= nh * B and max_seq >= T. */
int  lg_prefill_slot(lg_engine* e, const void* cond, const float* emb_mask, int T, int slot, int B, int use_cfg, void* dev_ws,
                     size_t ws_bytes, float* logits_out, void* stream);
/* Bytes of caller-provided scratch for lg_prefill_slot_prefix with a prefix of P tokens, P in [0, block_size - 1] (c2i and t2i models).
 * P = 0 gives lg_slot_workspace_bytes' size. */
int  lg_slot_prefix_workspace_bytes(lg_engine* e, int use_cfg, int P, size_t* bytes);
/* Start one image-completion request in slot `slot` (c2i and t2i models): lg_prefill_slot with the request's first P image tokens.
 * cond: c2i dev int32 [1] (the class id), t2i as for lg_prefill_slot; emb_mask: t2i only (dev f32 [T] or NULL), NULL for c2i.
 * prefix dev int32 [P], ids in [0, vocab_size), P in [0, block_size - 1] (NULL allowed only with P = 0). Writes the K / V of
 * positions 0 .. T + P - 1 of row `slot` and, with use_cfg, of row B + slot (the null condition there), and nothing else of the
 * workspace. logits_out dev f32 [nh, V]: the head output at position T + P - 1 (the logits of token P), rounded as lg_prefill_slot
 * rounds them. Each row is one prefill chunk of T + P positions (lg_generate_prefix's chunk of one row), then one head GEMM over the
 * nh rows: the arithmetic depends on neither slot, B nor any other row. dev_ws: 256-byte aligned, at least
 * lg_slot_prefix_workspace_bytes. Every argument is checked before any launch; the workspace needs rows >= nh * B and
 * max_seq >= T + P. lg_prefill_slot is the P = 0 case of this function (t2i only). */
int  lg_prefill_slot_prefix(lg_engine* e, const void* cond, const float* emb_mask, int T, const int32_t* prefix, int P, int slot, int B,
                            int use_cfg, void* dev_ws, size_t ws_bytes, float* logits_out, void* stream);
/* lg_decode_rows for t2i models: row r takes the token embedding of tokens[r % B] at position pos_rows[r] (every row is past its
 * condition), writes its K / V there and attends over [0, pos_rows[r]]. emb_mask dev f32 [B, T] or NULL: row r attends to condition
 * key j < T iff emb_mask[r % B][j] != 0 or j is its own position (lg_generate's rule). logits_out dev f32 [R, V]. */
int  lg_decode_rows_t2i(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, const float* emb_mask, int B, int use_cfg,
                        float* logits_out, void* stream);

/* ---- negative prompts: a caption in place of the null condition of CFG ---------------------------------------------------------
 * Every *_neg entry point is its sibling without the suffix plus one pair (neg_cond, neg_mask), and the sibling is the call with
 * both NULL. neg_cond: NULL (the unconditional rows take uncond_embedding, as in the sibling) or dev [B, T, caption_dim] in the model
 * dtype, one negative per image (lg_prefill_slot_prefix_neg: [T, caption_dim], the request's), prepared as cond is (left-padded,
 * padding zeroed); the unconditional row of image b embeds neg_cond[b] instead of uncond_embedding. neg_mask: NULL (the
 * unconditional rows attend with emb_mask's rows, as in the sibling) or dev f32 [B, T] (lg_prefill_slot_prefix_neg: [T]); the
 * unconditional row of image b attends to condition key j < T iff neg_mask[b][j] != 0 or j is its own position. A pair that is not
 * NULL needs a t2i model and CFG (cfg_scale > 1, or use_cfg); neg_mask needs neg_cond (lg_decode_rows_t2i_neg takes neg_mask alone)
 * and emb_mask (all ones for an unmasked condition). Every argument is checked before any launch. The negative of
 * uncond_embedding with neg_mask = emb_mask computes exactly what the sibling computes. */
int  lg_generate_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T, int S,
                     const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits, const int32_t* teacher, void* stream);
int  lg_generate_prefix_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B,
                            int T, int S, const lg_sample_cfg* sc, const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes,
                            int32_t* out_tokens, float* dbg_logits, void* stream);
int  lg_generate_sjd_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                         int S, const lg_sample_cfg* sc, int L, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* iters_out,
                         float* dbg_probs, void* stream);
/* The join of a request with a negative (t2i): row B + slot is prefilled with neg_cond [T, caption_dim] and neg_mask [T]. */
int  lg_prefill_slot_prefix_neg(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int T,
                                const int32_t* prefix, int P, int slot, int B, int use_cfg, void* dev_ws, size_t ws_bytes,
                                float* logits_out, void* stream);
/* neg_mask dev f32 [B, T] or NULL: row B + s reads neg_mask[s] instead of emb_mask[s] (needs use_cfg and emb_mask). A serving slot
 * without a negative keeps its emb_mask row there. */
int  lg_decode_rows_t2i_neg(lg_engine* e, const int32_t* tokens, const int32_t* pos_rows, const float* emb_mask, const float* neg_mask,
                            int B, int use_cfg, float* logits_out, void* stream);
/* lg_sample with per-request RNG streams: image b draws with seed_rows[b] at token index step_rows[b] (exactly the draw a
 * batch-of-one lg_generate with that seed makes), result -> out_idx[b] and/or out_seq[b*seq_stride + step_rows[b]]. */
int  lg_sample_rows(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                    const int32_t* step_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream);
/* lg_sample_rows with per-request guidance. cfg_rows dev f32 [B] or NULL: image b mixes with scale cfg_rows[b] in place of
 * sc->cfg_scale, and only when cfg_rows[b] > 1 (a row at scale <= 1 takes its conditional logits and never reads row B + b).
 * interval_rows dev int32 [B] or NULL: image b drops the mix after decode iteration interval_rows[b] in place of sc->cfg_interval
 * (-1 = never). A row given scale s > 1 and interval k draws exactly what lg_sample_rows with cfg_scale = s, cfg_interval = k and
 * mix_cfg draws for it; a row at s <= 1 what lg_sample_rows without mix_cfg draws from its conditional row. A non-NULL cfg_rows or
 * interval_rows needs mix_cfg (logits of 2B rows). lg_sample_rows is this call with both NULL. */
int  lg_sample_rows_guided(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                           const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                           int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream);
/* lg_sample_rows_guided with per-row image indices (parallel sampling: several images of one request). img_rows dev int32 [B], values
 * >= 0, or NULL: image b draws what image img_rows[b] of a lg_generate call with seed seed_rows[b] draws at token index step_rows[b]
 * (lg_sample of that image at that step), where NULL keys every row as image 0 (a batch-of-one call). lg_sample_rows_guided is this
 * call with img_rows NULL. */
int  lg_sample_rows_keyed(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                          const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                          const int32_t* img_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream);
/* KV fan-out of a parallel-sampling join: copies positions [0, len) of every layer's K and V from the rows of slot src_slot (row
 * src_slot and, with use_cfg, row B + src_slot) to the same rows of every slot in dst_slots (host int32 [n_dst]), on `stream`, in
 * whatever the cache stores (the model dtype or e4m3 codes; an fp8 cache's scales are per layer and shared by every row, so they need
 * no copy). Nothing else of the workspace changes. lg_prefill_slot* write the same bytes whatever the slot, so a destination holds
 * what a prefill of it would have written. Refused before any launch: a slot outside [0, B), a destination equal to the source or
 * repeated, len outside [0, max_seq], and a workspace with fewer than nh * B rows. One launch per 64 destinations. */
int  lg_copy_slot_kv(lg_engine* e, int src_slot, const int32_t* dst_slots, int n_dst, int B, int use_cfg, int len, void* stream);
/* ---- token log-probabilities of the sample kernel's draws ----------------------------------------------------------------------
 * x is the f32 row a draw takes its token from: the logits rounded to round_dtype, CFG-mixed with the row's scale and interval,
 * divided by max(temperature, 1e-5), tokens removed by top-k / top-p at -inf. With m = max x and Z = sum exp(x - m) (the kernel's own),
 * the logprob of token v is (x_v - m) - logf(Z), so exp(logprob) is, up to rounding, lg_sample's out_probs. A greedy draw reports the
 * distribution it took the argmax of. Every member is NULL (off) or dev memory indexed as the token row out_seq, element
 * b * seq_stride + step (lg_generate_logprobs: b * S + k):
 *   logprob      f32: the drawn token's logprob;
 *   rank         int32: 1 + #{v : x_v > x_drawn} (on x: distinct logits can round to the same expf);
 *   top_ids      int32 [.., top_n]: the top_n kept tokens by (x descending, id ascending); -1 past the last kept token;
 *   top_logprob  f32 [.., top_n]: their logprobs; -inf past the last kept token.
 * 0 <= top_n <= 20; top_n > 0 needs both top_ids and top_logprob (top_n = 0 ignores them). A NULL lg_logprobs, or one with every
 * member NULL, is off. Turning logprobs on changes no draw. */
typedef struct lg_logprobs {
    float*   logprob;
    int32_t* rank;
    int32_t* top_ids;
    float*   top_logprob;
    int32_t  top_n;
} lg_logprobs;
/* lg_sample_rows_keyed (cfg_rows, interval_rows and img_rows may each be NULL) plus token log-probabilities; lp NULL or off is that
 * call. Logprobs need out_seq (they are indexed as it is). */
int  lg_sample_rows_logprobs(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                             const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                             const int32_t* img_rows, const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq, int seq_stride,
                             void* stream);
/* lg_sample_rows_logprobs with the inpainting select (serving's inpainting requests): given dev int32 [B, seq_stride] or NULL, indexed
 * as out_seq; where given[b][step_rows[b]] >= 0 that token replaces image b's draw in out_idx and out_seq, and every other row draws
 * what lg_sample_rows_logprobs draws. cfg_rows, interval_rows, img_rows, given and lp may each be NULL; given needs out_seq. */
int  lg_sample_rows_given(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                          const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                          const int32_t* img_rows, const int32_t* given, const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq,
                          int seq_stride, void* stream);
/* Composable guidance inside a mixed batch (serving's composed requests): lg_sample_rows_given with mix_cfg = 1, plus a gather table.
 * logits f32 [rows, V], rows >= 2B. mix_rows dev int32 [B][1 + 8] and mix_weights dev f32 [B][8], both NULL or both given; entry 0 of
 * row b is its role:
 *   -2      a condition row: nothing of row b is written (its logits are read by the lead row that names them);
 *   -1      a plain row: conditional row b and unconditional row B + b, cfg_rows[b] / interval_rows[b], exactly what
 *           lg_sample_rows_given draws for it;
 *   u >= 0  a lead row: x = u + w_1 (c_1 - u) + ... + w_K (c_K - u) with u = logits row u, c_i = logits row mix_rows[b][i] for
 *           i = 1 .. K (1 <= K <= 8; entry K + 1, if any, is -1) and w_i = mix_weights[b][i - 1], every row rounded to round_dtype
 *           first and the sum accumulated left to right in fp32, as in lg_generate_composed; always mixed, except that interval_rows[b]
 *           drops the mix as for a plain row (sc->cfg_scale and cfg_rows[b] are unused).
 * The RNG key (seed_rows[b], step_rows[b], img_rows[b]), the given select, the logprobs and out_idx[b] / out_seq[b, step] are row b's.
 * The row indices inside mix_rows are unchecked on the device (the caller's contract: in [0, rows)). With mix_rows NULL this is
 * lg_sample_rows_given with mix_cfg = 1. Every argument the host can check is checked before any launch. */
int  lg_sample_rows_composed(const float* logits, int rows, int B, int V, int round_dtype, const lg_sample_cfg* sc,
                             const uint64_t* seed_rows, const int32_t* step_rows, const float* cfg_rows, const int32_t* interval_rows,
                             const int32_t* img_rows, const int32_t* given, const int32_t* mix_rows, const float* mix_weights,
                             const lg_logprobs* lp, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream);
/* generate() with token log-probabilities [B, S] (top: [B, S, top_n]), in one call covering lg_generate (neg_cond NULL, P = 0),
 * lg_generate_neg (neg_cond, neg_mask as there) and lg_generate_prefix(_neg) (1 <= P <= S - 1, prefix and dev_ws as there; P = 0
 * needs neither and ignores them). The tokens are those of that call. Rows k < P (given tokens) get logprob 0, rank 0, top ids -1 and
 * top logprobs -inf, so the row sum of logprob is the cumulative logprob of the drawn tokens. No teacher or dbg_logits: lg_generate
 * and lg_score cover those. */
int  lg_generate_logprobs(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                          int S, const lg_sample_cfg* sc, const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes,
                          const lg_logprobs* lp, int32_t* out_tokens, void* stream);
/* Fused CFG-mix + temperature + top-k + top-p + softmax + (argmax | multinomial): generate.py:57-66,95-97.
 * logits f32 [rows, V] (rows = 2B when mix_cfg, cond rows first); writes out_idx int32 [B] and, when
 * non-NULL, out_probs f32 [B, V] (the post-filter softmax the reference returns as `probs`).
 * round_dtype: LG_DTYPE_BF16 / LG_DTYPE_F16 round raw logits to bf16 / fp16 first (the reference's `.float()` of a 16-bit head);
 * LG_DTYPE_F32 uses them as they are. */
int  lg_sample(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
               uint64_t step, int32_t* out_idx, float* out_probs, void* stream);
/* Whole generate(): prefill + (S-1) decode steps, tokens never leave the device.
 * out_tokens dev int32 [B, S]. dbg_logits: NULL or dev f32 [S, B, V] receiving the (CFG-mixed, unfiltered)
 * logits of every step. teacher: NULL or dev int32 [B, S] tokens to feed instead of the sampled ones. */
int  lg_generate(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S,
                 const lg_sample_cfg* sc, int32_t* out_tokens, float* dbg_logits,
                 const int32_t* teacher, void* stream);

/* ---- image completion: generate() after a given prefix of every image's tokens ---------------------------------------------- */
/* Bytes of caller-provided scratch for lg_generate_prefix's prefill of `rows` rows (2 per image under CFG) of `seq` = T + P positions. */
int  lg_prefix_workspace_bytes(lg_engine* e, int rows, int seq, size_t* bytes);
/* generate() that continues given images: token indices 0 .. P - 1 of image b are prefix[b, 0 .. P - 1] (dev int32 [B, P],
 * 1 <= P <= S - 1) and are copied to out_tokens[b, 0 .. P - 1]. Positions 0 .. T + P - 1 (the condition as lg_prefill embeds it, with
 * the null condition for CFG rows and emb_mask as in lg_prefill, then the prefix embeddings) are written into the KV cache of
 * lg_engine_set_workspace in one forward pass, not P decode steps. Token P is sampled from the logits of position T + P - 1 with step
 * P; decoding then continues at position T + P with steps P + 1 .. S - 1 exactly as in lg_generate (graph, fused tail, chains). Token
 * k >= P is drawn with lg_generate's RNG key and cfg_interval rule for index k. dbg_logits: NULL or dev f32 [S, B, V]; rows k >= P
 * are written, rows k < P are left as they are. The prefix ids must lie in [0, vocab_size): they index the token embedding table on
 * the device unchecked (generate(prefix=...) checks them on the host). The workspace needs rows >= R and max_seq >= T + S, as for
 * lg_generate. dev_ws
 * (256-byte aligned, at least lg_prefix_workspace_bytes of one image's rows) holds the prefill's activations only; the prefill runs
 * in chunks of cache rows that fit ws_bytes and the attention grid. */
int  lg_generate_prefix(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc,
                        const int32_t* prefix, int P, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, float* dbg_logits,
                        void* stream);

/* ---- inpainting: generate() that keeps any given tokens of every image and draws the rest ----------------------------------------
 * given: HOST int32 [B, S]; given[b][k] in [0, vocab_size) is image b's token k, -1 means token k of image b is drawn. At least one
 * token must be drawn. The call cuts [0, S) into segments, one rule and no option:
 *   LEAD    the leading run of tokens given to every image (length P >= 0): prefilled with the condition in one pass, as
 *           lg_generate_prefix (P > 0) or lg_generate (P = 0) prefill; its head draws token P;
 *   DECODE  one decode step (lg_generate's graph, fused tail and chains) per token that some image draws; images whose token is
 *           given there take it;
 *   EXTEND  each interior run of K tokens given to every image: one window pass feeds tokens k .. k + K (k: the drawn token before the
 *           run) at positions T + k .. in chunks of at most 64 rows, writes their K / V, and the head over its last row gives the
 *           logits of token k + K + 1;
 *   TAIL    a trailing run given to every image: copied, no forward pass.
 * A drawn token k of image b is drawn as lg_generate draws it (RNG key (seed, b, k), cfg_interval by token index, the same
 * temperature / top-k / top-p), from logits that have seen every token before k, given or drawn; never a given token after k.
 * out_tokens dev int32 [B, S]: given tokens where given, drawn ones elsewhere. A mask that gives only a leading run of P tokens is
 * lg_generate_prefix's call, and one that gives nothing is lg_generate's, bit for bit. neg_cond, neg_mask: NULL, or a negative
 * prompt as for lg_generate_neg. dev_ws: 256-byte aligned, lg_given_workspace_bytes of this given array; the call uploads given into
 * it once, on `stream` before any other work of the call, from the engine's pinned staging buffer: the host waits only until the
 * previous call's upload has read that buffer, never for the rest of the stream. Bytes past what lg_given_workspace_bytes counts before the prefill go to the prefill, which runs in chunks of rows as
 * lg_generate_prefix's does (at least one image's rows must fit). Every argument is checked before any launch; the workspace needs
 * rows >= nh * B and max_seq >= T + S. */
int  lg_given_workspace_bytes(lg_engine* e, const int32_t* given, int B, int S, int use_cfg, size_t* bytes);
int  lg_generate_given(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int T,
                       int S, const lg_sample_cfg* sc, const int32_t* given, void* dev_ws, size_t ws_bytes, int32_t* out_tokens,
                       void* stream);
/* ---- composable guidance: generate() that steers every image with K weighted conditions -------------------------------------------
 * B images, K conditions each (1 <= K <= 8, B * K <= 65535). Image j's K conditions are rows j K + i of R = B K conditional rows
 * (image-major), paired with R unconditional rows; the prefill, decode, attention, masks and KV cache run on them as on R images of
 * lg_generate (the workspace needs rows >= 2R and max_seq >= T + S). Per row (R rows, image-major): cond (c2i: int32 [R] class ids in
 * [0, num_classes), unchecked on the device; t2i: [R, T, caption_dim]), emb_mask [R, T] or NULL, neg_cond / neg_mask as for
 * lg_generate_neg or NULL, prefix dev int32 [R, P], given HOST int32 [R, S] (as lg_generate_given's): the caller repeats an image's
 * negative, prefix and given row K times (the call refuses given rows of an image that differ). weights: dev f32 [B, K], finite.
 * Every token of image j is drawn from x = u + d, d = w_1 (c_1 - u) + w_2 (c_2 - u) + ... accumulated left to right in fp32, where
 * c_i is the logit row of row j K + i and u that of unconditional row R + j K (the null condition, or the negative; it attends with
 * row j K's emb_mask, or its neg_mask), each row rounded to the model dtype first. Temperature, top-k, top-p, greedy and the RNG key
 * (seed, token index, image j) are lg_generate's; sc->cfg_scale is unused (the weights are the scales) and sc->cfg_interval must be
 * < 0 unless K = 1, where it drops the mix as in lg_generate. So K = 1 with weight s > 1 draws lg_generate's tokens at cfg_scale = s,
 * and a zero weight drops its condition. The other R - B unconditional rows are computed and never read.
 * out_tokens dev int32 [B, S]; lp: NULL or logprobs as for lg_generate_logprobs, [B, S] (of the composed distribution). P = 0 and
 * given NULL: lg_generate's plan; 1 <= P <= S - 1: lg_generate_prefix's (dev_ws as there, for 2R rows); given: lg_generate_given's
 * (dev_ws: lg_given_workspace_bytes of the R given rows with use_cfg; no prefix, no logprobs). Every argument is checked before any
 * launch. */
int  lg_generate_composed(lg_engine* e, const void* cond, const float* emb_mask, const void* neg_cond, const float* neg_mask, int B, int K,
                          int T, int S, const lg_sample_cfg* sc, const float* weights, const int32_t* prefix, int P, const int32_t* given,
                          void* dev_ws, size_t ws_bytes, const lg_logprobs* lp, int32_t* out_tokens, void* stream);
/* Bytes of caller-provided scratch for lg_extend_slot with a run of K given tokens, K in [1, block_size - 2] (c2i and t2i models). */
int  lg_slot_extend_workspace_bytes(lg_engine* e, int use_cfg, int K, size_t* bytes);
/* The EXTEND of one serving slot (an inpainting request): tokens dev int32 [S], the slot's token row, holds the drawn token a - 1 and
 * the given tokens a .. a + K - 1 (1 <= a, K >= 1, a + K <= S - 1). Feeds tokens a - 1 .. a + K - 1 at positions T + a - 1 .. of row
 * `slot` and, with use_cfg, of row B + slot, each row alone in window chunks of at most 64 positions (lg_generate_given's extend pass of
 * one image and one row), and writes the K / V of positions T + a - 1 .. T + a + K - 1 of those rows and nothing else of the workspace.
 * emb_mask (t2i only): dev f32 [T] or NULL, the conditional row's mask; neg_mask: dev f32 [T] or NULL, the unconditional row's (needs
 * use_cfg and emb_mask; NULL: emb_mask). logits_out dev f32 [nh, V]: the head output at position T + a + K - 1 (the logits of token
 * a + K), one head GEMM over the request's nh rows, rounded as lg_prefill_slot rounds them. The arithmetic depends on neither slot, B
 * nor any other row. dev_ws: 256-byte aligned, at least lg_slot_extend_workspace_bytes. Every argument, and the attention kernel of
 * every chunk, is checked before any launch; the workspace needs rows >= nh * B and max_seq >= T + a + K. */
int  lg_extend_slot(lg_engine* e, const int32_t* tokens, int S, int a, int K, int slot, int B, int use_cfg, const float* emb_mask,
                    const float* neg_mask, void* dev_ws, size_t ws_bytes, float* logits_out, void* stream);

/* ---- teacher-forced scoring: Transformer.forward(idx, cond_idx, targets) (gpt.py:341-382, eval mode) ----------------------- */
/* Bytes of caller-provided scratch for lg_score over `rows` sequences (rows = 2B under CFG) of `seq` positions (T + S - 1). */
int  lg_score_workspace_bytes(lg_engine* e, int rows, int seq, size_t* bytes);
/* Teacher-forced forward (gpt.py:341-382, eval mode): for each image b the sequence is the condition (T positions, as lg_prefill
 * embeds it; emb_mask as in lg_prefill) followed by the token embeddings of idx[b, 0..S-2]. Scores the S positions T-1 .. T+S-2.
 * idx dev int32 [B, S-1] (NULL iff S == 1); targets dev int32 [B, S] or NULL.
 * use_cfg: rows doubled with the null condition, as lg_prefill does; both halves read the same idx. The scored logits are
 * uncond + (cond - uncond) * cfg_scale (generate.py:79-82,95-97).
 * logits_out: NULL or dev f32 [B, S, V]. Holds the head output rounded to the model dtype, as lg_prefill / lg_decode_step return it,
 * CFG-mixed when use_cfg. nll_out: NULL or dev f32 [B, S], -log_softmax(logits)[target] (needs targets; NaN for a target outside
 * [0, V)). At least one of the two is given.
 * Uses only dev_ws (lg_score_workspace_bytes, 256-byte aligned); never touches the workspace of lg_engine_set_workspace, so a
 * generation's KV cache survives. K and V are kept for one layer at a time, always in the model dtype (also after
 * lg_engine_set_kv_cache). May process the batch in image chunks that fit ws_bytes; a CFG twin always stays in its image's chunk. */
int  lg_score(lg_engine* e, const void* cond, const float* emb_mask, const int32_t* idx, const int32_t* targets, int B, int T, int S,
              int use_cfg, float cfg_scale, void* dev_ws, size_t ws_bytes, float* logits_out, float* nll_out, void* stream);

/* ---- speculative Jacobi decoding (Teng et al. 2024): up to L tokens per forward pass, same distribution as lg_generate ------------ */
/* Bytes of caller-provided scratch for lg_generate_sjd with B images and window L (use_cfg: rows doubled). */
int  lg_sjd_workspace_bytes(lg_engine* e, int B, int use_cfg, int L, size_t* bytes);
/* generate() with a window of L tokens per pass (2 <= L <= 64, L <= S - 1). Token 0 is drawn by the prefill exactly as lg_generate
 * draws it. Each pass feeds image b's last final token and L - 1 drafts at positions T + s_b - 1 .. T + s_b + L - 2 (s_b: the first
 * token index the window predicts; near the end of the sequence the window is held at s_b = S - L and re-feeds final tokens), then:
 *   accept: for token k = n_b, ... (n_b tokens final) in order, draft d_k is accepted iff u_acc(k) * q_k(d_k) < p_k(d_k), q_k the
 *     distribution it was drawn from; the first rejected k is drawn from normalize(max(0, p_k - q_k)) with u_res(k) by inverse CDF
 *     (an all-zero residual takes x_k, the redraw below); with every draft accepted, the bonus token s_b + L - 1 is x of that slot.
 *     Greedy (sc->greedy): accept iff d_k = argmax p_k; a rejected k and the bonus token take argmax p.
 *   refresh: a draft whose p this pass computed becomes x_k (q_k = p_k); a new index k takes floor(u_init(k) * V) (q = 1 / V).
 * p_k is the distribution lg_generate samples token k from (rounding, CFG mix with cfg_interval by token index, temperature, top-k,
 * top-p). x_k is the sample kernel's own draw from p_k (lg_sample_rows with seed_rows = pass_seed(b, pass), step_rows = k; argmax when
 * greedy). With C1 = 0xA0761D6478BD642F, C2 = 0xE7037ED1A0B428DB, C3 = 0x8EBC6AF09C88C6E3, C4 = 0x9E6C63D0676A9A99,
 * C5 = 0xD6E8FEB86659FD93 and splitmix64 as in lg_sample, all arithmetic mod 2^64:
 *   u_purpose(k) = top 24 bits of sm(sm(sm(seed ^ C1 (k + 1)) ^ C2 (b + 1)) ^ C3 purpose) / 2^24, purpose accept 1, residual 2, init 3
 *   pass_seed(b, pass) = sm(sm(seed ^ C4 (b + 1)) ^ C5 (pass + 1)), pass = 0, 1, ... counting the passes.
 * A finished image's rows keep running; their outputs are unused. out_tokens dev int32 [B, S]; iters_out dev int32 [1]: the passes run.
 * dbg_probs: NULL or dev f32 [S - 1][B][L][V], pass j's p rows at [j] (rows of finished images unspecified). Uses the KV cache of
 * lg_engine_set_workspace (rows >= R, max_seq >= T + S) and dev_ws (lg_sjd_workspace_bytes, 256-byte aligned) for everything else.
 * The host waits for each pass's done flag before it decides on launching the one after next. */
int  lg_generate_sjd(lg_engine* e, const void* cond, const float* emb_mask, int B, int T, int S, const lg_sample_cfg* sc, int L,
                     void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* iters_out, float* dbg_probs, void* stream);

/* ---- SJD over serving slots (serve.LLM(sjd_window=L)): the state of lg_generate_sjd per slot instead of per call ------------------
 * Slot b (KV-cache rows b and, with use_cfg, B + b) is one image of a request with its own seed, image index j (0 unless its start
 * says otherwise) and pass counter, keyed as image j of lg_generate_sjd with that seed: u_purpose(k) and pass_seed(j, pass) with the
 * slot's seed, pass counting the passes since the slot's
 * start (0 at the start). A slot with nfin >= S is frozen: a pass writes nothing of it (out row, window, q, counters); its rows keep
 * running. The state lives in dev_ws (lg_sjd_slots_workspace_bytes, 256-byte aligned); the KV cache is the workspace's
 * (rows >= (use_cfg ? 2 : 1) * B, max_seq >= T + S). Every argument is checked before any launch. */
int  lg_sjd_slots_workspace_bytes(lg_engine* e, int B, int use_cfg, int L, size_t* bytes);
/* Every slot free (frozen for any S): run once on a new scratch and whenever S changes. */
int  lg_sjd_slots_reset(lg_engine* e, int B, int use_cfg, int L, void* dev_ws, size_t ws_bytes, void* stream);
/* Start slot `slot` after its join drew token 0 into out_tokens[slot * S] (dev int32 [B, S]): nfin = 1, its rows at position T, pass
 * counter 0, window [token 0, u_init drafts of `seed`], and its L window rows' guidance (cfg_scale, cfg_interval; read with use_cfg). */
int  lg_sjd_slot_start(lg_engine* e, int slot, int B, int use_cfg, int L, int S, uint64_t seed, float cfg_scale, int cfg_interval,
                       const int32_t* out_tokens, void* dev_ws, size_t ws_bytes, void* stream);
/* lg_sjd_slot_start keyed as image `image` (>= 0) of the call: the slot draws what image `image` of lg_generate_sjd with `seed`
 * draws. lg_sjd_slot_start is this call with image 0. */
int  lg_sjd_slot_start_image(lg_engine* e, int slot, int B, int use_cfg, int L, int S, uint64_t seed, float cfg_scale, int cfg_interval,
                             int image, const int32_t* out_tokens, void* dev_ws, size_t ws_bytes, void* stream);
/* One pass over every slot: the window rows (nh * B * L, at the slots' positions; emb_mask [B, T] and neg_mask [B, T] as in
 * lg_decode_rows_t2i_neg) through the layers and the head, p and x of every row with its slot's seed, token index and guidance (sc: the
 * rest of the sampling configuration), acceptance and the next window, as one pass of lg_generate_sjd. nfin_out: host-pinned or dev
 * int32 [B], every slot's final count after the pass (copied on `stream`). dbg_p: NULL or dev f32 [B][L][V], this pass's p rows. */
int  lg_sjd_pass_slots(lg_engine* e, const lg_sample_cfg* sc, const float* emb_mask, const float* neg_mask, int B, int use_cfg, int S,
                       int L, void* dev_ws, size_t ws_bytes, int32_t* out_tokens, int32_t* nfin_out, float* dbg_p, void* stream);

/* ---- VQ tokenizer: replaces VQModel.decode_code / VectorQuantizer (vq_model.py) ------------------- */
typedef struct lg_vq_cfg {
    int32_t codebook_size;
    int32_t codebook_embed_dim;
    int32_t z_channels;     /* 256 */
    int32_t ch;             /* 128 */
    int32_t num_res_blocks; /* 2 */
    int32_t n_mult;         /* len(decoder_ch_mult) */
    int32_t ch_mult[8];     /* decoder_ch_mult, vq_model.py:421-424 */
    int32_t l2_norm;        /* codebook_l2_norm */
} lg_vq_cfg;

int  lg_vq_create(const lg_vq_cfg* cfg, int device, lg_vq** out);
void lg_vq_destroy(lg_vq* v);
/* Bind by reference state_dict name ("quantize.embedding.weight", "post_quant_conv.weight",
 * "decoder.conv_in.weight", ...). All tensors are f32, NCHW-ordered conv weights as in the checkpoint. */
int  lg_vq_bind_weight(lg_vq* v, const char* name, const void* dev_ptr, const int64_t* shape, int ndim);
/* Repack conv weights to bf16 [Cout][ky][kx][Cin], L2-normalise the codebook once (vq_model.py:264).
 * Synchronises the device. */
int  lg_vq_finalize(lg_vq* v, void* stream);
int  lg_vq_workspace_bytes(lg_vq* v, int B, int grid, size_t* bytes);
/* decode_code (vq_model.py:52-55): codes dev int32 [B, grid*grid] -> out dev f32 NCHW [B,3,H,W]. */
int  lg_vq_decode(lg_vq* v, const int32_t* codes, int B, int grid, void* dev_ws, size_t ws_bytes,
                  float* out_nchw, void* stream);
/* decode_code followed by the samplers' pixel finishing (sample_c2i_ddp.py:141-143 without the optional resize):
 * clamp(127.5*x + 128, 0, 255) -> uint8, NHWC [B,H,W,3], written straight from conv_out's accumulator drain (no fp32 image in
 * HBM). Needs the wgmma conv path (every registry VQ model); bytes equal lg_vq_decode + lg_pixels_to_u8. */
int  lg_vq_decode_u8(lg_vq* v, const int32_t* codes, int B, int grid, void* dev_ws, size_t ws_bytes,
                     uint8_t* out_nhwc, void* stream);
/* VectorQuantizer.forward index path (vq_model.py:215-233): z dev f32 NCHW [B, e_dim, g, g] -> idx int64 [B*g*g]. */
int  lg_vq_argmin(lg_vq* v, const float* z_nchw, int B, int grid, int64_t* out_idx, void* stream);
/* VQModel.encode (vq_model.py:41-45): Encoder.forward :100-124 (Downsample :389-397) -> quant_conv -> VectorQuantizer.forward
 * :215-255 in eval mode. x dev f32 NCHW [B,3,H,W] (square, H a multiple of 2^(n_mult-1)) -> out_idx dev int64 [B*g*g];
 * optional out_quant dev f32 NCHW [B,e_dim,g,g] (the straight-through tensor z + (e[idx] - z)) and out_z (pre-quantisation
 * quant_conv output), either may be NULL. Needs the encoder.* and quant_conv.* tensors bound before lg_vq_finalize; the
 * encoder uses ch_mult of the cfg (the reference's encoder_ch_mult == decoder_ch_mult in both registry entries,
 * vq_model.py:418-422). Workspace: lg_vq_workspace_bytes(B, H / 2^(n_mult-1)). */
int  lg_vq_encode(lg_vq* v, const float* x_nchw, int B, int H, int W, void* dev_ws, size_t ws_bytes, int64_t* out_idx,
                  float* out_quant_nchw, float* out_z_nchw, void* stream);
/* Pixel finishing of the samplers (sample_c2i_ddp.py:141-143): optional F.interpolate(mode='bicubic') to out_h x out_w,
 * then clamp(127.5*x + 128, 0, 255) -> uint8, NCHW f32 in -> NHWC u8 out, one pass. */
int  lg_pixels_to_u8(const float* in_nchw, int B, int C, int H, int W, int out_h, int out_w, uint8_t* out_nhwc, void* stream);

/* ---- per-kernel-class device timing for bench.py's roofline leg --------------------------------------
 * While enabled, launches are bracketed by CUDA events on the launching stream (CUDA-graph replay is bypassed).
 * lg_profile_read synchronises the device and returns the summed duration / launch count of one class
 * (class ids: see `lg_profile_class_name`). */
/* Toggle programmatic dependent launch for subsequent launches (default: on, or LG_PDL=0/1). With it off, CUPTI
 * kernel durations are additive (no early-started kernels waiting on their dependency), which is what the
 * roofline leg of bench.py traces. */
int         lg_set_pdl(int on);
int         lg_profile_enable(int on);
int         lg_profile_reset(void);
int         lg_profile_read(int cls, double* total_ms, uint64_t* launches);
const char* lg_profile_class_name(int cls);   /* NULL past the last class */

/* Cap the number of CTAs (hence SMs) the VQ decoder's tensor-core convolutions occupy: ctas > 0 runs them as that many persistent
 * CTAs, 0 (or any negative value) restores one CTA per tile (the default). Process-wide; used by
 * SamplePipeline so that decoding batch i does not evict the latency-bound AR sampling of batch i+1 from the SMs
 * (the reference runs the two back to back, sample_c2i_ddp.py:128-143). */
int         lg_vq_set_cta_budget(int ctas);

/* ---- T5 text encoder (transformers T5EncoderModel: Flan-T5, T5 v1.1) ------------------------------- */
typedef struct lg_t5 lg_t5;
typedef struct {
    int32_t n_layer, d_model, d_kv, n_head, d_ff, vocab_size;
    int32_t num_buckets;     /* relative_attention_num_buckets (the bucket table itself comes with every call) */
    int32_t gated_gelu;      /* 1: feed_forward_proj "gated-gelu" (wi_0 | wi_1); 0 is refused */
    int32_t dtype;           /* LG_DTYPE_F32 or LG_DTYPE_BF16; LG_DTYPE_F16 is refused (T5 overflows fp16 without HF's clamps) */
    float eps;               /* layer_norm_epsilon */
} lg_t5_cfg;

/* Refuses d_kv != 64, a non-gated feed-forward, fp16 and any other dtype, with a message. */
int  lg_t5_create(const lg_t5_cfg* cfg, int device, lg_t5** out);
void lg_t5_destroy(lg_t5* t5);
/* Weights by their transformers names, dev pointers in the model dtype that stay valid while the encoder lives:
 * shared.weight [vocab][d_model]; encoder.block.{i}.layer.0.SelfAttention.{q,k,v}.weight [n_head * d_kv][d_model],
 * .o.weight [d_model][n_head * d_kv]; encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight [num_buckets][n_head]
 * (shared by every layer); encoder.block.{i}.layer.0.layer_norm.weight, encoder.block.{i}.layer.1.layer_norm.weight [d_model];
 * encoder.block.{i}.layer.1.DenseReluDense.wi_0.weight, wi_1.weight [d_ff][d_model], wo.weight [d_model][d_ff];
 * encoder.final_layer_norm.weight [d_model]. */
int  lg_t5_bind_weight(lg_t5* t5, const char* name, const void* dev_ptr, const int64_t* shape, int ndim, int dtype);
/* Checks every weight's name, dtype, shape and alignment. The encoder borrows the bound tensors and copies none of them, so a later
 * in-place write to one is used by the next lg_t5_encode. Launches nothing and allocates nothing. */
int  lg_t5_finalize(lg_t5* t5);
/* Scratch lg_t5_encode needs for B captions of T tokens (1 <= T <= 512). Needs no GPU. */
int  lg_t5_workspace_bytes(lg_t5* t5, int B, int T, size_t* bytes);
/* last_hidden_state of T5EncoderModel: out (dev [B][T][d_model], model dtype) for ids and mask (dev int32 [B][T]; ids in
 * [0, vocab), mask 1 for a valid token, 0 for padding) and buckets (dev int32 [2T - 1]: entry (j - i) + T - 1 is the relative
 * position bucket of key j seen from query i, values in [0, num_buckets)). Every query row is computed, padded ones too; a row
 * whose mask has no valid key yields finite values. A caption's output does not depend on B or on the other captions of the call:
 * every GEMM runs over fixed 256-row chunks with a plan that depends on its weight shape alone. ws: 256-byte aligned, at least
 * lg_t5_workspace_bytes. Every argument is checked before any launch. */
int  lg_t5_encode(lg_t5* t5, const int32_t* ids, const int32_t* mask, const int32_t* buckets, int B, int T, void* ws,
                  size_t ws_bytes, void* out, void* stream);

/* ---- stand-alone kernels exported for unit parity tests ------------------------------------------- */
/* T5 self-attention alone: out [B * T][H * 64] = softmax(q k^T + bias[bucket(j - i)][h] + mask) v per (caption, head), no 1/sqrt(d)
 * scaling, read from qkv (dev [B * T][3 * H * 64]: q | k | v). mask (dev int32 [B][T], 0 = padded key, which weighs exactly 0),
 * buckets (dev int32 [2T - 1]), bias (dev [num_buckets][H]); every tensor but the int32 ones in dtype. dtype LG_DTYPE_BF16 runs
 * t5_attn_tc_kernel (mma.sync), LG_DTYPE_F32 t5_attn_kernel (CUDA cores, fp32 throughout). path: NULL or receives 1 / 0 for those. */
int  lg_test_t5_attention(int dtype, int B, int T, int H, const void* qkv, const int32_t* mask, const int32_t* buckets, const void* bias,
                          int num_buckets, void* out, int* path, void* stream);

/* y[M,N] (f32) = x[M,K] * w[N,K]^T, operands in `dtype` (LG_DTYPE_F32, _BF16 or _F16); the same dispatch the engine uses. */
int  lg_test_gemm(const void* x, const void* w, int M, int N, int K, int dtype, float* y,
                  void* dev_scratch, size_t scratch_bytes, void* stream);

/* One linear layer of the transformer as the engine composes it, all tensors in `dtype` unless stated (dev, 16-byte aligned):
 * x [M][K]; wa [N][K]; wb [N][K] with epi 2 only (the w1 | w3 pair: the GEMM is x [wa; wb]^T, 2N columns, segment boundary N).
 * small = 0: the batched kernels. norm_in: x' = RMSNorm(x) * norm_in (eps) in scratch (rmsnorm_kernel), then the GEMM on the kernel
 * gemm_plan picks into fp32 split-K slabs, then the epilogue:
 *   epi 0: out_f32 [M][N] f32 = the slabs summed (reduce_f32_kernel)        epi 1: h [M][N] += T(acc) (residual_norm_kernel);
 *   with norm_out also out [M][N] = RMSNorm(h) * norm_out                  epi 2: out [M][N] = silu(T(acc_a)) * T(acc_b)
 *   epi 3: out [M][N] = T(acc)                                              epi 4: out [M][N] = gelu_tanh(T(acc)) (store_act_kernel)
 *   epi 6 (with wb, like epi 2): out [M][N] = T(gelu_tanh(T(acc_a))) * T(acc_b) (gelu_mul_kernel: T5's gated-GELU feed-forward)
 * acc_out (f32 [M][N or 2N], optional): the slabs summed in slab order, as the epilogues sum them.
 * small = 1: one gemv_small call (bf16 / fp16, M <= 8; norm_in is its RMSNorm prologue; epi 0, 1 without norm_out, or 2; no acc_out).
 * path (int[4], optional): {kernel, tile, ksplit, row blocks or PF}; kernel 0 = gemm_skinny_kernel, 1 = gemm_mma_kernel,
 * 2 = gemm_tc_kernel, 3 = gemv_small_kernel (tile: its weight rows per CTA, ksplit 1, then its k chunks in flight PF).
 * Every argument is checked before any launch. Scratch: 256-byte aligned (NULL when the call needs none); the call fails with the
 * size it needs when it is too small. */
int  lg_test_linear(int dtype, int M, int N, int K, const void* x, const void* norm_in, float eps, const void* wa, const void* wb,
                    int epi, const void* norm_out, void* h, void* out, float* out_f32, float* acc_out, int small, void* dev_scratch,
                    size_t scratch_bytes, int* path, void* stream);
/* The path of lg_test_linear without buffers or a GPU, after the same checks of the shape-only arguments: paired = wb is passed.
 * has_norm_in is accepted for symmetry with lg_test_linear; no dispatch rule depends on it. */
int  lg_test_linear_plan(int dtype, int M, int N, int K, int paired, int small, int epi, int has_norm_in, int* plan);

/* lg_test_linear / lg_test_linear_plan with fp8 weights: wa / wb are dev uint8 codes [N][K] in the stored K order with row scales
 * wa_scale / wb_scale (dev f32 [N], checked like lg_engine_finalize checks them: synchronises). fp8 weights run on gemm_tc_kernel
 * (kernel 2: bf16 / fp16, N % 128 == 0 - with wb, N is the segment boundary -, K % 64 == 0, LG_GEMM_TC other than 0) and on
 * gemv_small_kernel (kernel 3, its 16-bit rules and K % 64 == 0); any other call fails with the plan's message. Where both exist,
 * the plan equals lg_test_linear_plan's for the same arguments; acc_out holds the scaled sums scale[n] * sum_k x * code. */
int  lg_test_linear_w8(int dtype, int M, int N, int K, const void* x, const void* norm_in, float eps, const uint8_t* wa,
                       const float* wa_scale, const uint8_t* wb, const float* wb_scale, int epi, const void* norm_out, void* h, void* out,
                       float* out_f32, float* acc_out, int small, void* dev_scratch, size_t scratch_bytes, int* path, void* stream);
int  lg_test_linear_w8_plan(int dtype, int M, int N, int K, int paired, int small, int epi, int has_norm_in, int* plan);

/* One transformer attention call through the engine's own dispatch, attn_plan (honouring LG_ATTN_TMA, LG_ATTN_PREFILL_TC,
 * LG_ATTN_NST and LG_ATTN_DEEP). dtype: the model dtype (LG_DTYPE_F32, _BF16 or _F16); kv_dtype: dtype, or LG_DTYPE_E4M3 for a
 * 16-bit model with k_scale / v_scale powers of two in [2^-8, 2^7] (otherwise both 1). kcache / vcache: dev [n_layer][R][H][max_seq]
 * [hdp] in the KV dtype, hdp = the engine's row width: 112 for hd 100 in a bf16 / fp16 model, hd otherwise (dims hd..hdp-1 are
 * padding and do not affect the result); `layer` is the one attended to. The tensor maps span all n_layer layers, as
 * lg_engine_set_workspace builds them. Query row m = r * Tq + t sits at position pos(r) + t, pos(r) = pos_rows ? pos_rows[r] : (pos_dev ? *pos_dev : 0) + pos_value,
 * and attends keys j <= its position with j >= Tc or emb_mask[r % B][j] != 0 or j == its position (emb_mask dev f32 [B][Tc] or NULL).
 * Input: q (dev [R * Tq][H * hd], post-RoPE) or the QKV GEMM's split-K slabs qkv_partial (dev f32 [ksplit][R * Tq][3 * H * hd]) with
 * freqs (dev f32 [max_seq][hd / 2][2]): fuse = 0 runs the QKV epilogue (q -> q_out, K / V rows written at the query positions) and
 * then the attention; fuse = 1 lets the TMA decode kernel do the epilogue itself (Tq = 1). out: dev [R * Tq][H * hd].
 * path (int[3]) or NULL: kernel (0 = attention_kernel, 1 = attn_tma_kernel, 2 = attn_causal_tc_kernel: Tq > 128 from position 0 on a
 * 16-bit cache in the model dtype, 3 = attn_prefill_tc_kernel, 4 = attn_window_tc_kernel: 2 <= Tq <= 64 at pos_rows on such a cache),
 * TMA ring depth (0 for attention_kernel) and whether the QKV epilogue
 * was fused. R * Tq may exceed 65535 only on kernel 2. Every argument is checked before any launch;
 * the caller keeps *pos_dev + pos_value + Tq <= max_seq and pos_rows[r] < max_seq. */
int  lg_test_attention(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                       void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                       const int32_t* pos_rows, const float* emb_mask, int B, int Tc, const void* q, const float* qkv_partial,
                       int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path, void* stream);
/* lg_test_attention with emb_mask_uncond (dev f32 [B, Tc] or NULL, needs emb_mask): the mask rows r >= B read, row r % B of it (a
 * negative prompt's mask); NULL is lg_test_attention. */
int  lg_test_attention_neg(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                           void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                           const int32_t* pos_rows, const float* emb_mask, const float* emb_mask_uncond, int B, int Tc, const void* q,
                           const float* qkv_partial, int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path,
                           void* stream);
/* The dispatch of lg_test_attention without buffers or a GPU: after the same checks of the shape-only arguments, plan (int[3])
 * receives the (kernel, ring depth, fused) that lg_test_attention reports for the call over an n_layer-layer buffer. pos_kind: 0 =
 * pos_value alone, 1 = a device counter plus pos_value, 2 = per-row positions (pos_value 0). input: 0 = q, 1 = QKV slabs with
 * fuse = 0, 2 = QKV slabs with fuse = 1. The tensor maps count as built when lg_test_attention would build them (bf16 / fp16 rows of
 * a supported width, fewer than 2^31 rows over all layers); none is encoded. */
int  lg_test_attention_plan(int dtype, int kv_dtype, int R, int Tq, int H, int hd, int hdp, int max_seq, int n_layer, int pos_kind,
                            int pos_value, int input, int* plan);

/* Chunks the prefill of the engine's last lg_generate_prefix call ran in (over all chains); -1 for a null engine. chains: NULL or
 * receives the number of decode chains that call ran (1, or 2 under a multi-chain split). */
int  lg_test_prefix_chunks(lg_engine* e, int* chains);
/* Test hook: the segments of lg_generate_given's plan for given (host int32 [B, S]) as {kind (0 LEAD, 1 DECODE, 2 EXTEND, 3 TAIL),
 * start, length} triples, the first max_segs of them into segs_out; returns the number of segments, or -1. DECODE [start, start +
 * length) draws those tokens; EXTEND [start, start + length) holds the given run and draws token start + length; LEAD [0, length)
 * draws token length. */
int  lg_test_given_plan(const int32_t* given, int B, int S, int32_t* segs_out, int max_segs);
/* Test hook: the regions of one scratch layout, as the engine carves it, without a GPU. kind names a *_workspace_bytes function and
 * args (int64 [nargs]) its arguments: 0 lg_engine_workspace_bytes (rows, max_seq), or (rows, max_seq, g, n) for chain g's view of it
 * when n chains split it; 1 lg_score (rows, seq); 2 lg_prefix (rows, seq); 3 lg_slot (use_cfg); 4 lg_slot_prefix (use_cfg, P);
 * 5 lg_slot_extend (use_cfg, K); 6 lg_given (B, S, use_cfg, chains) with given (host int32 [B, S]), the extend windows laid out for
 * that many decode chains; 7 lg_sjd (B, use_cfg, L); 8 lg_sjd_slots (B, use_cfg, L). The first cap regions go to out (int64 [cap][4])
 * as {offset from the scratch's start, bytes, class (0 float or 16-bit data, 1 int32 / uint64 state, 2 KV cache), chain}, in carving
 * order; a chain view reports chain g's part of each region. Returns the number of regions, or -1 after the kind's own checks. */
int  lg_test_scratch_regions(lg_engine* e, int kind, const int64_t* args, int nargs, const int32_t* given, int64_t* out, int cap);
/* Test hook: lg_sample_rows (seed_rows, step_rows dev, as there) with the inpainting select: given dev int32 [B, seq_stride]; where
 * given[b][step_rows[b]] >= 0 that token replaces image b's draw in out_idx (NULL allowed), out_seq (dev [B, seq_stride]) and
 * next_tokens (dev [B] or NULL). Given all -1, every draw is lg_sample_rows' draw. */
int  lg_test_sample_given(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc,
                          const uint64_t* seed_rows, const int32_t* step_rows, const int32_t* given, int32_t* out_idx, int32_t* out_seq,
                          int seq_stride, int32_t* next_tokens, void* stream);
/* Test hook: the sample kernel's composable-guidance mix alone. logits f32 [2 B K, V]: image b's conditional rows b K + i and its
 * unconditional row B K + b K (the other unconditional rows are not read); weights dev f32 [B, K]; seed_rows / step_rows dev [B] (both
 * NULL: sc->seed, step 0, image b). out_idx dev int32 [B]; next_tokens dev int32 [B K] or NULL (image b's token in all K rows). */
int  lg_test_sample_groups(const float* logits, int B, int K, int V, int round_dtype, const lg_sample_cfg* sc, const float* weights,
                           const uint64_t* seed_rows, const int32_t* step_rows, int32_t* out_idx, int32_t* next_tokens, void* stream);
/* The acceptance step of lg_generate_sjd alone, on caller buffers (dev): p, q f32 [B * L][V], qflag, x, win int32 [B * L], nfin,
 * start int32 [B] (updated), out int32 [B][S] (accepted tokens written). Every image must have nfin < S. */
int  lg_test_sjd_verify(int B, int S, int L, int V, int greedy, uint64_t seed, const float* p, const float* q, const int32_t* qflag,
                        const int32_t* x, const int32_t* win, int32_t* nfin, int32_t* start, int32_t* out, void* stream);
/* Test entry: one per-slot pass's verify + refresh (lg_sjd_pass_slots without the forward) on given rows: p dev f32 [B][L][V], x dev
 * int32 [B][L]; the slot state q [B][L][V], qflag, win [B][L], nfin, start [B], seed_slots (uint64) and pass_slots [B] in and out;
 * seed_rows (uint64) / step_rows [B][L] and out [B][S] out. Frozen slots (nfin >= S) are left as they are. */
int  lg_test_sjd_slots(int B, int S, int L, int V, int greedy, const float* p, const int32_t* x, float* q, int32_t* qflag, int32_t* win,
                       int32_t* nfin, int32_t* start, uint64_t* seed_slots, int32_t* pass_slots, uint64_t* seed_rows, int32_t* step_rows,
                       int32_t* out, void* stream);

/* One launch of the sample kernel with every input the engine can give it (dev buffers). logits, B, V, mix_cfg, round_dtype, sc as
 * lg_sample; the step is step, or *step_dev when step_dev is given, or step_rows[b] with seed_rows[b] as the seed (lg_sample_rows);
 * row_offset is added to the image index of the RNG stream and of the dbg_logits row. Optional outputs: out_idx [B], out_probs [B][V],
 * out_seq [B][seq_stride] (element step), next_tokens [B] (the pick, or teacher[b][step] with teacher [B][seq_stride]),
 * dbg_logits [step + 1][dbg_batch or B][V] (the mixed logits before temperature, row row_offset + b).
 * Fused tail (16-bit round_dtype, emb_table [V][D] in that type, D even): rows b, B + b, ... < emb_rows of emb_h [emb_rows][D] take
 * the next token's embedding and, with emb_xn / emb_norm_w [D], of emb_xn its RMSNorm (emb_eps) times emb_norm_w.
 * adv_pos / adv_step (int32 [1] or NULL): advanced by one after every CTA has read the step, through an arrival ticket this call
 * owns; the call then synchronises and fails if the ticket was not left at zero.
 * path: NULL or dev int32 [B][3]: top-k select (0 none, 1 histogram, 2 radix fallback), whether the nucleus trimmed ties at its
 * boundary value (0 / 1), draw ending (0 greedy, 1 claimed by a segment, 2 past-the-end fallback). vec_loads: NULL or host int, 1
 * when the row is staged with 16-byte loads (V % 4 == 0 and logits, dbg_logits 16-byte aligned), 0 for element-wise loads.
 * Every argument is checked before any launch. */
int  lg_test_sample(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, uint64_t step,
                    const int32_t* step_dev, int row_offset, const uint64_t* seed_rows, const int32_t* step_rows, int32_t* out_idx,
                    float* out_probs, int32_t* out_seq, int seq_stride, const int32_t* teacher, int32_t* next_tokens,
                    float* dbg_logits, int dbg_batch, const void* emb_table, void* emb_h, void* emb_xn, const void* emb_norm_w,
                    float emb_eps, int D, int emb_rows, int32_t* adv_pos, int32_t* adv_step, int32_t* path, int* vec_loads,
                    void* stream);
/* The score head of lg_score on caller slabs: partial dev f32 [ks][P * nh][V] (row p * nh + h, h = 1 the unconditional twin).
 * logits (dev f32 [P][V] or NULL): the slabs summed in slab order, rounded to dtype, CFG-mixed with cfg_scale when nh == 2.
 * nll (dev f32 [P] or NULL, needs targets dev int32 [P]): logsumexp(logits[p]) - logits[p][target], NaN for a target outside [0, V). */
int  lg_test_score_head(const float* partial, int ks, int P, int V, int nh, float cfg_scale, int dtype, const int32_t* targets,
                        float* logits, float* nll, void* stream);

/* One VQ decoder/encoder convolution through the decoder's own dispatch (the mma.sync gather kernel or either wgmma kernel,
 * honouring LG_CONV_TC, LG_CONV_SWAP, LG_GN_FUSE and the CTA budget), optionally followed by GroupNorm(32, eps 1e-6)
 * [+ swish] of its output the way a ResnetBlock hands one to the other (statistics taken from the conv's drain when it wrote them).
 * x bf16 NHWC [B,Hin,Win,Cin]; w f32 [Cout][Cin][k][k] (checkpoint layout, repacked here like lg_vq_finalize), bias f32 [Cout].
 * up: 0 = same size, 1 = nearest-2x upsample folded in (k = 3), 2 = Downsample (k = 3, stride 2 over the input zero-padded
 * right/bottom by one). residual: bf16 NHWC or NULL, may alias out_bf. Exactly one output: out_bf (bf16 NHWC), out_nchw (f32 NCHW)
 * or out_u8 (clamp(127.5*y + 128, 0, 255) as uint8 NHWC). gn_gamma / gn_beta: f32 [Cout] or NULL; gn_out: bf16 NHWC.
 * *path: 0 = mma.sync gather kernel, 1 = conv_tc_kernel, 2 = conv_tcw_kernel. *gn_splits: splits of the GroupNorm partial
 * statistics the conv's drain wrote (0: none), copied to gn_partial [B][splits][32][2] (sum, sum of squares) when non-NULL.
 * Scratch: 256-byte aligned; the call fails with the size it needs when it is too small. */
int  lg_test_vq_conv(const void* x, int B, int Hin, int Win, int Cin, const float* w, const float* bias, int Cout, int ksize, int up,
                     const void* residual, void* out_bf, float* out_nchw, uint8_t* out_u8, const float* gn_gamma,
                     const float* gn_beta, int gn_swish, void* gn_out, float* gn_partial, size_t gn_partial_floats,
                     void* dev_scratch, size_t scratch_bytes, int* path, int* gn_splits, void* stream);
/* The stand-alone GroupNorm(32, eps 1e-6) [+ swish] of the VQ models (statistics pass + apply pass): x, y bf16 NHWC [B,HW,C],
 * gamma / beta f32 [C]. Scratch: at least B * 64 * 64 floats. */
int  lg_test_group_norm(const void* x, int B, int HW, int C, const float* gamma, const float* beta, int swish, void* y,
                        void* dev_scratch, size_t scratch_bytes, void* stream);
/* One AttnBlock (vq_model.py:327-351) through the decoder's own run_attn: x bf16 NHWC [B,H,W,C] is read and overwritten with
 * x + proj_out(softmax(q k^T / sqrt(C)) v). The checkpoint tensors (f32; convs [C,C,1,1], vectors [C]) are packed by the engine's own
 * weight setup. attn_bc: images per score chunk, 0 = the engine's rule (S of a chunk <= 256 MiB). Optional outputs (NULL or dev):
 * hn bf16 [B*N,C] (GroupNorm), qk bf16 [B*N,2C] (q | k), vt bf16 [B,C,N] (v transposed), o bf16 [B*N,C] (softmax(.) v of every
 * image), s f32 and p bf16 [bc,N,N]: scores and probabilities of the last chunk (bc images). N = H*W. Synchronises the stream.
 * Scratch: 256-byte aligned; the call fails with the size it needs when it is too small. */
int  lg_test_vq_attn(void* x, int B, int H, int W, int C, const float* norm_w, const float* norm_b, const float* q_w, const float* q_b,
                     const float* k_w, const float* k_b, const float* v_w, const float* v_b, const float* proj_w, const float* proj_b,
                     int attn_bc, void* hn, void* qk, void* vt, void* o, float* s, void* p, void* dev_scratch, size_t scratch_bytes,
                     void* stream);
/* The first layer of lg_vq_decode: codebook cb f32 [n_e,ed] normalised as lg_vq_finalize does (l2 = 0: copied) into cb_out [n_e,ed]
 * with squared row norms sq_out [n_e], then rows cb_out[codes[i]] (codes dev int32 [n]) through post_quant_conv (pq_w f32 [Z,ed,1,1],
 * pq_b [Z]) into out bf16 NHWC [n,Z]. */
int  lg_test_vq_lookup(const int32_t* codes, int n, const float* cb, int n_e, int ed, int l2, const float* pq_w, const float* pq_b, int Z,
                       float* cb_out, float* sq_out, void* out, void* stream);
/* The encoder's first conv as lg_vq_encode runs it: x f32 NCHW [B,3,H,W] (W % 4 == 0), w f32 [ch,3,3,3], bias [ch], ch % 8 == 0
 * -> out bf16 NHWC [B,H,W,ch], 3x3 pad 1 in fp32. */
int  lg_test_vq_conv_in_rgb(const float* x, int B, int H, int W, const float* w, const float* bias, int ch, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LLAMAGEN_B200_H */
