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
/* LG_DTYPE_E4M3 (fp8 e4m3, finite, max +-448) is a KV-cache storage type only (lg_engine_set_kv_cache); never a model dtype. */
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
 * except freqs_cis (always f32).  The caller keeps the tensor alive. */
int  lg_engine_bind_weight(lg_engine* e, const char* name, const void* dev_ptr,
                           const int64_t* shape, int ndim, int dtype);
/* Validate that every tensor the configured model needs is bound. */
int  lg_engine_finalize(lg_engine* e);
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
/* lg_sample with per-request RNG streams: image b draws with seed_rows[b] at token index step_rows[b] (exactly the draw a
 * batch-of-one lg_generate with that seed makes), result -> out_idx[b] and/or out_seq[b*seq_stride + step_rows[b]]. */
int  lg_sample_rows(const float* logits, int B, int V, int mix_cfg, int round_dtype, const lg_sample_cfg* sc, const uint64_t* seed_rows,
                    const int32_t* step_rows, int32_t* out_idx, int32_t* out_seq, int seq_stride, void* stream);
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

/* ---- stand-alone kernels exported for unit parity tests ------------------------------------------- */
/* y[M,N] (f32) = x[M,K] * w[N,K]^T, operands in `dtype` (LG_DTYPE_F32, _BF16 or _F16); the same dispatch the engine uses. */
int  lg_test_gemm(const void* x, const void* w, int M, int N, int K, int dtype, float* y,
                  void* dev_scratch, size_t scratch_bytes, void* stream);

/* One transformer attention call through the engine's own dispatch (honouring LG_ATTN_TMA, LG_ATTN_PREFILL_TC, LG_ATTN_NST
 * and LG_ATTN_DEEP). dtype: the model dtype (LG_DTYPE_F32, _BF16 or _F16); kv_dtype: dtype, or LG_DTYPE_E4M3 for a
 * 16-bit model with k_scale / v_scale powers of two in [2^-8, 2^7] (otherwise both 1). kcache / vcache: dev [n_layer][R][H][max_seq]
 * [hdp] in the KV dtype, hdp = the engine's row width: 112 for hd 100 in a bf16 / fp16 model, hd otherwise (dims hd..hdp-1 are
 * padding and do not affect the result); `layer` is the one attended to. The tensor maps span all n_layer layers, as
 * lg_engine_set_workspace builds them. Query row m = r * Tq + t sits at position pos(r) + t, pos(r) = pos_rows ? pos_rows[r] : (pos_dev ? *pos_dev : 0) + pos_value,
 * and attends keys j <= its position with j >= Tc or emb_mask[r % B][j] != 0 or j == its position (emb_mask dev f32 [B][Tc] or NULL).
 * Input: q (dev [R * Tq][H * hd], post-RoPE) or the QKV GEMM's split-K slabs qkv_partial (dev f32 [ksplit][R * Tq][3 * H * hd]) with
 * freqs (dev f32 [max_seq][hd / 2][2]): fuse = 0 runs the QKV epilogue (q -> q_out, K / V rows written at the query positions) and
 * then the attention; fuse = 1 lets the TMA decode kernel do the epilogue itself (Tq = 1). out: dev [R * Tq][H * hd].
 * path (int[3]) or NULL: kernel (0 = attention_kernel, 1 = attn_tma_kernel, 3 = attn_prefill_tc_kernel; 2 is unused),
 * TMA ring depth (0 for attention_kernel) and whether the QKV epilogue was fused. Every argument is checked before any launch;
 * the caller keeps *pos_dev + pos_value + Tq <= max_seq and pos_rows[r] < max_seq. */
int  lg_test_attention(int dtype, int kv_dtype, float k_scale, float v_scale, int R, int Tq, int H, int hd, int hdp, int max_seq,
                       void* kcache, void* vcache, int n_layer, int layer, int pos_value, const int32_t* pos_dev,
                       const int32_t* pos_rows, const float* emb_mask, int B, int Tc, const void* q, const float* qkv_partial,
                       int ksplit, const float* freqs, int fuse, void* q_out, void* out, int* path, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* LLAMAGEN_B200_H */
