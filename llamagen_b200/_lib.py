"""ctypes binding of libllamagen_b200.so (the C-ABI declared in include/llamagen_b200.h).

There is NO fallback: if the shared library is missing and cannot be built, or a call is made without
a CUDA device, the import / call fails loudly.  torch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64,
                    c_void_p)

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LG_LIB_PATH") or os.path.join(HERE, "lib", "libllamagen_b200.so")

LG_DTYPE_F32, LG_DTYPE_BF16, LG_DTYPE_F16 = 0, 1, 2
LG_DTYPE_E4M3 = 3   # fp8 e4m3: storage of the KV cache (lg_engine_set_kv_cache) and of GEMM weights (lg_engine_bind_weight)
LG_MODEL_C2I, LG_MODEL_T2I = 0, 1


class LgError(RuntimeError):
    """Raised when a C-ABI call returns a negative status (message from lg_last_error())."""


def dtype_code(dtype) -> int:
    """LG_DTYPE_* of a torch dtype (float32, bfloat16 or float16); any other dtype raises LgError."""
    import torch
    codes = {torch.float32: LG_DTYPE_F32, torch.bfloat16: LG_DTYPE_BF16, torch.float16: LG_DTYPE_F16}
    if dtype not in codes:
        raise LgError(f"unsupported precision {dtype}: the sm_90a engine implements fp32, bf16 and fp16")
    return codes[dtype]


class ModelCfg(Structure):
    _fields_ = [("n_layer", c_int32), ("n_head", c_int32), ("dim", c_int32), ("ffn_dim", c_int32),
                ("vocab_size", c_int32), ("cls_token_num", c_int32), ("block_size", c_int32),
                ("num_classes", c_int32), ("caption_dim", c_int32), ("model_type", c_int32),
                ("dtype", c_int32), ("norm_eps", c_float)]


class SampleCfg(Structure):
    """lg_sample_cfg. The four trailing device pointers (0 = NULL, the default) give every image its own temperature (f32), top_k
    (int32), top_p (f32) and greedy flag (int32); positional constructions of the first seven fields keep their meaning."""
    _fields_ = [("cfg_scale", c_float), ("cfg_interval", c_int32), ("temperature", c_float),
                ("top_k", c_int32), ("top_p", c_float), ("greedy", c_int32), ("seed", c_uint64),
                ("temperature_rows", c_void_p), ("top_k_rows", c_void_p), ("top_p_rows", c_void_p), ("greedy_rows", c_void_p)]


class Logprobs(Structure):
    """lg_logprobs: device pointers (0 = off) of the logprob outputs, and top_n in [0, 20]."""
    _fields_ = [("logprob", c_void_p), ("rank", c_void_p), ("top_ids", c_void_p), ("top_logprob", c_void_p), ("top_n", c_int32)]


MAX_TOP_LOGPROBS = 20
MAX_COMPOSE = 8     # conditions per image of composable guidance (lg_generate_composed)


class T5Cfg(Structure):
    _fields_ = [("n_layer", c_int32), ("d_model", c_int32), ("d_kv", c_int32), ("n_head", c_int32), ("d_ff", c_int32),
                ("vocab_size", c_int32), ("num_buckets", c_int32), ("gated_gelu", c_int32), ("dtype", c_int32), ("eps", c_float)]


class VqCfg(Structure):
    _fields_ = [("codebook_size", c_int32), ("codebook_embed_dim", c_int32), ("z_channels", c_int32),
                ("ch", c_int32), ("num_res_blocks", c_int32), ("n_mult", c_int32),
                ("ch_mult", c_int32 * 8), ("l2_norm", c_int32)]


# name -> (restype, argtypes); every symbol include/llamagen_b200.h declares
SIGNATURES = {
    "lg_version": (c_int, []),
    "lg_last_error": (c_char_p, []),
    "lg_launch_count": (c_uint64, []),
    "lg_reset_launch_count": (None, []),
    "lg_engine_create": (c_int, [POINTER(ModelCfg), c_int, POINTER(c_void_p)]),
    "lg_engine_destroy": (None, [c_void_p]),
    "lg_engine_bind_weight": (c_int, [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int, c_int]),
    "lg_engine_finalize": (c_int, [c_void_p]),
    "lg_engine_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_engine_set_workspace": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_int]),
    "lg_engine_set_kv_cache": (c_int, [c_void_p, c_int, POINTER(c_float)]),
    "lg_prefill": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "lg_decode_step": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "lg_decode_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "lg_slot_workspace_bytes": (c_int, [c_void_p, c_int, POINTER(c_size_t)]),
    "lg_prefill_slot": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_slot_prefix_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_prefill_slot_prefix": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_size_t,
                                       c_void_p, c_void_p]),
    "lg_decode_rows_t2i": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "lg_decode_rows_t2i_neg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "lg_prefill_slot_prefix_neg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int,
                                           c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_generate_neg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p,
                                c_void_p, c_void_p, c_void_p]),
    "lg_generate_prefix_neg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p,
                                       c_int, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "lg_generate_sjd_neg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_int,
                                    c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_sample_rows": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                               c_void_p]),
    "lg_sample_rows_guided": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_int, c_void_p]),
    "lg_sample_rows_keyed": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "lg_sample_rows_logprobs": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, POINTER(Logprobs), c_void_p, c_void_p, c_int, c_void_p]),
    "lg_sample_rows_given": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, POINTER(Logprobs), c_void_p, c_void_p, c_int, c_void_p]),
    "lg_sample_rows_composed": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p, c_void_p, POINTER(Logprobs), c_void_p, c_void_p, c_int, c_void_p]),
    "lg_generate_logprobs": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p,
                                     c_int, c_void_p, c_size_t, POINTER(Logprobs), c_void_p, c_void_p]),
    "lg_copy_slot_kv": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "lg_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_uint64, c_void_p,
                          c_void_p, c_void_p]),
    "lg_generate": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p,
                            c_void_p, c_void_p, c_void_p]),
    "lg_prefix_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_generate_prefix": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_int, c_void_p,
                                   c_size_t, c_void_p, c_void_p, c_void_p]),
    "lg_test_prefix_chunks": (c_int, [c_void_p, POINTER(c_int)]),
    "lg_given_workspace_bytes": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_size_t)]),
    "lg_generate_given": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p,
                                  c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_generate_composed": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg),
                                     c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t, POINTER(Logprobs), c_void_p, c_void_p]),
    "lg_test_sample_groups": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "lg_slot_extend_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_extend_slot": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t,
                               c_void_p, c_void_p]),
    "lg_test_given_plan": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int]),
    "lg_test_sample_given": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_int, c_void_p, c_void_p]),
    "lg_score_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_score": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_size_t,
                         c_void_p, c_void_p, c_void_p]),
    "lg_sjd_workspace_bytes": (c_int, [c_void_p, c_int, c_int, c_int, POINTER(c_size_t)]),
    "lg_generate_sjd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(SampleCfg), c_int, c_void_p, c_size_t,
                                c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_sjd_slots_workspace_bytes": (c_int, [c_void_p, c_int, c_int, c_int, POINTER(c_size_t)]),
    "lg_sjd_slots_reset": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "lg_test_scratch_regions": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int]),
    "lg_sjd_slot_start": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_uint64, c_float, c_int, c_void_p, c_void_p, c_size_t,
                                  c_void_p]),
    "lg_sjd_slot_start_image": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_uint64, c_float, c_int, c_int, c_void_p, c_void_p,
                                        c_size_t, c_void_p]),
    "lg_sjd_pass_slots": (c_int, [c_void_p, POINTER(SampleCfg), c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_size_t,
                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_test_sjd_verify": (c_int,[c_int, c_int, c_int, c_int, c_int, c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_test_sjd_slots": (c_int, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_test_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_int, POINTER(SampleCfg), c_uint64, c_void_p, c_int, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p, POINTER(c_int), c_void_p]),
    "lg_test_score_head": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "lg_t5_create": (c_int, [POINTER(T5Cfg), c_int, POINTER(c_void_p)]),
    "lg_t5_destroy": (None, [c_void_p]),
    "lg_t5_bind_weight": (c_int, [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int, c_int]),
    "lg_t5_finalize": (c_int, [c_void_p]),
    "lg_t5_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_t5_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_test_t5_attention": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, POINTER(c_int),
                                     c_void_p]),
    "lg_vq_create": (c_int, [POINTER(VqCfg), c_int, POINTER(c_void_p)]),
    "lg_vq_destroy": (None, [c_void_p]),
    "lg_vq_bind_weight": (c_int, [c_void_p, c_char_p, c_void_p, POINTER(c_int64), c_int]),
    "lg_vq_finalize": (c_int, [c_void_p, c_void_p]),
    "lg_vq_workspace_bytes": (c_int, [c_void_p, c_int, c_int, POINTER(c_size_t)]),
    "lg_vq_decode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_vq_decode_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "lg_vq_argmin": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "lg_vq_encode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p,
                             c_void_p]),
    "lg_pixels_to_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "lg_set_pdl": (c_int, [c_int]),
    "lg_vq_set_cta_budget": (c_int, [c_int]),
    "lg_profile_enable": (c_int, [c_int]),
    "lg_profile_reset": (c_int, []),
    "lg_profile_read": (c_int, [c_int, POINTER(ctypes.c_double), POINTER(c_uint64)]),
    "lg_profile_class_name": (c_char_p, [c_int]),
    "lg_test_gemm": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t,
                             c_void_p]),
    "lg_test_linear": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, POINTER(c_int), c_void_p]),
    "lg_test_linear_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int)]),
    "lg_quantize_rows_e4m3": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "lg_weight_fp8_stored_index": (c_int, [c_int]),
    "lg_test_linear_w8": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t, POINTER(c_int), c_void_p]),
    "lg_test_linear_w8_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int)]),
    "lg_test_attention": (c_int, [c_int, c_int, c_float, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                  c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                  c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int), c_void_p]),
    "lg_test_attention_neg": (c_int, [c_int, c_int, c_float, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                      c_int, c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int), c_void_p]),
    "lg_test_attention_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                       POINTER(c_int)]),
    "lg_test_vq_conv": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t,
                                c_void_p, c_size_t, POINTER(c_int), POINTER(c_int), c_void_p]),
    "lg_test_group_norm": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t,
                                   c_void_p]),
    "lg_test_vq_attn": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_size_t, c_void_p]),
    "lg_test_vq_lookup": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "lg_test_vq_conv_in_rgb": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
}

_lib = None


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """dlopen the in-tree library (building it with nvcc first when it is absent and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise LgError(f"{LIB_PATH} is missing; run `python -m llamagen_b200.build`")
        from . import build as _build
        _build.build()
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == ABI mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str = "") -> None:
    if status < 0:
        msg = load().lg_last_error()
        raise LgError(f"{what}: {msg.decode() if msg else 'unknown error'}")


def require_cuda(t, what: str):
    if not t.is_cuda:
        raise LgError(f"{what}: tensor must live on a CUDA device (llamagen_b200 has no CPU path)")
    return t


def ptr(t) -> c_void_p:
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def current_stream(device) -> c_void_p:
    import torch
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def weight_fp8_stored_index(K: int):
    """int64 [K]: the byte of a stored fp8 weight row that holds column k's code (lg_weight_fp8_stored_index), so that
    stored[:, index] is the row in column order and natural.new_empty(...)[:, index] = natural packs one."""
    import torch
    lib = load()
    return torch.tensor([lib.lg_weight_fp8_stored_index(k) for k in range(K)], dtype=torch.int64)


def shape_array(shape):
    arr = (c_int64 * len(shape))(*[int(s) for s in shape])
    return arr
