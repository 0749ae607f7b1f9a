"""CPU: the fp8 (e4m3) KV-cache format, its C-ABI entry point and the samplers' --kv-cache-dtype flag."""
import ctypes
import math
import os
import re

import pytest
import torch

from kv_fp8_oracle import KvFp8Oracle, e4m3_bytes, e4m3_values

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SAMPLERS = ["sample_c2i", "sample_c2i_ddp", "sample_t2i", "sample_t2i_ddp"]


def _byte(x, s=1.0):
    return int(e4m3_bytes(torch.tensor([x], dtype=torch.float32), s)[0])


def test_quantiser_matches_hand_computed_bytes():
    # e4m3: sign | 4 exponent bits (bias 7) | 3 mantissa bits; 1.0 = 0x38
    assert _byte(1.0) == 0x38 and _byte(-1.0) == 0xB8 and _byte(0.0) == 0x00
    assert _byte(1.0625) == 0x38            # halfway between 1.0 and 1.125: ties to even (mantissa 000)
    assert _byte(1.1875) == 0x3A            # halfway between 1.125 and 1.25: ties to even -> 1.25
    assert _byte(1.125) == 0x39
    assert _byte(2.0 ** -6) == 0x08          # smallest normal
    assert _byte(2.0 ** -9) == 0x01          # smallest subnormal
    assert _byte(3 * 2.0 ** -9) == 0x03
    assert _byte(2.0 ** -10) == 0x00         # half the smallest subnormal: ties to even -> 0
    assert _byte(448.0) == 0x7E and _byte(-448.0) == 0xFE
    assert _byte(464.0) == 0x7E              # rounds to 448 (no inf in e4m3fn)
    for big in (480.0, 1000.0, 65504.0, float("inf")):
        assert _byte(big) == 0x7E and _byte(-big) == 0xFE   # saturated, never NaN (0x7F)
    # power-of-two scales divide exactly: x / s lands on the same code as x at scale 1
    assert _byte(4.0, 4.0) == 0x38 and _byte(-0.25, 0.25) == 0xB8 and _byte(1000.0, 4.0) == _byte(250.0)
    assert _byte(448.0 * 128, 128.0) == 0x7E and _byte(2.0 ** -17, 2.0 ** -8) == 0x01


def test_dequantised_values_are_exact_in_16_bit():
    codes = torch.arange(256, dtype=torch.uint8)
    vals = codes.view(torch.float8_e4m3fn).float()
    finite = torch.isfinite(vals)
    for e in (-8, 0, 7):
        v = vals[finite] * 2.0 ** e
        for dt in (torch.bfloat16, torch.float16):
            assert torch.equal(v.to(dt).float(), v), (e, dt)
    x = torch.randn(1000, dtype=torch.bfloat16) * 30
    assert torch.equal(e4m3_values(x, 2.0), (e4m3_bytes(x, 2.0).view(torch.float8_e4m3fn).float() * 2).bfloat16())


def test_oracle_default_scales_and_write_point():
    """The fp8 oracle differs from the 16-bit oracle only by the cache quantisation."""
    from util import seeded_state_dict
    cfg = dict(n_layer=2, n_head=2, dim=64, norm_eps=1e-5, rope_base=10000.0, num_classes=10, cls_token_num=1, block_size=16,
               model_type="c2i")
    F_ = 256
    shapes = {"tok_embeddings.weight": (512, 64), "cls_embedding.embedding_table.weight": (11, 64), "norm.weight": (64,),
              "output.weight": (512, 64)}
    for l in range(2):
        p = f"layers.{l}."
        shapes.update({p + "attention.wqkv.weight": (192, 64), p + "attention.wo.weight": (64, 64),
                       p + "feed_forward.w1.weight": (F_, 64), p + "feed_forward.w3.weight": (F_, 64),
                       p + "feed_forward.w2.weight": (64, F_), p + "attention_norm.weight": (64,), p + "ffn_norm.weight": (64,)})
    sd = {k: v.bfloat16() for k, v in seeded_state_dict(shapes, 5).items()}
    orc = KvFp8Oracle(sd, cfg)
    orc.generate(torch.tensor([1, 2]), 4, cfg_scale=4.0, sample_logits=False)
    for l in range(2):
        for cache in (orc.k[l].tensor, orc.v[l].tensor):
            assert torch.equal(cache, e4m3_values(cache)), l     # every stored value is an e4m3 value
        assert orc.k[l].tensor[:, :, 5:].abs().sum() == 0                # rows past the context stay zero


def test_e4m3_dtype_code_matches_header():
    from llamagen_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "llamagen_b200.h")).read()
    assert re.search(r"LG_DTYPE_E4M3\s*=\s*3\b", hdr)
    assert _lib.LG_DTYPE_E4M3 == 3
    assert "lg_engine_set_kv_cache" in hdr and "lg_engine_set_kv_cache" in _lib.SIGNATURES


def _engine(dtype, n_layer=3):
    from llamagen_b200 import _lib
    lib = _lib.load()
    cfg = _lib.ModelCfg(n_layer, 2, 128, 256, 512, 1, 16, 10, 64, _lib.LG_MODEL_C2I, dtype, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    return lib, h


def _set(lib, h, kv_dtype, scales):
    arr = (ctypes.c_float * len(scales))(*scales) if scales is not None else None
    return lib.lg_engine_set_kv_cache(h, kv_dtype, arr)


def test_set_kv_cache_validates_arguments():
    from llamagen_b200 import _lib
    lib, h = _engine(_lib.LG_DTYPE_BF16)
    try:
        assert _set(lib, h, _lib.LG_DTYPE_E4M3, None) == 0
        assert _set(lib, h, _lib.LG_DTYPE_E4M3, [0.5, 2.0, 1.0, 1.0, 2.0 ** -8, 2.0 ** 7]) == 0
        assert _set(lib, h, _lib.LG_DTYPE_BF16, None) == 0                   # back to the model's own dtype
        for bad in (3.0, 2.0 ** 8, 2.0 ** -9, 0.0, -1.0, float("nan"), float("inf"), -0.5):
            assert _set(lib, h, _lib.LG_DTYPE_E4M3, [1.0, 1.0, 1.0, bad, 1.0, 1.0]) < 0, bad
            msg = lib.lg_last_error().decode()
            assert "power" in msg and "layer 1" in msg and "V scale" in msg, msg
        for dt in (_lib.LG_DTYPE_F16, _lib.LG_DTYPE_F32, 4, -1):
            assert _set(lib, h, dt, None) < 0, dt
            assert "unsupported KV-cache dtype" in lib.lg_last_error().decode()
    finally:
        lib.lg_engine_destroy(h)
    lib, h = _engine(_lib.LG_DTYPE_F32)
    try:
        assert _set(lib, h, _lib.LG_DTYPE_E4M3, None) < 0
        assert "bf16 or fp16 model" in lib.lg_last_error().decode()
    finally:
        lib.lg_engine_destroy(h)
    # E4M3 is a cache format, never a model dtype
    cfg = _lib.ModelCfg(2, 2, 128, 256, 512, 1, 16, 10, 64, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_E4M3, 1e-5)
    h2 = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h2)) < 0


def test_set_kv_cache_halves_the_kv_region():
    """fp8 workspaces shrink by exactly the K/V bytes (one byte per element instead of two), up to 256-byte alignment."""
    from llamagen_b200 import _lib
    for hd_dim, n_head, hdp in ((128, 2, 64), (256, 2, 128), (400, 4, 112)):
        lib = _lib.load()
        cfg = _lib.ModelCfg(3, n_head, hd_dim, 256, 512, 1, 16, 10, 64, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_F16, 1e-5)
        h = ctypes.c_void_p()
        assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
        try:
            sizes = []
            for kv in (_lib.LG_DTYPE_F16, _lib.LG_DTYPE_E4M3):
                assert _set(lib, h, kv, None) == 0
                n = ctypes.c_size_t()
                assert lib.lg_engine_workspace_bytes(h, 6, 24, ctypes.byref(n)) == 0
                sizes.append(n.value)
            kv_fp8 = 2 * 3 * 6 * n_head * 24 * hdp
            assert abs((sizes[0] - sizes[1]) - kv_fp8) <= 2 * 256, (hd_dim, sizes, kv_fp8)
        finally:
            lib.lg_engine_destroy(h)


def test_transformer_set_kv_cache_validates_on_cpu():
    from llamagen_b200 import GPT_models
    m = GPT_models["GPT-B"](vocab_size=512, block_size=16)
    m.set_kv_cache("fp8", [[1.0, 2.0]] * m.n_layer)
    assert m._kv_cache[0] == "fp8" and m._kv_cache[1][:2] == (1.0, 2.0)
    for bad in (dict(dtype="int8"), dict(dtype="auto", scales=[[1.0, 1.0]] * m.n_layer), dict(dtype="fp8", scales=[[1.0, 1.0]])):
        with pytest.raises(ValueError):
            m.set_kv_cache(**bad)
    m.set_kv_cache("auto")
    assert m._kv_cache == ("auto", None)


@pytest.mark.parametrize("script", SAMPLERS)
def test_kv_cache_dtype_flag_parses(script):
    import importlib
    mod = importlib.import_module(f"llamagen_b200.sample.{script}")
    assert mod.build_parser().parse_args([]).kv_cache_dtype == "auto"
    assert mod.build_parser().parse_args(["--kv-cache-dtype", "fp8"]).kv_cache_dtype == "fp8"
    with pytest.raises(SystemExit):
        mod.build_parser().parse_args(["--kv-cache-dtype", "e5m2"])


def test_load_gpt_fp8_on_cpu_and_fp32_refusal():
    from llamagen_b200.sample import sample_c2i
    from llamagen_b200.sample.common import load_gpt
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--precision", "fp16", "--kv-cache-dtype", "fp8"])
    m = load_gpt(args, "cpu", 16)
    assert m._kv_cache == ("fp8", None)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--precision", "none", "--kv-cache-dtype", "fp8"])
    with pytest.raises(SystemExit, match="--kv-cache-dtype fp8 needs --precision bf16 or fp16"):
        load_gpt(args, "cpu", 16)


def test_serve_llm_keeps_or_sets_the_kv_cache_setting():
    from llamagen_b200 import GPT_models
    from llamagen_b200.serve import LLM
    m = GPT_models["GPT-B"](vocab_size=512, block_size=16)
    scales = [[0.5, 2.0]] * m.n_layer
    m.set_kv_cache("fp8", scales)
    setting = m._kv_cache
    LLM(m, cfg_scale=4.0, seed=1)                               # default: the model's setting, scales included
    assert m._kv_cache == setting
    LLM(m, cfg_scale=4.0, seed=1, kv_cache_dtype="fp8")         # the dtype it already has: scales kept
    assert m._kv_cache == setting
    LLM(m, cfg_scale=4.0, seed=1, kv_cache_dtype="auto")
    assert m._kv_cache == ("auto", None)
    LLM(m, cfg_scale=4.0, seed=1, kv_cache_dtype="fp8")
    assert m._kv_cache == ("fp8", None)
