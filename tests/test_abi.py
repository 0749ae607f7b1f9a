"""CPU: the C-ABI library builds, loads without a GPU and exports every symbol include/llamagen_b200.h declares."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "llamagen_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lg_[a-z0-9_]+)\s*\(", src)))


def test_library_loads_and_exports_header_symbols():
    from llamagen_b200 import _lib
    lib = _lib.load()
    assert lib.lg_version() == 1
    names = _header_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert set(names) == set(_lib.SIGNATURES), "ctypes signature table out of sync with the header"


def test_no_libcuda_link_dependency():
    # the .so must be loadable on a CPU-only box: static cudart, no DT_NEEDED on libcuda
    from llamagen_b200 import _lib
    import subprocess
    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out


def test_error_reporting_without_gpu():
    from llamagen_b200 import _lib
    lib = _lib.load()
    cfg = _lib.ModelCfg(2, 2, 100, 256, 512, 1, 16, 10, 64, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    rc = lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h))     # head_dim 50 is unsupported
    assert rc < 0 and b"head_dim" in lib.lg_last_error()
    cfg.dim = 128
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    assert lib.lg_engine_finalize(h) < 0 and b"missing weight" in lib.lg_last_error()
    lib.lg_engine_destroy(h)


_GPT_L = dict(n_layer=24, n_head=16, dim=1024, ffn_dim=2816, vocab_size=16384, cls_token_num=1, num_classes=1000, caption_dim=0)
_TINY_T2I = dict(n_layer=2, n_head=4, dim=256, ffn_dim=704, vocab_size=1024, cls_token_num=8, num_classes=0, caption_dim=64)
_TINY_HD100 = dict(n_layer=2, n_head=2, dim=200, ffn_dim=544, vocab_size=1024, cls_token_num=1, num_classes=10, caption_dim=0)


@pytest.mark.parametrize("m, t2i, dtype, kv_fp8, sizes", [
    (_GPT_L, False, "bf16", False, {(2, 17): 3632896, (128, 257): 3252356096}),
    # ffn_dim 704: the w1 | w3 boundary is not on a 128-row tile, so that GEMM plans mma.sync (one slab) instead of wgmma (two)
    (_TINY_T2I, True, "bf16", False, {(2, 17): 234240, (128, 257): 77857792}),
    (_GPT_L, False, "f16", False, {(2, 17): 3632896, (128, 257): 3252356096}),
    (_GPT_L, False, "f32", False, {(2, 17): 7002880, (128, 257): 6487933952}),
    (_TINY_HD100, False, "bf16", False, {(2, 17): 92672, (128, 257): 60867584}),     # 112-wide cache rows
    (_GPT_L, False, "bf16", True, {(2, 17): 1961728, (128, 257): 1635451904}),
], ids=["c2i_bf16_hd64", "t2i_bf16_caption_ffn704", "c2i_f16", "c2i_f32", "c2i_bf16_hd100", "c2i_bf16_kv_fp8"])
def test_workspace_bytes_are_pinned(m, t2i, dtype, kv_fp8, sizes, monkeypatch):
    """The workspace layout (KV caches, activations, GEMM partials, logits, tokens, counters) is host arithmetic: its size, computed
    without a GPU, must not move. The GEMM partials follow the default GEMM plan."""
    from llamagen_b200 import _lib
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    lib = _lib.load()
    dt = {"bf16": _lib.LG_DTYPE_BF16, "f16": _lib.LG_DTYPE_F16, "f32": _lib.LG_DTYPE_F32}[dtype]
    cfg = _lib.ModelCfg(m["n_layer"], m["n_head"], m["dim"], m["ffn_dim"], m["vocab_size"], m["cls_token_num"], 256, m["num_classes"],
                        m["caption_dim"], _lib.LG_MODEL_T2I if t2i else _lib.LG_MODEL_C2I, dt, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    try:
        if kv_fp8:
            assert lib.lg_engine_set_kv_cache(h, _lib.LG_DTYPE_E4M3, None) == 0, lib.lg_last_error()
        got = {}
        for rows, seq in sizes:
            n = ctypes.c_size_t()
            assert lib.lg_engine_workspace_bytes(h, rows, seq, ctypes.byref(n)) == 0, lib.lg_last_error()
            got[(rows, seq)] = n.value
        assert got == sizes
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("ch, ch_mult, z, n_e, sizes", [
    (128, (1, 1, 2, 2, 4), 256, 16384, {(1, 16): 51257344, (64, 16): 3280470016, (3, 24): 349304832,
                                        (128, 16): 6407168000}),          # 128 images at 16x16: chunks of 125
    (128, (1, 2, 2, 4), 256, 16384, {(1, 16): 25894912, (64, 32): 6389596160}),
    (32, (1, 2), 32, 64, {(2, 4): 90112, (4, 16): 3375104}),
], ids=["vq16", "vq8", "tiny"])
def test_vq_workspace_bytes_are_pinned(ch, ch_mult, z, n_e, sizes):
    """The VQ workspace (activations, attention scores, GroupNorm partials, encoder latents) per chunk of images is host
    arithmetic: its size, computed without a GPU, must not move."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    cfg = _lib.VqCfg(n_e, 8, z, ch, 2, len(ch_mult), (ctypes.c_int32 * 8)(*ch_mult), 1)
    h = ctypes.c_void_p()
    assert lib.lg_vq_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
    try:
        got = {}
        for B, grid in sizes:
            n = ctypes.c_size_t()
            assert lib.lg_vq_workspace_bytes(h, B, grid, ctypes.byref(n)) == 0, lib.lg_last_error()
            got[(B, grid)] = n.value
        assert got == sizes
    finally:
        lib.lg_vq_destroy(h)


def test_product_never_imports_oracle():
    """The shipped package must not route through the CPU oracle (graded constraint ③)."""
    pkg = os.path.join(ROOT, "llamagen_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f"{f} imports oracle"
