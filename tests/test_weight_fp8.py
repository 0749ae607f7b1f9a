"""CPU: the fp8 (e4m3) weight format (scale rule, stored K order), the dispatch of fp8-weight GEMMs through lg_test_linear_w8_plan, and
the Python / CLI surface of `set_weight_dtype`."""
import ctypes
import importlib
import os

import pytest
import torch

import test_linear_gpu as tl
import weight_fp8_oracle as wo
from test_linear_plan import REGISTRY

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "llamagen_b200.h")


# --------------------------------------------------------------------------------------------------- the format
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_scale_rule(dtype):
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * torch.logspace(-2, 2, 64)[:, None]).to(dtype)     # inside fp16's exponent clamp
    w[5] = 0
    codes, s = wo.quantize_rows(w, dtype)
    m, e = torch.frexp(s)
    assert (m == 0.5).all() and s[5] == 1.0                                   # powers of two; a zero row gets 1
    scaled = w.float().abs().amax(1) / s
    live = torch.arange(64) != 5
    assert ((scaled > 224) & (scaled <= 448))[live].all()
    assert (codes[5] == 0).all() and (codes & 0x7F).max() <= 0x7E              # finite codes only
    deq = wo.code_values(codes) * s[:, None]
    assert torch.equal(wo.dequantize(codes, s, dtype).float(), deq)           # code * s is exact in the model dtype
    assert ((deq - w.float()).abs() <= w.float().abs() * 2.0 ** -4 + s[:, None] * 2.0 ** -10).all()   # 3 mantissa bits, RNE
    # re-quantising code * s changes no value
    c2, s2 = wo.quantize_rows(deq.to(dtype), dtype)
    assert torch.equal(wo.code_values(c2) * s2[:, None], deq)


def test_fp16_exponent_clamp_keeps_every_value_representable():
    lo, hi = wo.EXPONENTS[torch.float16]
    assert (lo, hi) == (-15, 7)
    tiny = torch.full((2, 64), 2.0 ** -20, dtype=torch.float16)               # unclamped e would be -29
    codes, s = wo.quantize_rows(tiny, torch.float16)
    assert (s == 2.0 ** -15).all()
    assert torch.equal(wo.dequantize(codes, s, torch.float16), tiny)          # code 2^-5 times 2^-15
    assert 2.0 ** -9 * 2.0 ** lo == 2.0 ** -24                                # the smallest e4m3 subnormal lands on fp16's
    big = torch.full((2, 64), 65504.0, dtype=torch.float16)
    codes, s = wo.quantize_rows(big, torch.float16)
    assert (s == 2.0 ** 7).all() and (codes == 0x7E).all()                    # saturates at 448 * 2^7 = 57344, finite in fp16
    assert torch.isfinite(wo.dequantize(codes, s, torch.float16)).all()
    assert wo.row_scales(torch.full((1, 64), 3e38), torch.bfloat16)[0] == 2.0 ** 64


def test_stored_k_order_round_trip():
    """The stored order is the documented permutation of every 64-wide k-block, and packing then unpacking is the identity."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    K = 192
    idx = _lib.weight_fp8_stored_index(K)
    for k in range(K):
        c, s, h, q, b = k // 64, (k >> 4) & 3, (k >> 3) & 1, (k >> 1) & 3, k & 1
        assert idx[k] == 64 * c + 16 * q + 4 * s + 2 * h + b
    assert sorted(idx.tolist()) == list(range(K)) and lib.lg_weight_fp8_stored_index(-1) < 0
    # piece q of a k-block is, step by step, the m16n8k16 A fragment of lane q: columns 2q, 2q+1, 8+2q, 8+2q+1 of each K = 16 step
    inv = torch.empty(K, dtype=torch.int64)
    inv[idx] = torch.arange(K)
    for q in range(4):
        assert inv[16 * q: 16 * q + 16].tolist() == [16 * s + 8 * h + 2 * q + b for s in range(4) for h in range(2) for b in range(2)]
    codes = torch.randint(0, 256, (5, K), dtype=torch.uint8)
    stored = torch.empty_like(codes)
    stored[:, idx] = codes
    assert torch.equal(stored[:, idx], codes) and not torch.equal(stored, codes)
    hdr = open(HEADER).read()
    assert "64 c + 16 q + 4 s + 2 h + b" in hdr and "lg_weight_fp8_stored_index" in hdr


def test_header_and_bindings_carry_the_new_entry_points():
    from llamagen_b200 import _lib
    hdr = open(HEADER).read()
    for name in ("lg_quantize_rows_e4m3", "lg_weight_fp8_stored_index", "lg_test_linear_w8", "lg_test_linear_w8_plan"):
        assert name in hdr and name in _lib.SIGNATURES
    assert "KV-cache storage type only" not in hdr
    assert _lib.load().lg_version() == 1


def test_compiler_reports_no_spills_and_no_serialised_wgmma():
    """ptxas, on the build's own log: no instantiation of the GEMM and small-row kernels (16-bit or fp8 weights) spills, and no wgmma
    of the fp8 GEMM is serialised because another instruction defines its register operand inside an open wgmma group (C7513)."""
    import re
    from llamagen_b200 import build
    build.build()
    for src, n_kernels in (("gemm_tc", 20), ("gemv_small", 12), ("weight_fp8", 2)):
        path = os.path.join(build.OUT_DIR, f"{src}.ptxas.log")
        if not os.path.exists(path):                                          # a library built before this log was kept
            build.build(force=True)
        log = open(path).read()
        assert "C7513" not in log and "serialized" not in log, src
        frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
        assert len(frames) == n_kernels and all(f == ("0", "0", "0") for f in frames), (src, frames)


def test_signature_follows_in_place_writes_to_fp8_parameters_only():
    m = _tiny()
    sig = m._signature()
    with torch.no_grad():
        m.output.weight.copy_(torch.ones_like(m.output.weight))
    assert m._signature() == sig                                              # 16-bit weights are borrowed: nothing to re-make
    m.set_weight_dtype("fp8")
    sig8 = m._signature()
    with torch.no_grad():
        m.tok_embeddings.weight.add_(1.0)                                     # not an fp8 weight
    assert m._signature() == sig8
    m.load_state_dict({k: v + 1 for k, v in m.state_dict().items()})          # in place: same storage, new versions
    assert m._signature() != sig8


# --------------------------------------------------------------------------------------------------- dispatch
def _plan(monkeypatch, fn, dt, M, N, K, paired=False, small=False, epi=0, tc=True):
    from llamagen_b200 import _lib
    lib = _lib.load()
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    if not tc:
        monkeypatch.setenv("LG_GEMM_TC", "0")
    out = (ctypes.c_int * 4)(-9, -9, -9, -9)
    rc = getattr(lib, fn)(tl.LG_DT[dt], M, N, K, int(paired), int(small), epi, 0, out)
    return rc, tuple(out), lib.lg_last_error().decode()


def test_registry_layers_plan_like_16_bit_weights(monkeypatch):
    """Every registry layer GEMM at R = 2, 8, 16, 128 and 1920 rows (the t2i prefill of 16 rows) plans the wgmma kernel with the
    tile and k-slices of the 16-bit plan, so slabs and epilogues line up; R = 2 (batch 1 under CFG) also plans the small-row kernel."""
    seen = 0
    for (name, (D, F)), dt, M in ((m, d, r) for m in REGISTRY.items() for d in ("bf16", "f16") for r in (2, 8, 16, 128, 1920)):
        for N, K, paired in [(3 * D, D, False), (D, D, False), (F, D, True), (D, F, False), (tl.V, D, False)]:
            epi = 2 if paired else 0
            rc8, p8, err = _plan(monkeypatch, "lg_test_linear_w8_plan", dt, M, N, K, paired, epi=epi)
            rc16, p16, _ = _plan(monkeypatch, "lg_test_linear_plan", dt, M, N, K, paired, epi=epi)
            assert rc8 == 0 and rc16 == 0, (name, M, N, K, err)
            assert p8 == p16 == tl.plan_model(dt, M, N, K, paired, False) and p8[0] == 2, (name, M, N, K, p8, p16)
            if M == 2:                                                        # R = 8 rows of the widest K exceed the kernel's shared memory
                rc8, s8, err = _plan(monkeypatch, "lg_test_linear_w8_plan", dt, M, N, K, paired, small=True, epi=epi)
                assert rc8 == 0 and s8 == tl.plan_model(dt, M, N, K, paired, True), (name, M, N, K, s8, err)
            seen += 1
    assert seen == len(REGISTRY) * 2 * 5 * 5


@pytest.mark.parametrize("kw,msg", [
    (dict(dt="bf16", M=16, N=200, K=512), "fp8 weights need N=200 and the segment boundary 0 on 128-row tiles"),
    (dict(dt="f16", M=64, N=704, K=256, paired=True, epi=2), "fp8 weights need N=1408 and the segment boundary 704 on 128-row tiles"),
    (dict(dt="f32", M=4, N=256, K=512), "fp8 weights need a bf16 or fp16 model"),
    (dict(dt="bf16", M=16, N=256, K=1000), "fp8 weights need K=1000 a multiple of 64"),
    (dict(dt="bf16", M=16, N=256, K=512, tc=False), "fp8 weights run on the wgmma kernel only (LG_GEMM_TC=0)"),
    (dict(dt="bf16", M=4, N=256, K=288, small=True), "gemv_small: fp8 weights need K=288 a multiple of 64"),
    (dict(dt="bf16", M=9, N=256, K=512, small=True), "gemv_small: R=9 rows outside 1..8"),
    (dict(dt="f32", M=4, N=256, K=512, small=True), "gemv_small: dtype 0 is not bf16 / fp16"),
])
def test_planned_errors(kw, msg, monkeypatch):
    """A call no fp8 kernel takes is an error with its reason, never a 16-bit kernel: the same calls plan fine for 16-bit weights."""
    rc, plan, err = _plan(monkeypatch, "lg_test_linear_w8_plan", **kw)
    assert rc < 0 and msg in err, err
    if kw["dt"] != "f32" and kw["M"] <= 8 or not kw.get("small"):
        rc16, _, _ = _plan(monkeypatch, "lg_test_linear_plan", **kw)
        assert rc16 == 0


def test_gpu_cases_plan_the_paths_they_assert(monkeypatch):
    import test_weight_fp8_gpu as tw
    for c in tw.CASES:
        rc, got, err = _plan(monkeypatch, "lg_test_linear_w8_plan", c.dt, c.M, c.N, c.K, c.epi == 2, c.small, c.epi)
        assert rc == 0 and got == c.expect, (c.id, got, c.expect, err)


# --------------------------------------------------------------------------------------------------- Python and CLI
def _tiny():
    from llamagen_b200.gpt import ModelArgs, Transformer
    return Transformer(ModelArgs(n_layer=2, n_head=2, dim=128, block_size=16, vocab_size=512))


def test_set_weight_dtype_validates_and_changes_the_signature():
    m = _tiny()
    assert m._weight_dtype == ("auto", True) and m.fp8_weight_names() == []
    sig = m._signature()
    m.set_weight_dtype("fp8")
    assert m._signature() != sig
    names = m.fp8_weight_names()
    assert len(names) == 2 * 5 + 1 and names[-1] == "output.weight" and "layers.1.feed_forward.w3.weight" in names
    assert not any("norm" in n or "embed" in n for n in names) and set(names) <= set(m.state_dict())
    sig8 = m._signature()
    m.set_weight_dtype("fp8", head=False)
    assert m._signature() != sig8 and "output.weight" not in m.fp8_weight_names()
    for bad in (dict(dtype="int8"), dict(dtype="e4m3"), dict(dtype="fp8", head=1)):
        with pytest.raises(ValueError):
            m.set_weight_dtype(**bad)
    m.set_weight_dtype("auto", head=False)
    assert m._signature() == sig                                              # back to the default setting
    assert set(wo.fp8_names(m.state_dict())) == {n for n in m.state_dict() if n.split(".", 2)[-1] in wo.LAYER_WEIGHTS} | {"output.weight"}


@pytest.mark.parametrize("script", ["sample_c2i", "sample_t2i", "sample_c2i_ddp", "sample_t2i_ddp"])
def test_weight_dtype_flag_parses(script):
    """score_c2i takes the same add_common_args and load_gpt."""
    mod = importlib.import_module(f"llamagen_b200.sample.{script}")
    assert mod.build_parser().parse_args([]).weight_dtype == "auto"
    a = mod.build_parser().parse_args(["--weight-dtype", "fp8", "--kv-cache-dtype", "fp8", "--precision", "fp16"])
    assert (a.weight_dtype, a.kv_cache_dtype, a.precision) == ("fp8", "fp8", "fp16")
    with pytest.raises(SystemExit):
        mod.build_parser().parse_args(["--weight-dtype", "int4"])


def test_load_gpt_applies_the_flag_and_refuses_fp32():
    from llamagen_b200.sample import sample_c2i
    from llamagen_b200.sample.common import load_gpt
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--precision", "fp16", "--weight-dtype", "fp8"])
    m = load_gpt(args, "cpu", 16)
    assert m._weight_dtype == ("fp8", True) and m._kv_cache == ("auto", None)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--precision", "none", "--weight-dtype", "fp8"])
    with pytest.raises(SystemExit, match="--weight-dtype fp8 needs --precision bf16 or fp16"):
        load_gpt(args, "cpu", 16)


def test_serve_llm_keeps_or_sets_the_weight_dtype():
    from llamagen_b200.serve import LLM
    m = _tiny()
    m.set_weight_dtype("fp8", head=False)
    LLM(m, cfg_scale=4.0, seed=1)
    assert m._weight_dtype == ("fp8", False)
    LLM(m, cfg_scale=4.0, seed=1, weight_dtype="fp8")                         # the dtype it already has: head choice kept
    assert m._weight_dtype == ("fp8", False)
    LLM(m, cfg_scale=4.0, seed=1, weight_dtype="auto")
    assert m._weight_dtype == ("auto", True)
    LLM(m, cfg_scale=4.0, seed=1, weight_dtype="fp8")
    assert m._weight_dtype == ("fp8", True)
