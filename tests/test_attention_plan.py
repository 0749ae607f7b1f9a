"""CPU: the attention dispatch (attn_plan) through lg_test_attention_plan, which runs lg_test_attention's checks and plan without
buffers or a GPU. Every call of the GPU attention suites (test_attention_gpu, the causal cases of test_score_gpu and the window
cases of test_sjd_gpu) must plan the (kernel, ring depth, fused) triple those suites assert of the kernel that ran, under the case's
switches; so the table of all five kernels is pinned on any machine. Then the rejections that need no buffer."""
import ctypes

import pytest

import test_attention_gpu as ta
import test_score_gpu as ts
import test_sjd_gpu as tw

SWITCHES = ("LG_ATTN_TMA", "LG_ATTN_PREFILL_TC", "LG_ATTN_DEEP", "LG_ATTN_NST")
LG_DT = {"f32": 0, "bf16": 1, "f16": 2}
LG_E4M3 = 3
POS_KIND = {"scalar": 0, "dev": 1, "rows": 2}
INPUT = {"q": 0, "slab": 1, "fused": 2}

GPU_CASES = ta.CASES + ts._causal_cases() + list(tw.WCASES.values())
CASES = {c.id: c for c in GPU_CASES}
assert len(CASES) == len(GPU_CASES)


def _plan(monkeypatch, env, dt, kv, R, Tq, H, hd, hdp, S, n_layer, pos, inp):
    """(status, (kernel, stages, fused), error) of one call under exactly the attention switches in env."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kind, val = pos
    value = 0 if kind == "rows" else min(val, 7) if kind == "dev" else val     # as test_attention_gpu._run passes the positions
    out = (ctypes.c_int * 3)(-9, -9, -9)
    rc = lib.lg_test_attention_plan(LG_DT[dt], LG_E4M3 if kv == "fp8" else LG_DT[dt], R, Tq, H, hd, hdp, S, n_layer, POS_KIND[kind],
                                    value, INPUT[inp], out)
    return rc, tuple(out), lib.lg_last_error().decode()


@pytest.mark.parametrize("cid", list(CASES))
def test_plan_is_the_kernel_the_gpu_suites_assert(cid, monkeypatch):
    c = CASES[cid]
    rc, got, err = _plan(monkeypatch, c.env, c.dt, c.kv, c.R, c.Tq, c.H, c.hd, c.hdp, c.S, c.layers[0], c.pos, c.inp)
    assert rc == 0, err
    assert got == c.expect, f"{cid}: plans {got}, the GPU suites assert {c.expect}"


def test_gpu_cases_cover_every_kernel_and_ring():
    assert {c.expect[0] for c in GPU_CASES} == {0, 1, 2, 3, 4}
    assert {c.expect[:2] for c in GPU_CASES} == {(0, 0), (1, 2), (1, 3), (1, 8), (2, 2), (3, 1), (4, 2)}


BASE = dict(env={}, dt="bf16", kv="auto", R=2, Tq=1, H=2, hd=64, hdp=64, S=300, n_layer=2, pos=("scalar", 0), inp="q")


@pytest.mark.parametrize("kw, msg", [
    (dict(inp="fused", Tq=2), "fused QKV"),                                    # only the decode kernel (Tq = 1) fuses the epilogue
    (dict(inp="fused", dt="f32"), "fused QKV"),
    (dict(inp="fused", env={"LG_ATTN_TMA": "0"}), "fused QKV"),
    (dict(R=600, Tq=120), "65535"),                                            # kernel 3 would take it; only kernel 2 lifts the limit
    (dict(R=1100, Tq=64, pos=("rows", [0] * 1100)), "65535"),                       # kernel 4 likewise
    (dict(R=58, Tq=1143, S=1150, env={"LG_ATTN_TMA": "0"}), "65535"),          # kernel 2's case on attention_kernel
    (dict(R=58, Tq=1143, S=1150, dt="f32", hd=64, hdp=64), "65535"),
    (dict(hd=100, hdp=100), "row width"),
    (dict(pos=("scalar", 300)), "exceeds max_seq"),
], ids=["fused_tq2", "fused_f32", "fused_tma_off", "prefill_rows", "window_rows", "causal_tma_off", "causal_f32", "row_width",
        "position"])
def test_rejections_without_buffers(kw, msg, monkeypatch):
    rc, got, err = _plan(monkeypatch, **dict(BASE, **kw))
    assert rc < 0 and msg in err and err.startswith("lg_test_attention_plan:"), (kw, rc, got, err)
