"""CPU: the GEMM / GEMV dispatch (gemm_plan, gemv_small_plan) through lg_test_linear_plan, which runs lg_test_linear's checks and plan
without buffers or a GPU, and a self-check of the checker test_linear_gpu.py uses.

Every case of test_linear_gpu must plan the path that suite asserts of the kernel that ran; the registry models at every row count
the engine uses must plan the wgmma kernel; gemv_small must admit exactly its documented shapes; the scratch lg_test_linear asks for
must hold the slabs its plan writes; and four deliberately wrong epilogue chains must fail checks 2 and 3."""
import ctypes
import itertools
import math
import re

import pytest
import torch

import test_linear_gpu as tl

LG_DT = tl.LG_DT


def _plan(monkeypatch, dt, M, N, K, paired=False, small=False, epi=0, tc=True):
    """(status, path, error) of lg_test_linear_plan under exactly the GEMM switch tc."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    if not tc:
        monkeypatch.setenv("LG_GEMM_TC", "0")
    out = (ctypes.c_int * 4)(-9, -9, -9, -9)
    rc = lib.lg_test_linear_plan(LG_DT[dt], M, N, K, int(paired), int(small), epi, 0, out)
    return rc, tuple(out), lib.lg_last_error().decode()


@pytest.mark.parametrize("cid", list(tl.CASE_BY_ID))
def test_plan_is_the_path_the_gpu_suite_asserts(cid, monkeypatch):
    c = tl.CASE_BY_ID[cid]
    rc, got, err = _plan(monkeypatch, c.dt, c.M, c.N, c.K, c.epi == 2, c.small, c.epi, c.tc)
    assert rc == 0, err
    assert got == c.expect, f"{cid}: plans {got}, test_linear_gpu asserts {c.expect}"


def test_gpu_cases_cover_every_path():
    cases = tl.CASES
    assert {c.expect[:2] for c in cases} == {(0, 8), (1, 32), (1, 64), (1, 128), (2, 16), (2, 32), (2, 64), (2, 128), (2, 256),
                                             (3, 8), (3, 16), (3, 32)}
    assert {c.expect[0] for c in cases if c.epi == 2} == {0, 1, 2, 3}            # the w1 | w3 pair on every kernel
    assert any(c.epi == 2 and c.N % 128 and not c.small and c.expect[0] == 1 for c in cases)   # F = 704 on mma.sync
    assert {c.M for c in cases if c.small} >= set(range(1, 9))
    assert {1, 16} <= {c.expect[2] for c in cases if c.expect[0] == 2}
    assert any(c.expect[0] == 0 and c.expect[2] == 5 and c.K == 2816 for c in cases)   # skinny: the last k-slice is empty
    assert {(c.dt, c.epi) for c in cases if not c.small} >= {(d, e) for d in ("bf16", "f16") for e in range(5)}


# -------------------------------------------------------------------------------------------------------- registry sweep
REGISTRY = {"GPT-B": (768, 2048), "GPT-L": (1024, 2816), "GPT-XL": (1280, 3584), "GPT-XXL": (1536, 4096), "GPT-XXXL": (2560, 6912),
            "GPT-1B": (2048, 5632), "GPT-3B": (3200, 8704), "GPT-7B": (4096, 11008)}
ROWS = [*range(1, 9), 16, 64, 128, 256]


def _layer_gemms(D, F):
    """(N, K, paired): QKV, wo, w1 | w3, w2, head."""
    return [(3 * D, D, False), (D, D, False), (F, D, True), (D, F, False), (tl.V, D, False)]


def test_registry_models_plan_wgmma_at_every_row_count(monkeypatch):
    from llamagen_b200.gpt import _SHAPES, ModelArgs
    for name, (D, F) in REGISTRY.items():
        assert ModelArgs(dim=_SHAPES[name][2]).ffn_dim == F and _SHAPES[name][2] == D, name
    seen = 0
    for (name, (D, F)), dt, R in itertools.product(REGISTRY.items(), ("bf16", "f16"), ROWS):
        # decode rows (R), the t2i prefill (R * 120) and a teacher-forced score of R sequences of 256 / 576 positions
        for M in (R, R * 120, R * 256, R * 576):
            for N, K, paired in _layer_gemms(D, F):
                rc, got, err = _plan(monkeypatch, dt, M, N, K, paired, epi=2 if paired else 0)
                assert rc == 0, (name, M, N, K, err)
                rblk = min(M, 256)
                assert got[0] == 2 and got[1] == max(16, 1 << (rblk - 1).bit_length()) and got[3] == -(-M // rblk), (name, M, N, got)
                assert 1 <= got[2] <= 16 and got == tl.plan_model(dt, M, N, K, paired, False), (name, M, N, got)
                seen += 1
    assert seen == len(REGISTRY) * 2 * len(ROWS) * 4 * 5


def _small_rule(R, N, K, dt, paired):
    return dt != "f32" and 1 <= R <= 8 and K % 32 == 0 and K >= 256 and R * (2 * K + 16) <= 90 * 1024 and N > 0 and \
        N % (16 if paired else 32) == 0


def test_gemv_small_admits_exactly_its_rule(monkeypatch):
    for dt, R, N, K, paired in itertools.product(("f32", "bf16", "f16"), range(0, 10), (16, 32, 48, 256, 2048, 2080, 8192, 8224, 16384),
                                                 (224, 256, 264, 288, 1280, 8704, 9184, 9216, 11008), (False, True)):
        rc, got, err = _plan(monkeypatch, dt, R, N, K, paired, small=True, epi=2 if paired else 0)
        if _small_rule(R, N, K, dt, paired):
            assert rc == 0 and got == tl.plan_model(dt, R, N, K, paired, True), (dt, R, N, K, paired, got, err)
        else:
            assert rc < 0 and "gemv_small" in err, (dt, R, N, K, paired, got)


@pytest.mark.parametrize("name, r_max", [("GPT-B", 8), ("GPT-XXL", 8), ("GPT-3B", 5), ("GPT-7B", 4)])
def test_small_path_row_limits_of_registry_models(name, r_max, monkeypatch):
    """The engine takes the small path only when all five GEMMs of a step fit gemv_small: GPT-3B leaves it at R >= 6 and GPT-7B at
    R >= 5, because w2's K = ffn_dim rows of activations no longer fit the 90 KiB of shared memory."""
    D, F = REGISTRY[name]
    for R in range(1, 9):
        ok = all(_plan(monkeypatch, "bf16", R, N, K, p, small=True, epi=2 if p else 0)[0] == 0 for N, K, p in _layer_gemms(D, F))
        assert ok == (R <= r_max), (name, R)


def test_scratch_covers_the_planned_slabs(monkeypatch):
    """lg_test_linear sizes its scratch from gemm_partial_floats; with none it fails before any launch and names the size, which
    must hold the ksplit * M * columns floats the plan writes (plus the normalised activations with a prologue)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    fake = ctypes.c_void_p(1 << 20)                   # never dereferenced: the call fails on the scratch check
    for c in tl.CASES:
        if c.small:
            continue
        rc = lib.lg_test_linear(LG_DT[c.dt], c.M, c.N, c.K, fake, fake if c.norm_in else None, ctypes.c_float(1e-5), fake,
                                fake if c.epi == 2 else None, c.epi, fake if c.norm_out else None, fake if c.epi == 1 else None,
                                fake if (c.epi >= 2 or c.norm_out) else None, fake if c.epi == 0 else None, None, 0, None,
                                ctypes.c_size_t(0), None, None)
        err = lib.lg_last_error().decode()
        m = re.search(r"scratch 0 < (\d+)", err)
        assert rc < 0 and m, (c.id, err)
        ncol = 2 * c.N if c.epi == 2 else c.N
        esz = 4 if c.dt == "f32" else 2
        want = tl.plan_model(c.dt, c.M, c.N, c.K, c.epi == 2, False, True)   # LG_GEMM_TC unset here
        need = -(-want[2] * c.M * ncol * 4 // 256) * 256 + (c.M * c.K * esz if c.norm_in else 0)
        assert int(m.group(1)) == need, (c.id, int(m.group(1)), need)


BASE = dict(dt="bf16", M=16, N=256, K=512, paired=False, small=False, epi=0)


@pytest.mark.parametrize("kw, msg", [
    (dict(K=500), "K=500 a multiple of 8"),
    (dict(N=255), "N=255 must be even"),
    (dict(small=True, dt="f32", M=2), "gemv_small: dtype 0 is not bf16 / fp16"),
    (dict(small=True, M=2, K=224), "K=224 must be a multiple of 32 and at least 256"),
    (dict(small=True, M=2, K=264), "K=264 must be a multiple of 32 and at least 256"),
    (dict(small=True, M=2, N=264, paired=True, epi=2), "N=264 must be a positive multiple of 16"),
    (dict(small=True, M=2, N=272), "N=272 must be a positive multiple of 32"),
    (dict(small=True, M=9), "R=9 rows outside 1..8"),
    (dict(small=True, M=6, K=8704), "exceed 90 KiB"),
    (dict(small=True, M=2, epi=3), "no store or gelu epilogue"),
    (dict(epi=1, N=4160), "N %% 4 == 0 and N <= 4096".replace("%%", "%")),
    (dict(epi=2), "wb goes with the SwiGLU epilogue"),
    (dict(paired=True), "wb goes with the SwiGLU epilogue"),
    (dict(dt="f32", epi=5), "epilogue 5 outside 0..4"),
], ids=["k_mod8", "odd_n", "small_f32", "small_k224", "small_k264", "small_paired_n16", "small_n32", "small_r9", "small_smem",
        "small_store", "residual_n4160", "swiglu_without_wb", "wb_without_swiglu", "epi5"])
def test_rejections_without_buffers(kw, msg, monkeypatch):
    a = dict(BASE, **kw)
    rc, got, err = _plan(monkeypatch, a["dt"], a["M"], a["N"], a["K"], a["paired"], a["small"], a["epi"])
    assert rc < 0 and msg in err and err.startswith("lg_test_linear_plan:"), (kw, rc, got, err)


# -------------------------------------------------------------------------------------------------------- the checker itself
def _acc_case(dt, epi, norm_out=False, seed=0, M=64, N=256, K=1024):
    """A float64 accumulator with its bound, as check 1 builds them, and the fp32 accumulator a correct kernel would hand over."""
    g = torch.Generator().manual_seed(seed)
    t = tl.TDT[dt]
    x = torch.randn(M, K, generator=g).to(t).double()
    w = (torch.randn(2 * N if epi == 2 else N, K, generator=g) / math.sqrt(K)).to(t).double()
    if epi == 2:
        w[N:] *= 4
    ref = x @ w.t()
    E = tl.E_REL * (x.abs() @ w.abs().t())
    h = torch.randn(M, N, generator=g).to(t) if epi == 1 else None
    nw = (1 + 0.1 * torch.randn(N, generator=g)).to(t) if norm_out else None
    return ref, E, ref.float(), h, nw, K


MUTANTS = [("silu_no_inner_round", "bf16", 2, False), ("silu_no_inner_round", "f16", 2, False),
           ("residual_unrounded_branch", "bf16", 1, False), ("residual_unrounded_branch", "f16", 1, True),
           ("norm_no_round", "bf16", 1, True), ("norm_no_round", "f16", 1, True),
           ("bf16_in_f16", "f16", 2, False), ("bf16_in_f16", "f16", 3, False), ("bf16_in_f16", "f16", 1, True)]


@pytest.mark.parametrize("dt, epi, norm_out", sorted({(d, e, n) for _, d, e, n in MUTANTS} | {("bf16", 4, False), ("f16", 4, False),
                                                                                                ("f32", 1, True), ("f32", 2, False)}))
def test_checker_accepts_the_right_chain(dt, epi, norm_out):
    ref, E, acc, h, nw, K = _acc_case(dt, epi, norm_out)
    got = tl.restate(dt, epi, acc, h=h, norm_out=nw)
    assert tl.restated_problem(dt, got, tl.restate(dt, epi, acc, h=h, norm_out=nw), epi, acc) is None
    p = tl.chain_problem(got, tl.chain64(dt, epi, ref, E, h=h, norm_out=nw), tl.cap(dt, K, 2 if epi == 2 else 1))
    assert p is None, p


@pytest.mark.parametrize("mut, dt, epi, norm_out", MUTANTS, ids=[f"{m}-{d}-epi{e}{'-norm' if n else ''}" for m, d, e, n in MUTANTS])
def test_checker_rejects_a_wrong_chain(mut, dt, epi, norm_out):
    """Outputs of a deliberately wrong rounding chain, computed from a correct fp32 accumulator, fail check 2 (against the
    restatement) and check 3 (against the float64 chain)."""
    ref, E, acc, h, nw, K = _acc_case(dt, epi, norm_out, seed=1)
    bad = tl.restate(dt, epi, acc, h=h, norm_out=nw, mut=mut)
    assert tl.restated_problem(dt, bad, tl.restate(dt, epi, acc, h=h, norm_out=nw), epi, acc) is not None
    assert tl.chain_problem(bad, tl.chain64(dt, epi, ref, E, h=h, norm_out=nw), tl.cap(dt, K, 2 if epi == 2 else 1)) is not None
