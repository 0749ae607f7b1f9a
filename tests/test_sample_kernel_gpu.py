"""GPU: the sample kernel (sampling.cu) one launch at a time through lg_test_sample, and the score head (xf_kernels.cu) through
lg_test_score_head, against a float64 restatement of the same operation.

The row. Everything up to the filter is IEEE fp32 with fixed roundings: the 16-bit rounding of the cond and uncond logits,
u + (c - u) * s (three roundings, the mix dropped once step - 1 > cfg_interval), then x / max(t, 1e-5). It is restated bit-exactly in
numpy fp32 and dbg_logits must equal it.

After that point, with x the staged row, m its kept maximum and float64 p the softmax of the kept set:
- top-k keeps x >= the k-th largest value, ties included; the select is exact, so the kept set must equal the reference's exactly.
- top-p orders the kept tokens by (value descending, index ascending); a token is kept iff E, the float64 mass of the tokens before it
  in that order, is <= top_p (the first token always). E counts the earlier ties at the boundary value, which is the kernel's
  "acc + j * p* <= top_p". The kernel sums the masses with fp32 shared-memory atomics in no fixed order and divides by an fp32 Z, each
  of at most V terms of at most 1, so its E is within NUC_BAND(V) = 2 V 2^-24 of the float64 E; a token whose E lies within that
  band of top_p may go either way. This is a known property of the kernel: the atomic order is free, so such a token can flip from
  run to run.
- out_probs = e / Z, e = expf(x - m) (2 ulp, plus |x - m| 2^-24 from rounding x - m), Z an fp32 sum of ceil(V / 1024) terms per
  thread and two 32-way trees, then one division: relative error <= (|x - m| + ceil(V / 1024) + 18) 2^-24, plus 2^-120
  absolute for kept tokens whose weight underflows. Filtered tokens are exactly 0.
- greedy picks the lowest-index maximum of the kernel's own out_probs.
- a draw with uniform u picks the token whose float64 CDF interval over the kernel's own out_probs holds u, to within
  DRAW_BAND(V) = (ceil(V / 1024) + 16) 2^-24: the segment walk adds ceil(V / 1024) terms to a prefix built by two 5-level scans, the
  target is one product, and out_probs' roundings move the normalised CDF by 2 ulp. Its probability is > 0.
"""
import ctypes
import math
import zlib
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

import sjd_oracle as so

DEV = "cuda"
U24 = 2.0 ** -24
RD = {"f32": 0, "bf16": 1, "f16": 2}
TDT = {"bf16": torch.bfloat16, "f16": torch.float16}


def NUC_BAND(V):
    return 2 * V * U24


def DRAW_BAND(V):
    return (math.ceil(V / 1024) + 16) * U24


# ------------------------------------------------------------------------------------------------ float64 / fp32 restatement
def round16(x, rd):
    """x (float32 array) rounded to bf16 / fp16 (round to nearest even), back in float32; f32: x."""
    if rd == "f32":
        return x
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(TDT[rd]).float().numpy()


def mix_on(mix, step, interval):
    return bool(mix) and not (interval > -1 and step >= 1 and step - 1 > interval)


def restate_row(lc, lu, mix, s, rd):
    """The mixed logits (dbg_logits) of one image in fp32: round16(c), round16(u), u + (c - u) * s."""
    c = round16(lc, rd)
    if not mix:
        return c
    u = round16(lu, rd)
    with np.errstate(invalid="ignore"):
        return (u + (c - u) * np.float32(s)).astype(np.float32)


def stage(x, temperature):
    return (x / np.float32(max(np.float32(temperature), np.float32(1e-5)))).astype(np.float32)


def ref_filter(xs, top_k, top_p):
    """(kept, either): the kept mask after top-k and top-p, and the mask of tokens whose E lies within NUC_BAND of top_p."""
    V = xs.shape[0]
    keep = np.ones(V, bool)
    if top_k > 0:
        k = min(max(top_k, 1), V)
        if k < V:
            keep = xs >= np.sort(xs)[::-1][k - 1]
    amb = np.zeros(V, bool)
    if top_p < 1.0:
        xk = np.where(keep, xs.astype(np.float64), -np.inf)
        e = np.exp(xk - xk.max())
        p = e / e.sum()
        order = np.lexsort((np.arange(V), -xk))
        E = np.concatenate([[0.0], np.cumsum(p[order])[:-1]])
        ok = E <= top_p
        ok[0] = True
        near = np.abs(E - top_p) <= NUC_BAND(V)
        near[0] = False
        kk = np.zeros(V, bool)
        kk[order] = ok
        amb[order] = near & keep[order]
        keep = keep & kk
    return keep, amb


def u_draw(seed, step, rrow):
    """The sample kernel's uniform (sampling.cu): stream key rrow = b + 1 + row_offset, or 1 with a per-row seed."""
    M = so.M64
    r = so.splitmix64(so.splitmix64(seed ^ ((so.C1 * (step + 1)) & M)) ^ ((so.C2 * rrow) & M))
    return float((r >> 40) * U24)


def u_draw_np(seed, steps, rrows):
    """u_draw over numpy uint64 arrays (broadcast)."""
    def sm(x):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))
    with np.errstate(over="ignore"):
        a = np.uint64(seed) ^ (np.uint64(so.C1) * (np.asarray(steps, np.uint64) + np.uint64(1)))
        r = sm(sm(a) ^ (np.uint64(so.C2) * np.asarray(rrows, np.uint64)))
    return (r >> np.uint64(40)).astype(np.float64) * U24


def check_draw(probs, pick, u, V):
    """pick's float64 CDF interval over the kernel's probs holds u within DRAW_BAND(V), and its probability is > 0."""
    p = probs.astype(np.float64)
    assert p[pick] > 0, ("zero-probability pick", pick)
    C = np.cumsum(p)
    lo = (C[pick - 1] if pick > 0 else 0.0) / C[-1]
    hi = C[pick] / C[-1]
    band = DRAW_BAND(V)
    assert lo - band <= u <= hi + band, ("draw outside its interval", pick, u, lo, hi)


# ------------------------------------------------------------------------------------------------ the call
def P(t):
    from llamagen_b200 import _lib
    return _lib.ptr(t)


def sample_call(logits, B, V, *, mix=False, rd="f32", cfg_scale=1.0, interval=-1, temperature=1.0, top_k=0, top_p=1.0, greedy=False,
                seed=1, step=0, step_dev=None, row_offset=0, seed_rows=None, step_rows=None, out_seq=None, seq_stride=0, teacher=None,
                next_tokens=None, dbg=None, dbg_batch=0, emb=None, adv=None, probs=True, path=True):
    """lg_test_sample. Returns (idx, probs or None, path [B][3] or None, vec_loads); writes the optional buffers in place.
    emb: dict(table, h, xn, norm_w, eps, D, rows) or None; adv: (pos, step) int32 tensors or None."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    idx = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    pr = torch.empty(B, V, dtype=torch.float32, device=DEV) if probs else None
    pa = torch.full((B, 3), -1, dtype=torch.int32, device=DEV) if path else None
    sc = _lib.SampleCfg(cfg_scale, interval, temperature, top_k, top_p, 1 if greedy else 0, seed)
    vec = ctypes.c_int(-1)
    e = emb or {}
    _lib.check(lib.lg_test_sample(
        P(logits), B, V, int(mix), RD[rd], ctypes.byref(sc), step, P(step_dev), row_offset, P(seed_rows), P(step_rows), P(idx), P(pr),
        P(out_seq), seq_stride, P(teacher), P(next_tokens), P(dbg), dbg_batch, P(e.get("table")), P(e.get("h")), P(e.get("xn")),
        P(e.get("norm_w")), ctypes.c_float(e.get("eps", 0.0)), e.get("D", 0), e.get("rows", 0), P(adv[0] if adv else None),
        P(adv[1] if adv else None), P(pa), ctypes.byref(vec), _lib.current_stream(DEV)), "lg_test_sample")
    torch.cuda.synchronize()
    return idx.cpu().numpy(), (pr.cpu().numpy() if probs else None), (pa.cpu().numpy() if path else None), vec.value


# ------------------------------------------------------------------------------------------------ the case matrix
@dataclass
class Case:
    id: str
    V: int
    B: int
    kind: str = "gauss"          # gauss | const | neginf | ties2000 | tiedboundary
    rd: str = "f32"
    mix: bool = False
    cfg: float = 1.0
    interval: int = -1
    step: int = 0
    temp: float = 1.0
    top_k: int = 0
    top_p: float = 1.0
    greedy: bool = False
    stepmode: str = "value"      # value | dev | rows
    row_offset: int = 0
    offset4: bool = False        # logits at a 4-byte offset
    expect_topk: int = None      # top-k select path every row must report (None: not asserted)
    expect_trim: int = None      # nucleus tie trim every row must report
    expect_end: set = field(default_factory=lambda: None)   # draw endings the rows must report (and together cover)


def _cases():
    cs = []
    def topk_path(V, k, kind="gauss"):
        if k <= 0 or min(k, V) >= V:
            return 0
        return 2 if kind in ("const", "neginf", "ties2000") else 1
    # top-k: k = 1, 2, 1000, V - 1, V, V + 5 on Gaussian rows, greedy and drawn
    for V in (1000, 16384):
        for k in sorted({1, 2, 1000, V - 1, V, V + 5}):
            cs.append(Case(f"topk{k}_V{V}_greedy", V, 7, top_k=k, greedy=True, expect_topk=topk_path(V, k), expect_end={0}))
            cs.append(Case(f"topk{k}_V{V}_draw", V, 7, top_k=k, step=3, expect_topk=topk_path(V, k), expect_end={1}))
    # degenerate rows: the radix fallback
    cs.append(Case("const_row_k50", 16384, 7, kind="const", top_k=50, step=1, expect_topk=2, expect_end={1}))
    cs.append(Case("neginf_row_k100", 16384, 7, kind="neginf", top_k=100, step=2, expect_topk=2, expect_end={1}))
    cs.append(Case("neginf_row_mix_k3000", 16384, 7, kind="neginf", mix=True, cfg=4.0, top_k=3000, greedy=True, expect_topk=2))
    cs.append(Case("ties2000_k1000", 16384, 7, kind="ties2000", top_k=1000, step=4, expect_topk=2, expect_end={1}))
    cs.append(Case("ties2000_k1000_greedy", 16384, 4, kind="ties2000", top_k=1000, greedy=True, expect_topk=2, expect_end={0}))
    # 16-bit rounding: heavy ties
    for rd in ("bf16", "f16"):
        cs.append(Case(f"{rd}_k1000_mix", 16384, 64, rd=rd, mix=True, cfg=4.0, top_k=1000, step=5, expect_end={1}))
        cs.append(Case(f"{rd}_k50_p09_greedy", 16384, 7, rd=rd, mix=True, cfg=7.5, top_k=50, top_p=0.9, greedy=True, expect_end={0}))
    # top-p alone and with top-k
    for p in (0.9, 0.5, 1e-4, 0.0, -1.0):
        cs.append(Case(f"topp{p}", 16384, 7, top_p=p, step=6, expect_topk=0, expect_end={1}))
        cs.append(Case(f"topp{p}_k1000", 16384, 7, top_k=1000, top_p=p, greedy=True, expect_topk=1, expect_end={0}))
    cs.append(Case("tied_boundary", 1000, 7, kind="tiedboundary", top_p=0.0, step=2, expect_topk=0, expect_trim=1, expect_end={1}))
    cs.append(Case("tied_boundary_greedy", 1000, 4, kind="tiedboundary", top_p=0.0, greedy=True, expect_trim=1, expect_end={0}))
    # shapes: V = 2, 3 (scalar loads), 16383 (scalar), 51200 (the shared-memory limit); B up to 300 (more than one wave)
    cs.append(Case("V2", 2, 64, step=1, expect_end={1}))
    cs.append(Case("V3_k2", 3, 64, top_k=2, step=1, expect_topk=1, expect_end={1}))
    cs.append(Case("V16383_k1000_p09", 16383, 64, top_k=1000, top_p=0.9, step=2, expect_topk=1, expect_end={1}))
    cs.append(Case("V51200_k1000", 51200, 7, top_k=1000, step=1, expect_topk=1, expect_end={1}))
    cs.append(Case("V51200_bf16_greedy", 51200, 4, rd="bf16", mix=True, cfg=4.0, greedy=True, expect_end={0}))
    cs.append(Case("B300_p09", 16384, 300, top_p=0.9, mix=True, cfg=4.0, step=9, expect_end={1}))
    cs.append(Case("B1_k1000", 16384, 1, top_k=1000, step=2, expect_topk=1, expect_end={1}))
    # cfg_interval: the mix is on for step - 1 <= interval and off after
    for st in (0, 4, 5):
        cs.append(Case(f"interval3_step{st}", 16384, 7, mix=True, cfg=4.0, interval=3, step=st, rd="bf16", top_k=100, expect_end={1}))
    # temperature: 1e-6 (clamped to 1e-5), 0.7, 3
    for t in (1e-6, 0.7, 3.0):
        cs.append(Case(f"temp{t}", 16384, 7, temp=t, top_k=1000, step=2, expect_topk=1, expect_end={1}))
    # streams: step_dev, row_offset, per-row seeds
    cs.append(Case("step_dev_offset", 16384, 64, stepmode="dev", step=11, row_offset=5, top_k=1000, expect_end={1}))
    cs.append(Case("rows_stream", 16384, 64, stepmode="rows", top_k=0, expect_end={1}))
    # u = 1 - 2^-24 on every row (seed_rows, step 3): the walk may run past the last segment
    cs.append(Case("past_the_end", 16384, 300, stepmode="rows", step=3, expect_end={1, 2}))
    # the element-wise load path for a row that is not 16-byte aligned
    cs.append(Case("offset4_k1000", 16384, 7, offset4=True, top_k=1000, step=1, expect_topk=1, expect_end={1}))
    cs.append(Case("offset4_mix_bf16", 1000, 7, offset4=True, mix=True, cfg=4.0, rd="bf16", step=1, expect_end={1}))
    return cs


CASES = _cases()
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES)
PAST_END_SEED = 1848047   # sample uniform 1 - 2^-24 at step 3 (checked in the test)


def vec_expected(c):
    return c.V % 4 == 0 and not c.offset4


def test_case_matrix_covers_every_kernel_path():
    """Every case asserts the paths it must take, so the table's expectations are what the GPU run covered."""
    assert {c.expect_topk for c in CASES} >= {0, 1, 2}
    assert {c.expect_trim for c in CASES} >= {1}
    assert {vec_expected(c) for c in CASES} == {False, True}
    assert set().union(*[c.expect_end for c in CASES if c.expect_end]) == {0, 1, 2}
    assert {c.rd for c in CASES} == {"f32", "bf16", "f16"} and {2, 3, 1000, 16383, 16384, 51200} <= {c.V for c in CASES}
    assert {1, 7, 64, 300} <= {c.B for c in CASES} and {c.stepmode for c in CASES} == {"value", "dev", "rows"}
    assert abs(u_draw(PAST_END_SEED, 3, 1) - (1 - U24)) == 0 and u_draw(PAST_END_SEED, 3, 1) == so.sample_uniform(PAST_END_SEED, 3)


def make_logits(c, gen):
    rows = 2 * c.B if c.mix else c.B
    x = (torch.randn(rows, c.V, generator=gen) * 2.7).numpy().astype(np.float32)
    if c.kind == "const":
        x[:] = 1.5
    elif c.kind == "neginf":
        cut = rows // 2 if c.mix else rows   # -inf in cond rows only: -inf - -inf would be NaN in the mix
        sel = torch.rand(cut, c.V, generator=gen).numpy() < 0.1
        x[:cut][sel] = -np.inf
    elif c.kind == "ties2000":
        for r in range(rows):
            perm = torch.randperm(c.V, generator=gen).numpy()
            x[r] = -np.abs(x[r]) - 1.0
            x[r, perm[:500]] = 5.0 + np.abs(x[r, perm[:500]])   # 500 values above the tie
            x[r, perm[500:2500]] = 2.0                            # 2000 exact ties: the 1000th largest is 2.0
    elif c.kind == "tiedboundary":
        # top_p = 0 keeps the first maximum alone; its ties at the boundary value are trimmed in index order
        for r in range(rows):
            perm = torch.randperm(c.V, generator=gen).numpy()
            x[r] = np.minimum(x[r], 3.0)
            x[r, perm[:6]] = 4.0
    return x


def run_case(c):
    seed = zlib.crc32(c.id.encode())
    gen = torch.Generator().manual_seed(seed)
    x = make_logits(c, gen)
    B, V = c.B, c.V
    flat = torch.from_numpy(x.reshape(-1))
    if c.offset4:
        buf = torch.zeros(flat.numel() + 1, dtype=torch.float32, device=DEV)
        buf[1:] = flat.to(DEV)
        logits = buf[1:]
        assert logits.data_ptr() % 16 == 4
    else:
        logits = flat.to(DEV)
    step = c.step
    kw = dict(mix=c.mix, rd=c.rd, cfg_scale=c.cfg, interval=c.interval, temperature=c.temp, top_k=c.top_k, top_p=c.top_p,
              greedy=c.greedy, seed=seed & 0xFFFF, row_offset=c.row_offset)
    seed_rows = step_rows = None
    if c.stepmode == "dev":
        kw["step_dev"] = torch.tensor([step], dtype=torch.int32, device=DEV)
        kw["step"] = 999   # ignored
    elif c.stepmode == "rows":
        if c.id == "past_the_end":
            seed_rows = np.full(B, PAST_END_SEED, np.uint64)
            step_rows = np.full(B, 3, np.int64)
        else:
            seed_rows = (np.arange(B, dtype=np.uint64) * np.uint64(7919) + np.uint64(seed))
            step_rows = (np.arange(B) * 5 + 1) % 37
        kw["seed_rows"] = torch.from_numpy(seed_rows.view(np.int64)).to(DEV)
        kw["step_rows"] = torch.from_numpy(step_rows.astype(np.int32)).to(DEV)
    else:
        kw["step"] = step
    steps = step_rows if step_rows is not None else np.full(B, step)
    S = int(steps.max()) + 1
    seq = torch.full((B, S + 2), -5, dtype=torch.int32, device=DEV)
    dbg_batch = c.row_offset + B
    dbg = torch.full((S, dbg_batch, V), 7.0, dtype=torch.float32, device=DEV) if c.stepmode != "rows" else None
    idx, probs, path, vec = sample_call(logits, B, V, out_seq=seq, seq_stride=S + 2, dbg=dbg, dbg_batch=dbg_batch if dbg is not None
                                        else 0, **kw)
    assert vec == int(vec_expected(c)), (vec, c.id)
    seq = seq.cpu().numpy()
    mix = [mix_on(c.mix, int(steps[b]), c.interval) for b in range(B)]
    for b in range(B):
        lc = x[b]
        lu = x[B + b] if c.mix else None
        xm = restate_row(lc, lu, mix[b], c.cfg, c.rd)
        if dbg is not None:
            got = dbg[int(steps[b]), c.row_offset + b].cpu().numpy()
            assert np.array_equal(got.view(np.int32), xm.view(np.int32)), ("dbg_logits differ from the fp32 restatement", b)
        xs = stage(xm, c.temp)
        keep, amb = ref_filter(xs, c.top_k, c.top_p)
        pb = probs[b]
        # kept set: filtered tokens exactly 0; tokens the reference keeps with a representable probability > 0
        xk = np.where(keep | amb | (pb > 0), xs.astype(np.float64), -np.inf)
        ref_e = np.exp(xk - xk.max())
        ref_p = ref_e / ref_e.sum()
        assert (pb[~keep & ~amb] == 0).all(), ("kept a filtered token", b, np.nonzero(~keep & ~amb & (pb != 0))[0][:8])
        must = keep & ~amb & (ref_p > 2.0 ** -110)
        assert (pb[must] > 0).all(), ("dropped a kept token", b, np.nonzero(must & (pb == 0))[0][:8])
        # probabilities over the kernel's kept set
        S_ = (pb > 0) | must
        xk = np.where(S_, xs.astype(np.float64), -np.inf)
        m = xk.max()
        ref_e = np.exp(xk - m)
        ref_p = ref_e / ref_e.sum()
        rel = (np.where(S_, np.abs(xs - m), 0) + math.ceil(V / 1024) + 18) * U24
        err = np.abs(pb.astype(np.float64) - ref_p)
        worst = float((err / np.maximum(ref_p, 1e-300)).max())
        assert (err <= rel * ref_p + 2.0 ** -120).all(), ("probability outside its bound", b, worst)
        # paths
        if c.expect_topk is not None:
            assert path[b, 0] == c.expect_topk, (b, path[b])
        if c.expect_trim is not None:
            assert path[b, 1] == c.expect_trim, (b, path[b])
        if c.expect_end is not None:
            assert path[b, 2] in c.expect_end, (b, path[b])
        # the pick
        pick = int(idx[b])
        assert seq[b, int(steps[b])] == pick
        if c.greedy:
            assert path[b, 2] == 0 and pick == int(np.argmax(pb)), (b, pick)
        else:
            if seed_rows is not None:
                u = u_draw(int(seed_rows[b]), int(steps[b]), 1)
            else:
                u = u_draw(kw["seed"], step, b + 1 + c.row_offset)
            check_draw(pb, pick, u, V)
            if path[b, 2] == 2:   # past the end: the row's last positive weight, u within the band of 1
                assert pick == int(np.nonzero(pb > 0)[0][-1]) and u >= 1 - DRAW_BAND(V), (b, pick, u)
    # out_seq holds the pick at the step and nothing else
    mask = np.ones_like(seq, bool)
    mask[np.arange(B), steps] = False
    assert (seq[mask] == -5).all()
    return idx, probs, path


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASE_BY_ID))
def test_sample_call(cid):
    c = CASE_BY_ID[cid]
    idx, probs, path = run_case(c)
    if c.id == "past_the_end":
        assert (path[:, 2] == 2).any() and (path[:, 2] == 1).any(), np.bincount(path[:, 2])
    if c.kind == "ties2000":
        assert ((probs > 0).sum(1) == 2500).all()


@pytest.mark.gpu
def test_step_dev_equals_step_value():
    """*step_dev and the same step by value: the same stream, the same dbg row, the same picks."""
    gen = torch.Generator().manual_seed(5)
    B, V = 64, 16384
    x = (torch.randn(2 * B, V, generator=gen) * 2.7).to(DEV)
    outs = []
    for dev in (False, True):
        dbg = torch.zeros(8, B + 3, V, device=DEV)
        kw = dict(step_dev=torch.tensor([6], dtype=torch.int32, device=DEV), step=0) if dev else dict(step=6)
        idx, pr, _, _ = sample_call(x, B, V, mix=True, rd="bf16", cfg_scale=4.0, interval=10, top_k=1000, seed=77, row_offset=3,
                                    dbg=dbg, dbg_batch=B + 3, **kw)
        outs.append((idx, pr, dbg.cpu()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    assert (outs[0][2][6, 3:].abs().sum(-1) > 0).all() and outs[0][2][:6].abs().sum() == 0 and outs[0][2][6, :3].abs().sum() == 0


@pytest.mark.gpu
def test_misaligned_logits_take_the_scalar_path():
    """Logits at a 4-byte offset with V % 4 == 0 are staged element by element and sample exactly as the aligned copy."""
    gen = torch.Generator().manual_seed(9)
    B, V = 16, 16384
    x = torch.randn(2 * B, V, generator=gen) * 2.7
    buf = torch.zeros(2 * B * V + 4, device=DEV)
    res = []
    for off in (0, 1, 2, 3):
        buf.zero_()
        buf[off:off + 2 * B * V] = x.reshape(-1).to(DEV)
        dbg = torch.zeros(1, B, V, device=DEV)
        idx, pr, path, vec = sample_call(buf[off:off + 2 * B * V], B, V, mix=True, rd="bf16", cfg_scale=4.0, top_k=500, seed=3,
                                         step=0, dbg=dbg)
        assert vec == (1 if off == 0 else 0)
        res.append((idx, pr, dbg.cpu()))
    for r in res[1:]:
        assert np.array_equal(r[0], res[0][0]) and np.array_equal(r[1], res[0][1]) and torch.equal(r[2], res[0][2])


@pytest.mark.gpu
def test_vocab_past_the_shared_memory_stage_is_rejected():
    from llamagen_b200 import _lib
    x = torch.zeros(51201, device=DEV)
    with pytest.raises(_lib.LgError, match="vocab 51201 too large for the shared-memory row stage"):
        sample_call(x, 1, 51201)


# ------------------------------------------------------------------------------------------------ fused tail
@pytest.mark.gpu
@pytest.mark.parametrize("rd", ["bf16", "f16"])
@pytest.mark.parametrize("B,D,teach", [(1, 1024, False), (7, 1026, True), (300, 2304, False), (64, 1024, True)])
def test_fused_tail(rd, B, D, teach):
    """emb_h rows b and B + b take table[next] bit for bit (next = the pick, or the teacher's token); emb_xn is
    round16(round16(x r) g) with r = 1 / sqrt(mean(x^2) + eps) within the fp32 error of the kernel's r; the counters move by one and the
    ticket returns to zero (lg_test_sample checks it)."""
    gen = torch.Generator().manual_seed(B * 7 + D)
    V, eps, S = 4096, 1e-5, 6
    dt = TDT[rd]
    x = (torch.randn(2 * B, V, generator=gen) * 2.7).to(DEV)
    table = (torch.randn(V, D, generator=gen) * 0.5).to(dt).to(DEV)
    table[17] = 0   # an all-zero row: r = 1 / sqrt(eps)
    norm_w = (1 + 0.3 * torch.randn(D, generator=gen)).to(dt).to(DEV)
    R = 2 * B
    h = torch.full((R + 3, D), 9.0, dtype=dt, device=DEV)
    xn = torch.full((R + 3, D), 9.0, dtype=dt, device=DEV)
    pos = torch.tensor([41], dtype=torch.int32, device=DEV)
    stp = torch.tensor([4], dtype=torch.int32, device=DEV)
    teacher = torch.randint(0, V, (B, S), generator=gen, dtype=torch.int32)
    teacher[0, 4] = 17
    teacher = teacher.to(DEV)
    nxt = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    emb = dict(table=table, h=h, xn=xn, norm_w=norm_w, eps=eps, D=D, rows=R)
    idx, _, _, _ = sample_call(x, B, V, mix=True, rd=rd, cfg_scale=4.0, top_k=100, seed=11, step=4, teacher=teacher if teach else None,
                               seq_stride=S, next_tokens=nxt, emb=emb, adv=(pos, stp), probs=False, path=False)
    assert pos.item() == 42 and stp.item() == 5
    want = teacher[:, 4].cpu().numpy() if teach else idx
    assert np.array_equal(nxt.cpu().numpy(), want)
    tab, g = table.float().cpu().numpy(), norm_w.float().cpu().numpy()
    hh, xx = h.float().cpu().numpy(), xn.float().cpu().numpy()
    assert (hh[R:] == 9).all() and (xx[R:] == 9).all()
    exact = 0
    for b in range(B):
        t = tab[want[b]]
        r64 = 1.0 / math.sqrt(float(np.mean(t.astype(np.float64) ** 2)) + eps)
        # the kernel's r: an fp32 sum of D squares (D / 256 terms per thread, two 32-way trees), /D, +eps, sqrtf, 1/x
        er = (D / 256 + 16) * U24

        def out(r):
            return round16((round16((t * np.float32(r)).astype(np.float32), rd) * g).astype(np.float32), rd)
        lo, mid, hi = out(r64 * (1 - er)), out(r64), out(r64 * (1 + er))
        for row in (b, B + b):
            assert np.array_equal(hh[row], t), (b, row)
            v = xx[row]
            assert ((v >= np.minimum(lo, hi)) & (v <= np.maximum(lo, hi))).all(), (b, row)
            exact += int((v == mid).sum())
    assert exact >= 0.999 * 2 * B * D, exact


@pytest.mark.gpu
def test_fused_tail_rejects_fp32_rounding():
    from llamagen_b200 import _lib
    V, D = 1000, 64
    x = torch.zeros(2, V, device=DEV)
    t = torch.zeros(V, D, dtype=torch.bfloat16, device=DEV)
    h = torch.zeros(2, D, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_lib.LgError, match="16-bit round dtype"):
        sample_call(x, 1, V, mix=True, rd="f32", emb=dict(table=t, h=h, D=D, rows=2))


# ------------------------------------------------------------------------------------------------ the draw, draw by draw
@pytest.mark.gpu
def test_draw_sweep_every_pick_in_its_interval():
    """4096 fixed rows x 1200 steps (about 4.9 million draws): every pick's float64 CDF interval, from the kernel's own out_probs,
    holds its uniform within DRAW_BAND, and every draw is claimed by a segment (ending 1) unless u is within the band of 1. The fp32
    segment prefixes have gaps and overlaps at a few per million of the mass; a target in a gap must still go to a neighbouring
    segment, never to an unrelated token."""
    B, V, steps, seed = 4096, 16384, 1200, 20240917
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(B, V, generator=gen) * 2.7).to(DEV)
    _, probs, _, _ = sample_call(x, B, V, seed=seed, step=0)
    C = torch.from_numpy(probs).to(DEV).double().cumsum(1)
    C = C / C[:, -1:]
    seq = torch.full((B, steps), -1, dtype=torch.int32, device=DEV)
    ends = torch.empty(steps, B, dtype=torch.int32, device=DEV)
    from llamagen_b200 import _lib
    lib = _lib.load()
    sc = _lib.SampleCfg(1.0, -1, 1.0, 0, 1.0, 0, seed)
    pa = torch.empty(B, 3, dtype=torch.int32, device=DEV)
    st = _lib.current_stream(DEV)
    for j in range(steps):
        _lib.check(lib.lg_test_sample(P(x), B, V, 0, 0, ctypes.byref(sc), j, None, 0, None, None, None, None, P(seq), steps, None,
                                      None, None, 0, None, None, None, None, ctypes.c_float(0), 0, 0, None, None, P(pa), None, st),
                   "lg_test_sample")
        ends[j] = pa[:, 2]
    u = torch.from_numpy(u_draw_np(seed, np.arange(steps)[None, :], np.arange(1, B + 1)[:, None])).to(DEV)   # [B][steps]
    pick = seq.long()
    assert (pick >= 0).all()
    hi = C.gather(1, pick)
    lo = torch.where(pick > 0, C.gather(1, (pick - 1).clamp(min=0)), torch.zeros_like(hi))
    band = DRAW_BAND(V)
    bad = (u < lo - band) | (u > hi + band)
    ref = torch.searchsorted(C, u.contiguous(), right=True).clamp(max=V - 1)
    print(f"[sweep] {B * steps} draws, {int(bad.sum())} outside their interval, {int((ref != pick).sum())} differ from the float64 "
          f"inverse CDF, endings {torch.bincount(ends.flatten().long(), minlength=3).tolist()}")
    assert int(bad.sum()) == 0, [(int(b), int(s)) for b, s in bad.nonzero()[:10].tolist()]
    assert (torch.from_numpy(probs).to(DEV).gather(1, pick) > 0).all()
    e2 = ends.t() == 2
    assert ((ends.t() == 1) | (e2 & (u >= 1 - band))).all()


# ------------------------------------------------------------------------------------------------ score head
def score_call(partial, ks, Pn, V, nh, cfg, rd, targets):
    from llamagen_b200 import _lib
    lib = _lib.load()
    logits = torch.full((Pn, V), 3.0, device=DEV)
    nll = torch.full((Pn,), 3.0, device=DEV)
    _lib.check(lib.lg_test_score_head(P(partial), ks, Pn, V, nh, ctypes.c_float(cfg), RD[rd], P(targets), P(logits), P(nll),
                                      _lib.current_stream(DEV)), "lg_test_score_head")
    torch.cuda.synchronize()
    return logits.cpu().numpy(), nll.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("ks", [1, 3])
@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("V", [1000, 16383, 16384])
@pytest.mark.parametrize("nh", [1, 2])
def test_score_head(ks, rd, V, nh):
    """logits bit-equal to the fp32 restatement (slabs summed in slab order, rounded to the dtype, CFG-mixed); nll within
    NLL_BOUND of the float64 logsumexp(logits) - logits[target] of those logits: the online sum rescales each thread's fp32 sum at most
    once per element (3 roundings plus expf's 2 ulp), 512 threads merge in two 32-way trees, logf adds 1 ulp, so the sum is within
    (3 ceil(V / 512) + 16) 2^-24 relative; the final M + log(total) - logit is three fp32 roundings of numbers up to |M| + |logit|.
    A target of -1 or V gives NaN."""
    Pn, cfg = 9, 4.0
    gen = torch.Generator().manual_seed(ks * 100 + V + nh)
    part = torch.randn(ks, Pn * nh, V, generator=gen) * 2.0
    part[:, 0, :7] += 1e4                            # large magnitude: the online rescale
    part[:, nh * 1, 100:110] -= 1e4
    part[0, nh * 2, ::3] = -np.inf                   # -inf in cond rows only (the mix of two -inf is NaN)
    part[0, nh * 3, 1:] = -np.inf                    # one finite logit
    part = part.contiguous()
    targets = torch.randint(0, V, (Pn,), generator=gen, dtype=torch.int32)
    targets[2], targets[3] = 1, 0                    # row 2: a finite target logit
    targets[5], targets[6] = -1, V
    logits, nll = score_call(part.to(DEV), ks, Pn, V, nh, cfg, rd, targets.to(DEV))
    pn = part.numpy()
    for p in range(Pn):
        def head(row):
            s = pn[0, row].copy()
            for k in range(1, ks):
                s = (s + pn[k, row]).astype(np.float32)
            return round16(s, rd)
        want = restate_row(head(p * nh), head(p * nh + 1) if nh == 2 else None, nh == 2, cfg, "f32")
        assert np.array_equal(logits[p].view(np.int32), want.view(np.int32)), p
        tg = int(targets[p])
        if not 0 <= tg < V:
            assert np.isnan(nll[p]), p
            continue
        l64 = logits[p].astype(np.float64)
        M = l64.max()
        lse = M + math.log(np.exp(l64 - M).sum())
        ref = lse - l64[tg]
        bound = (3 * math.ceil(V / 512) + 16) * U24 + 3 * (abs(M) + abs(lse) + abs(l64[tg])) * U24
        assert abs(float(nll[p]) - ref) <= bound, (p, float(nll[p]), ref, bound)


@pytest.mark.gpu
def test_score_head_rejects_bad_arguments():
    from llamagen_b200 import _lib
    lib = _lib.load()
    part = torch.zeros(1, 2, 16, device=DEV)
    nll = torch.zeros(2, device=DEV)
    assert lib.lg_test_score_head(P(part), 1, 2, 16, 1, ctypes.c_float(1), 1, None, None, P(nll), _lib.current_stream(DEV)) < 0
    assert b"needs targets" in lib.lg_last_error()
    assert lib.lg_test_score_head(P(part), 1, 1, 16, 3, ctypes.c_float(1), 1, None, P(part), None, _lib.current_stream(DEV)) < 0
    assert b"bad shape" in lib.lg_last_error()
