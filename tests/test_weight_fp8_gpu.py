"""GPU: fp8 (e4m3) GEMM weights (`Transformer.set_weight_dtype("fp8")`, the samplers' --weight-dtype fp8) through the register-A wgmma
GEMM, the small-row GEMV and the row quantiser.

One call at a time (lg_test_linear_w8), with the checks of tests/test_linear_gpu.py: the float64 reference is built from the operands
as the kernels read them (x in the model dtype, the integer codes, the scales), so the accumulator bound is the 16-bit one,
|acc - ref| <= 2^-16 s_n (|x| |code|^T): widening a code is exact and the scale is a power of two. End to end, the protocol of
tests/test_kv_fp8_gpu.py: the unmodified oracle on the dequantised weights code * s has exactly the engine's semantics, in fp32 (ref32)
and in the model dtype (ref16); the engine, teacher-forced on ref32's greedy stream, stays within 1.5 x |ref16 - ref32| plus the
dtype's floor."""
import ctypes
import math

import pytest
import torch

import test_linear_gpu as tl
import weight_fp8_oracle as wo
from oracle import GPTOracle
from util import build_gpt, cpu_state, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

FLOORS = {torch.bfloat16: (0.02, 0.005), torch.float16: (0.0025, 0.000625)}


# --------------------------------------------------------------------------------------------------- quantiser
def quantize_gpu(w):
    from llamagen_b200 import _lib
    lib = _lib.load()
    N, K = w.shape
    codes = torch.empty(N, K, dtype=torch.uint8, device="cuda")
    scales = torch.empty(N, dtype=torch.float32, device="cuda")
    _lib.check(lib.lg_quantize_rows_e4m3(_lib.ptr(w), N, K, _lib.dtype_code(w.dtype), _lib.ptr(codes), _lib.ptr(scales),
                                         _lib.current_stream(w.device)), "lg_quantize_rows_e4m3")
    torch.cuda.synchronize()
    return codes[:, _lib.weight_fp8_stored_index(K).cuda()].cpu(), scales.cpu()


def _quantiser_inputs(dtype):
    g = torch.Generator().manual_seed(11)
    N, K = 96, 1024
    lo, hi = wo.EXPONENTS[dtype]
    normal = torch.randn(N, K, generator=g) * 0.02
    heavy = torch.randn(N, K, generator=g) * 0.02 * torch.exp(2.0 * torch.randn(N, K, generator=g))
    zero_rows = normal.clone()
    zero_rows[::7] = 0
    zero_rows[3, 5:] = 0                                                     # one nonzero element
    top = 2.0 ** (14 if dtype == torch.float16 else 100)
    wide = torch.randn(N, K, generator=g) * torch.logspace(-6, math.log10(top), N)[:, None]     # rows over the whole range, no inf
    wide = wide.clamp(-60000.0, 60000.0) if dtype == torch.float16 else wide
    tiny = torch.randn(N, K, generator=g) * 2.0 ** (lo - 4)                  # below the exponent clamp, fp16 subnormals
    edges = torch.full((N, K), 0.001)
    edges[:, 0] = torch.tensor([448.0, 224.0, 224.5, 447.0, 449.0, 1.75, 0.875, 28.0] * (N // 8))   # absmax on and around binade edges
    return {"normal": normal, "heavy_tail": heavy, "zero_rows": zero_rows, "wide_range": wide, "tiny": tiny, "binade_edges": edges}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantiser_is_bit_equal_to_the_oracle(dtype):
    for name, w in _quantiser_inputs(dtype).items():
        w = w.to(dtype)
        assert torch.isfinite(w.float()).all(), name
        codes, scales = quantize_gpu(w.cuda().contiguous())
        want_c, want_s = wo.quantize_rows(w, dtype)
        assert torch.equal(scales, want_s), (name, (scales != want_s).nonzero()[:4])
        assert torch.equal(codes, want_c), (name, (codes != want_c).nonzero()[:4])
        if name == "normal":
            scaled = w.float().abs().amax(1) / scales
            assert ((scaled > 224) & (scaled <= 448)).all()
        assert torch.equal(wo.dequantize(codes, scales, dtype).float(), wo.code_values(codes) * scales[:, None]), name


def test_quantiser_refuses_bad_arguments():
    from llamagen_b200 import _lib
    lib = _lib.load()
    w = torch.zeros(8, 96, dtype=torch.bfloat16, device="cuda")
    c = torch.zeros(8, 96, dtype=torch.uint8, device="cuda")
    s = torch.zeros(8, dtype=torch.float32, device="cuda")
    st = _lib.current_stream(w.device)
    assert lib.lg_quantize_rows_e4m3(_lib.ptr(w), 8, 96, 1, _lib.ptr(c), _lib.ptr(s), st) < 0
    assert "multiple of 64" in lib.lg_last_error().decode()
    assert lib.lg_quantize_rows_e4m3(_lib.ptr(w), 8, 64, 0, _lib.ptr(c), _lib.ptr(s), st) < 0
    assert "bf16 or fp16" in lib.lg_last_error().decode()


# --------------------------------------------------------------------------------------------------- one call at a time
def run_linear_w8(dt, x, ca, sa, cb, sb, epi, small, norm_in=None, norm_out=None, h=None, eps=tl.EPS, check=True):
    """lg_test_linear_w8 on codes given with column k at index k. Returns ({"h" / "out": output}, acc_out or None, path), or the
    status and message with check=False."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    M, K = x.shape
    N = ca.shape[0]
    dev = x.device
    idx = _lib.weight_fp8_stored_index(K // 64 * 64).to(dev)

    def pack(c):
        if c is None or K % 64:            # K % 64 != 0 has no stored order: the call is refused before it reads a code
            return c
        s = torch.empty_like(c)
        s[:, idx] = c
        return s.contiguous()

    pa, pb = pack(ca), pack(cb)
    NN = 2 * N if cb is not None else N
    out_f32 = torch.empty(M, N, dtype=torch.float32, device=dev) if epi == 0 else None
    out = torch.empty(M, N, dtype=tl.TDT[dt], device=dev) if (epi >= 2 or norm_out is not None) else None
    hh = h.clone() if epi == 1 else None
    acc = None if small else torch.empty(M, NN, dtype=torch.float32, device=dev)
    nbytes = 0 if small else 16 * M * NN * 4 + 256 + (M * K * 4 if norm_in is not None else 0)
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    path = (ctypes.c_int * 4)(-9, -9, -9, -9)
    P = _lib.ptr
    rc = lib.lg_test_linear_w8(tl.LG_DT[dt], M, N, K, P(x), P(norm_in), ctypes.c_float(eps), P(pa), P(sa), P(pb), P(sb), epi, P(norm_out),
                               P(hh), P(out), P(out_f32), P(acc), int(small), P(scratch) if nbytes else None, ctypes.c_size_t(nbytes),
                               path, _lib.current_stream(dev))
    if not check:
        return rc, lib.lg_last_error().decode()
    _lib.check(rc, "lg_test_linear_w8")
    torch.cuda.synchronize()
    got = {}
    if epi == 0:
        got["out"] = out_f32
    if epi == 1:
        got["h"] = hh
    if out is not None:
        got["out"] = out
    return got, acc, tuple(path)


def C(cid, dt, M, N, K, **kw):
    return tl.Case(cid, dt, M, N, K, **kw)


CASES = [
    # gemm_tc_kernel with A from registers: every row pad x every epilogue x both dtypes, norm prologue, row blocks, ksplit 1 .. 16
    C("tc_bf16_pad16_m2_f32", "bf16", 2, 384, 1024, want=(2, 16)),
    C("tc_f16_pad16_m9_residual", "f16", 9, 256, 512, epi=1, want=(2, 16)),
    C("tc_bf16_pad16_norm_in", "bf16", 16, 256, 1024, norm_in=True, want=(2, 16)),
    C("tc_f16_pad32_store", "f16", 32, 128, 768, epi=3, want=(2, 32)),
    C("tc_bf16_pad32_gelu", "bf16", 20, 256, 512, epi=4, want=(2, 32)),
    C("tc_f16_pad64_gelu", "f16", 40, 512, 1024, epi=4, want=(2, 64)),
    C("tc_f16_pad64_f32", "f16", 64, 512, 128, want=(2, 64, 1)),
    C("tc_f16_pad128_residual_norm", "f16", 100, 256, 2048, epi=1, norm_out=True, want=(2, 128)),
    C("tc_bf16_pad128_store", "bf16", 128, 384, 512, epi=3, want=(2, 128)),
    C("tc_bf16_pad256_store", "bf16", 256, 384, 512, epi=3, want=(2, 256, 4, 1)),
    C("tc_f16_pad256_residual", "f16", 200, 256, 512, epi=1, want=(2, 256)),
    C("tc_bf16_m257_residual_norm", "bf16", 257, 256, 512, epi=1, norm_out=True, want=(2, 256, 4, 2)),
    C("tc_bf16_m1920_gelu", "bf16", 1920, 256, 512, epi=4, want=(2, 256, 4, 8)),
    C("tc_bf16_ks16", "bf16", 16, 256, 4096, want=(2, 16, 16)),
    C("tc_f16_ks16_short_tail", "f16", 24, 256, 2816, epi=3, want=(2, 32, 16)),       # 44 k-blocks by 3: short, then empty slice
    C("tc_bf16_odd_kblocks", "bf16", 12, 256, 1088, epi=3, want=(2, 16, 8)),          # 17 k-blocks by 3: a slice of 3 and one of 2
    C("pair_tc_bf16_f256_norm_in", "bf16", 16, 256, 512, epi=2, norm_in=True, want=(2, 16)),
    C("pair_tc_f16_f384_m300", "f16", 300, 384, 256, epi=2, want=(2, 256)),
    C("pair_tc_bf16_f128_m64", "bf16", 64, 128, 1024, epi=2, want=(2, 64)),
    # gemv_small_kernel: every R, each instantiation, chunk counts below PF and off the 8 warps
    *[C(f"small_r{R}_{tl.EPI_NAMES[(0, 1, 2)[R % 3]]}", "bf16" if R % 2 else "f16", R, 256, 512, epi=(0, 1, 2)[R % 3], small=True,
        norm_in=R % 2 == 0) for R in range(1, 9)],
    C("small_rows8_n2048_k256", "bf16", 2, 2048, 256, small=True, norm_in=True, want=(3, 8, 1, 12)),
    C("small_rows16_n4096", "f16", 3, 4096, 512, epi=1, small=True, want=(3, 16, 1, 4)),
    C("small_rows32_n16384", "bf16", 2, 16384, 256, small=True, norm_in=True, want=(3, 32, 1, 4)),
    C("small_paired_r8_k1280", "f16", 8, 512, 1280, epi=2, small=True, norm_in=True, want=(3, 32, 1, 4)),
    C("small_k320", "bf16", 3, 512, 320, epi=1, small=True),                          # 5 chunks of 64: three warps idle
    C("small_r5_k8704", "bf16", 5, 3200, 8704, epi=1, small=True),                    # GPT-3B w2
]
REGISTRY = ("GPT-B", "GPT-L", "GPT-3B")
for _n in REGISTRY:
    for _c in tl.layer_cases(_n, 2, True) + tl.layer_cases(_n, 128, False):
        CASES.append(_c)
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES)


def test_cases_cover_every_fp8_path():
    assert {c.expect[:2] for c in CASES} == {(2, 16), (2, 32), (2, 64), (2, 128), (2, 256), (3, 8), (3, 16), (3, 32)}
    assert {(c.dt, c.epi) for c in CASES if not c.small} >= {(d, e) for d in ("bf16", "f16") for e in range(5)}
    assert {c.M for c in CASES if c.small} >= set(range(1, 9))
    assert {1, 16} <= {c.expect[2] for c in CASES if c.expect[0] == 2}


def fp8_operands(c, seed):
    """tl.operands with the weights quantised: rows of one 128-row tile get scales up to 2^4 apart (scaled down only: outputs far in
    gelu's negative tail would measure tanhf's cancellation, not the GEMM), rows 0 / 1 of an fp32-output
    case sit at the two ends of the allowed exponent range, and the last column of three rows holds the largest code (a needle in
    the last k of the last k-slice)."""
    x, wa, wb, nin, h, nout = tl.operands(c, seed)
    dtype = tl.TDT[c.dt]

    def quant(w):
        n = torch.arange(w.shape[0], device=w.device)
        w = (w.float() * torch.ldexp(torch.ones_like(n, dtype=torch.float32), (n * 7) % 5 - 4)[:, None]).to(dtype)
        codes, s = wo.quantize_rows(w.cpu(), dtype)
        codes, s = codes.cuda(), s.cuda()
        for r, v in ((0, 0x7E), (w.shape[0] // 2 + 9, 0xFE), (w.shape[0] - 1, 0x7E)):
            codes[r, -1] = v
        if c.epi == 0:
            lo, hi = wo.EXPONENTS[dtype]
            s[0], s[1] = 2.0 ** lo, 2.0 ** hi
        return codes.contiguous(), s.contiguous()

    ca, sa = quant(wa)
    cb, sb = quant(wb) if wb is not None else (None, None)
    return x, ca, sa, cb, sb, nin, h, nout


def effective_weight(ca, sa, cb, sb):
    w = wo.code_values(ca.cpu()).double() * sa.cpu().double()[:, None]
    if cb is not None:
        w = torch.cat([w, wo.code_values(cb.cpu()).double() * sb.cpu().double()[:, None]])
    return w.cuda()


def check_case(c, got, acc, x, w, nin, h, nout):
    """Checks 1-3 of test_linear_gpu.run_case against the float64 weight w = code * s."""
    ref, E, xps = tl.reference(c, x, w, nin)
    for name, a in (("acc_out", acc), ("out_f32", got.get("out") if c.epi == 0 else None)):
        if a is not None:
            bad = (a.double() - ref).abs() > E
            assert not bad.any(), f"{c.id} {name}: {int(bad.sum())} of {bad.numel()} beyond E, worst " \
                                  f"{((a.double() - ref).abs() / E).max().item():.2f} E"
    if acc is not None:
        if c.epi == 0:
            assert torch.equal(got["out"], acc), f"{c.id}: out_f32 differs from the same slabs summed into acc_out"
        else:
            p = tl.restated_problem(c.dt, got, tl.restate(c.dt, c.epi, acc, h=h, norm_out=nout), c.epi, acc)
            assert p is None, f"{c.id}: {p}"
    ch = tl.chain64(c.dt, c.epi, ref, E, h=h, norm_out=nout)
    skip = None
    if len(xps) > 1:
        alts = [tl.chain64(c.dt, c.epi, xa @ w.t(), E, h=h, norm_out=nout) for xa in xps[1:]]
        skip = {k: (alts[0][k][0] != ch[k][0]) | (alts[1][k][0] != ch[k][0]) for k in ch}
    cap_frac = tl.cap(c.dt, c.K, 2 if c.epi == 2 else 1) if c.epi != 0 else None
    p = tl.chain_problem(got, ch, cap_frac, skip)
    assert p is None, f"{c.id}: {p}"


@pytest.mark.parametrize("cid", list(CASE_BY_ID))
def test_linear_layer_w8(cid, monkeypatch):
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    c = CASE_BY_ID[cid]
    x, ca, sa, cb, sb, nin, h, nout = fp8_operands(c, 1)
    got, acc, path = run_linear_w8(c.dt, x, ca, sa, cb, sb, c.epi, c.small, norm_in=nin, norm_out=nout, h=h)
    assert path == c.expect, f"{c.id}: ran {path}, expected {c.expect}"
    check_case(c, got, acc, x, effective_weight(ca, sa, cb, sb), nin, h, nout)


@pytest.mark.parametrize("R,N,K,epi", [(2, 768, 768, 0), (8, 512, 1024, 1), (5, 256, 512, 2), (1, 16384, 1024, 0)])
def test_small_and_batched_kernels_agree(R, N, K, epi):
    """The same R <= 8 call on gemv_small_kernel and on gemm_tc_kernel: fp32 results within fp32 reordering (2 x the accumulator
    bound apart), 16-bit results within one ulp."""
    c = C("agree", "bf16", R, N, K, epi=epi)
    x, ca, sa, cb, sb, nin, h, nout = fp8_operands(c, 2)
    small, _, ps = run_linear_w8("bf16", x, ca, sa, cb, sb, epi, True, h=h)
    batched, _, pb = run_linear_w8("bf16", x, ca, sa, cb, sb, epi, False, h=h)
    assert ps[0] == 3 and pb[0] == 2
    w = effective_weight(ca, sa, cb, sb)
    E = tl.E_REL * (x.double().abs() @ w.abs().t())
    for k in small:
        a, b = small[k].double(), batched[k].double()
        if epi == 0:
            assert ((a - b).abs() <= 2 * E).all()
        else:
            assert ((a - b).abs() <= tl.ulp(torch.maximum(a.abs(), b.abs()), "bf16")).all()
            assert (a == b).double().mean().item() >= 0.98


def test_bad_scales_and_shapes_are_errors_before_any_launch():
    c = C("err", "f16", 4, 256, 512)
    x, ca, sa, _, _, _, _, _ = fp8_operands(c, 3)
    for bad, what in ((3.0, "powers of two"), (2.0 ** 8, "powers of two"), (2.0 ** -16, "powers of two"), (0.0, "powers of two"),
                      (float("nan"), "powers of two")):
        s = sa.clone()
        s[17] = bad
        rc, err = run_linear_w8("f16", x, ca, s, None, None, 0, False, check=False)
        assert rc < 0 and what in err and "row 17" in err, (bad, err)
    rc, err = run_linear_w8("f16", x[:, :480].contiguous(), ca[:, :480].contiguous(), sa, None, None, 0, False, check=False)
    assert rc < 0 and "multiple of 64" in err, err
    rc, err = run_linear_w8("f16", x[:, :480].contiguous(), ca[:, :480].contiguous(), sa, None, None, 0, True, check=False)
    assert rc < 0 and "multiple of 64" in err, err
    rc, err = run_linear_w8("f16", x, ca[:200].contiguous(), sa[:200].contiguous(), None, None, 0, False, check=False)
    assert rc < 0 and "128-row tiles" in err, err
    torch.cuda.synchronize()


# --------------------------------------------------------------------------------------------------- end to end
def _gen(model, cond, S, em, **kw):
    from llamagen_b200 import generate
    toks, logits = generate(model, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), sample_logits=False,
                            return_logits=True, **kw)
    torch.cuda.synchronize()
    return toks.cpu(), logits.cpu()


def _w8_parity(m, cond, S, em=None, head=True, kv_fp8=False, report=None):
    """The engine with fp8 weights, teacher-forced on ref32's greedy stream, against the oracles on the dequantised weights."""
    cfg = oracle_cfg(m)
    dt = m.tok_embeddings.weight.dtype
    sd = cpu_state(m)
    cond32 = cond if cond.dtype == torch.long else cond.float()
    if kv_fp8:
        from kv_fp8_oracle import KvFp8Oracle as Oracle
    else:
        Oracle = GPTOracle
    ref_t, ref_l = Oracle(wo.dequantized_state_dict(sd, dt, head, torch.float32), cfg).generate(cond32, S, emb_masks=em, cfg_scale=4.0,
                                                                                             sample_logits=False)
    _, h_l = Oracle(wo.dequantized_state_dict(sd, dt, head), cfg).generate(cond, S, emb_masks=em, cfg_scale=4.0, sample_logits=False,
                                                                           teacher=ref_t)
    fmax, fmean = FLOORS[dt]
    tol_max = 1.5 * (h_l - ref_l).abs().max().item() + fmax
    tol_mean = 1.5 * (h_l - ref_l).abs().mean().item() + fmean
    m.set_weight_dtype("fp8", head=head)
    m.set_kv_cache("fp8" if kv_fp8 else "auto")
    toks, logits = _gen(m, cond, S, em, cfg_scale=4.0, teacher=ref_t.clone())
    for name in m.fp8_weight_names()[:3] + m.fp8_weight_names()[-1:]:       # what was bound is what the oracle dequantised
        wc, ws = wo.quantize_rows(sd[name], dt)
        assert torch.equal(m.weight_codes(name).cpu(), wc) and torch.equal(m.weight_scales(name).cpu(), ws), name
    assert ("output.weight" in m.fp8_weight_names()) == head
    for other in (ref_l, h_l):
        err = (logits - other).abs()
        assert err.max().item() <= tol_max, (err.max().item(), tol_max)
        assert err.mean().item() <= tol_mean, (err.mean().item(), tol_mean)
    decisive = top2_gap(ref_l) > 2 * tol_max
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    assert torch.equal(toks.t()[decisive], ref_t.t()[decisive])
    if report is not None:
        # the cost of the quantisation itself, on these random weights only: fp8-weight logits against the UNQUANTISED fp32 oracle
        _, plain = GPTOracle(cpu_state(m, torch.float32), cfg).generate(cond32, S, emb_masks=em, cfg_scale=4.0, sample_logits=False,
                                                                        teacher=ref_t)
        q = (logits - plain).abs()
        print(f"\n[{report}] fp8-weight logits vs unquantised fp32 oracle: max {q.max().item():.4f} mean {q.mean().item():.5f} "
              f"(logit std {plain.std().item():.3f}); engine vs its own oracle: max {(logits - ref_l).abs().max().item():.4f}")
        assert q.max().item() <= 0.5 * plain.abs().max().item() + 1.0       # a loose sanity cap, not a quality claim
    return logits


@pytest.mark.parametrize("kv_fp8", [False, True])
@pytest.mark.parametrize("head", [True, False])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_tiny_goldens_teacher_forced(name, dtype, head, kv_fp8):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], dtype)
    cond = g["cond"] if name == "gpt_c2i.pt" else g["cond"].to(dtype)
    _w8_parity(m, cond, g["S"], g["emb_masks"], head=head, kv_fp8=kv_fp8, report=f"{name} {dtype} head={head}" if not kv_fp8 else None)


def _seeded(dtype, seed, **kw):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(seed)
    m = Transformer(ModelArgs(**kw))
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dtype).eval()


@pytest.mark.parametrize("B", [1, 9])
def test_head_dim_128_model(B):
    """hd 128; B = 1 runs the small-row path, B = 9 the batched one."""
    m = _seeded(torch.bfloat16, 5, n_layer=2, n_head=4, dim=512, block_size=64, vocab_size=2048)
    _w8_parity(m, torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(B)), 6, report=f"hd128 B={B}")


def test_gpt_3b_shaped_layer_head_dim_100():
    m = _seeded(torch.bfloat16, 3, n_layer=1, n_head=32, dim=3200, block_size=64, vocab_size=16384)
    _w8_parity(m, torch.tensor([1, 2, 3]), 5, report="GPT-3B layer")


def test_gpt_l_batch_1_and_40_fp16():
    m = _seeded(torch.float16, 1, n_layer=4, n_head=16, dim=1024, block_size=256, vocab_size=16384)
    _w8_parity(m, torch.tensor([7]), 6)
    _w8_parity(m, torch.randint(0, 1000, (40,), generator=torch.Generator().manual_seed(4)), 6, kv_fp8=True)


def test_dim_not_a_multiple_of_128_is_a_planned_error():
    from llamagen_b200 import _lib
    m = _seeded(torch.bfloat16, 2, n_layer=1, n_head=3, dim=192, block_size=16, vocab_size=1024)
    m.set_weight_dtype("fp8")
    with pytest.raises(_lib.LgError, match="cannot be fp8.*128-row tiles"):
        m.engine()
    m.set_weight_dtype("auto")
    m.engine()
    m32 = _seeded(torch.float32, 2, n_layer=1, n_head=2, dim=128, block_size=16, vocab_size=1024)
    m32.set_weight_dtype("fp8")
    with pytest.raises(_lib.LgError, match="bf16 or fp16"):
        m32.engine()


def _gpt_b(dtype=torch.bfloat16, block_size=64):
    from llamagen_b200 import GPT_models
    torch.manual_seed(0)
    m = GPT_models["GPT-B"](vocab_size=16384, block_size=block_size, num_classes=1000, cls_token_num=1, model_type="c2i")
    m = m.to("cuda", dtype).eval()
    m.output.weight.data.normal_(std=0.02)
    return m


def test_generate_is_reproducible_chains_agree_and_auto_restores(monkeypatch):
    from llamagen_b200 import generate
    m = _gpt_b()
    cond = torch.randint(0, 1000, (32,), generator=torch.Generator().manual_seed(3)).cuda()
    kw = dict(cfg_scale=4.0, temperature=1.0, top_k=200, top_p=1.0, seed=9)
    base16 = generate(m, cond, 24, **kw).cpu()
    m.set_weight_dtype("fp8")
    runs = {}
    for split in ("1", "2"):
        monkeypatch.setenv("LG_SPLIT", split)
        m._drop_engine()
        runs[split] = [generate(m, cond, 24, **kw).cpu() for _ in range(2)]
        assert torch.equal(*runs[split]), split
    monkeypatch.delenv("LG_SPLIT")
    assert torch.equal(runs["1"][0], runs["2"][0])
    assert not torch.equal(runs["1"][0], base16)
    m.set_weight_dtype("auto")
    back = generate(m, cond, 24, **kw).cpu()
    assert torch.equal(back, base16), "a model switched back to auto does not reproduce its 16-bit tokens"


def test_load_state_dict_into_a_live_fp8_engine_requantises():
    """load_state_dict writes the parameters in place (same storage): the engine's codes must follow, as a 16-bit engine's borrowed
    tensors do. A write through .data needs requantize()."""
    from llamagen_b200 import generate
    cond = torch.tensor([1, 2, 3, 4], device="cuda")
    a, b = (_seeded(torch.bfloat16, s, n_layer=2, n_head=4, dim=256, block_size=64, vocab_size=1024) for s in (21, 22))
    for m in (a, b):
        m.set_weight_dtype("fp8")
    want_b = generate(b, cond, 16, cfg_scale=4.0, sample_logits=False).cpu()
    got_a = generate(a, cond, 16, cfg_scale=4.0, sample_logits=False).cpu()
    assert not torch.equal(got_a, want_b)
    ptrs = [t.data_ptr() for t in a.state_dict().values()]
    a.load_state_dict(b.state_dict())
    assert ptrs == [t.data_ptr() for t in a.state_dict().values()]
    assert torch.equal(generate(a, cond, 16, cfg_scale=4.0, sample_logits=False).cpu(), want_b)
    name = "layers.1.feed_forward.w2.weight"
    assert torch.equal(a.weight_codes(name), b.weight_codes(name)) and torch.equal(a.weight_scales(name), b.weight_scales(name))
    a.output.weight.data.mul_(-1.0)
    a.requantize()
    a.engine()
    assert torch.equal(wo.code_values(a.weight_codes("output.weight").cpu()), -wo.code_values(b.weight_codes("output.weight").cpu()))


def test_greedy_sjd_tokens_are_argmax_of_score():
    """The 16-bit protocol of tests/test_sjd_gpu.py with fp8 weights (exact equality with plain greedy holds for fp32 models only: the
    window pass rounds 16-bit activations in other places): every greedy sjd_window token is score()'s argmax at its position, or
    within 4 units in the last place of bf16 at that row's largest logit."""
    from llamagen_b200 import generate, score
    m = _seeded(torch.bfloat16, 6, n_layer=4, n_head=8, dim=512, block_size=64, vocab_size=2048)
    m.set_weight_dtype("fp8")
    cond = torch.tensor([3, 500, 77, 901], device="cuda")
    toks = generate(m, cond, 48, cfg_scale=4.0, sample_logits=False, sjd_window=8)
    _, logits = score(m, cond, toks.long(), cfg_scale=4.0, return_logits=True)
    picked = logits.gather(-1, toks.long()[..., None])[..., 0]
    top = logits.max(-1).values
    _, e = torch.frexp(top.abs())
    margin = 4 * torch.ldexp(torch.ones_like(top), e - 8)
    assert (top - picked <= margin).all(), ((top - picked).max().item(), margin.min().item())


def test_score_matches_the_oracle_on_dequantised_weights():
    """A model whose 16-bit parameters already are code * s (re-quantising them reproduces the same values) scores, with fp8
    weights, within the score tests' bounds of the oracles on its state dict."""
    from test_score_gpu import _parity_16
    m = _seeded(torch.bfloat16, 7, n_layer=2, n_head=4, dim=256, block_size=64, vocab_size=1024)
    deq = wo.dequantized_state_dict(cpu_state(m), torch.bfloat16)
    for k, v in wo.dequantized_state_dict(deq, torch.bfloat16).items():
        assert torch.equal(v, deq[k]), k
    m.load_state_dict(deq)
    m.set_weight_dtype("fp8")
    _parity_16(m, torch.randint(0, 1000, (16,)), torch.randint(0, 1024, (16, 64)), 4.0)
    assert len(m._w8) == 2 * 5 + 1


def test_serve_llm_fp8_weights_match_generate():
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    gpt = _gpt_b()
    S, slots = 64, 4
    sp = SamplingParams(temperature=1.0, top_p=1.0, top_k=2000, max_tokens=S)
    llm = LLM(gpt, cfg_scale=4.0, num_classes=1000, max_num_seqs=slots, seed=11, weight_dtype="fp8")
    assert gpt._weight_dtype == ("fp8", True)
    labels = [207, 360, 387]
    outs = []
    for c in labels:
        llm.add_request([c], sp)
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): o.outputs[0].token_ids for o in outs}
    for rid, c in enumerate(labels):
        ref = generate(gpt, torch.full((slots,), c, device="cuda"), S, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, seed=11 + rid)
        assert ref[0].cpu().tolist() == got[rid], rid


def test_sample_c2i_cli_weight_fp8(tmp_path, monkeypatch):
    from llamagen_b200.sample import sample_c2i
    monkeypatch.chdir(tmp_path)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--image-size", "256", "--cfg-scale", "4.0", "--top-k", "2000",
                                                 "--seed", "1", "--weight-dtype", "fp8", "--kv-cache-dtype", "fp8"])
    sample_c2i.main(args)
    from PIL import Image
    img = Image.open(tmp_path / "sample_c2i.png")
    assert img.size == (4 * 256 + 5 * 2, 2 * 256 + 3 * 2)
