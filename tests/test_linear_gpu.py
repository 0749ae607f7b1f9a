"""Every transformer GEMM, small-row GEMV and row-epilogue path, one linear layer at a time, against a float64 reference.

lg_test_linear runs one linear layer as the engine composes it and reports the path it took: {kernel, tile, ksplit, row blocks or
PF}, kernel 0 = gemm_skinny_kernel, 1 = gemm_mma_kernel, 2 = gemm_tc_kernel (wgmma), 3 = gemv_small_kernel. Every case asserts the
path it expects (plan_model below restates the documented dispatch; tests/test_linear_plan.py holds the library's plan to it without
a GPU). The references are plain torch float64 on the GPU, from the operands exactly as the kernels read them. T() is the model
dtype's round-to-nearest-even of an fp32 value.

Three checks, because a rigorous float64 interval alone is too wide on 16-bit outputs:
  1. GEMM accumulator. E = 2^-16 |x'| |w|^T, x' the activation the GEMM multiplies. Every fp32 result (out_f32, and acc_out: the
     split-K slabs summed in slab order, as the epilogue kernels sum them) satisfies |acc - ref64| <= E. fp32 accumulation of K
     exact products drifts by ~2^-24 sqrt(K) |acc|, far inside E; a bf16-rounded fp16 operand (2^-9 relative), a TF32 product on
     fp32 (2^-11), a missing k-block or a swapped w1 | w3 segment miss it by orders of magnitude.
     With an RMSNorm prologue, x' = T(T(x r) w) with r = rsqrt(mean(x^2) + eps) in fp32. r's relative error is at most
     ((K/32 + 16) / 2 + 2) 2^-24 (the longest serial fp32 sum of squares is K/32 long, on gemv_small at R = 8; then the tree, sqrt
     and division), below 2^-16 for every K here, so r is given a relative width of 2^-16; x' then lies in [x'lo, x'hi] and E
     widens by |x'hi - x'lo| |w|^T.
  2. Batched epilogues against the kernel's own accumulator: an fp32 torch restatement of residual_norm_kernel, silu_mul_kernel and
     store_act_kernel (identity / gelu-tanh), applied to acc_out, is bit-equal on >= 99.9 % of the outputs and within one ulp of T
     everywhere. Only expf / tanhf and the row's fp32 RMS reduction order may differ between device and restatement. An fp32
     model has no rounding to absorb those differences: its outputs behind them are held to 64 fp32 ulps instead.
  3. Whole chain against float64 (the small path too, whose accumulator is not observable). The chain is evaluated in float64 with
     T() at the kernel's rounding points, once at the point value and once over the interval that acc in [ref - E, ref + E]
     propagates: every T is monotone, silu and gelu take their min / max over the interval (widened by 2^-20 relative plus
     2^-21 |v| for the fp32 expf / tanhf evaluation), the next norm's r gets the 2^-16 width above. Every output lies in its
     interval. The fraction of outputs that differ from the point value stays under
         cap = max(0.5 %, 8 n 2^-24 sqrt(K) 2^p),   p = 8 (bf16) / 11 (fp16), n = 1, or 2 for SwiGLU (two accumulators):
     an accumulator off by d = 2^-24 sqrt(K) relative flips a rounding with probability ~2 d / ulp, ulp >= 2^-p relative, so the
     cap is >= 4x the expected rate (bf16 K = 4096: 0.8 %; fp16 K = 1280 SwiGLU: 7 %). Outputs whose point value changes when the
     prologue's fp32 r moves by 2^-22 are not counted (the kernel's r and the float64 one can straddle a rounding of x'). fp32
     models have no cap. A missing or extra rounding point moves 20-50 % of the outputs; test_linear_plan.py checks on the CPU that
     checks 2 and 3 reject four such chains.
"""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TDT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
LG_DT = {"f32": 0, "bf16": 1, "f16": 2}
P_BITS = {"f32": 24, "bf16": 8, "f16": 11}
MIN_ULP = {"f32": 2.0 ** -149, "bf16": 2.0 ** -133, "f16": 2.0 ** -24}
EPS = 1e-5
E_REL = 2.0 ** -16           # check 1
DR = 2.0 ** -16              # relative width of an RMSNorm's r
FN_REL, FN_ABS = 2.0 ** -20, 2.0 ** -21
SILU_MIN_AT, GELU_MIN_AT = -1.2784645427610738, -0.7517915246935732
EPI_NAMES = {0: "f32", 1: "residual", 2: "swiglu", 3: "store", 4: "gelu"}


def cdiv(a, b):
    return -(-a // b)


# --------------------------------------------------------------------------------------------------- the documented dispatch
def plan_model(dt, M, N, K, paired, small, tc=True):
    """(kernel, tile, ksplit, row blocks or PF) that gemm_plan / gemv_small_plan document for a valid call."""
    if small:
        if paired:
            return (3, 32, 1, 4)
        return (3, 8, 1, 12) if N <= 2048 else (3, 16 if N <= 8192 else 32, 1, 4)
    NN, ns = (2 * N, N) if paired else (N, 0)
    if tc and dt != "f32" and NN % 128 == 0 and ns % 128 == 0:
        rblk = min(M, 256)
        pad = 16
        while pad < rblk:
            pad *= 2
        tiles = cdiv(NN, 128) * cdiv(M, 256)
        ks = min(max(1, 92 // tiles), max(1, cdiv(K, 64) // 2), 16)
        return (2, pad, ks, cdiv(M, rblk))
    if dt == "f32" or M <= 8:
        ctas = cdiv(NN, 16) * cdiv(M, 8)
        return (0, 8, min(max(1, 264 // ctas), max(1, K // 512), 16), cdiv(M, 8))
    bm = 32 if M <= 32 else (64 if M <= 64 else 128)
    ks = min(max(1, 132 // (cdiv(M, bm) * cdiv(NN, 128))), max(1, (K // 64) // 4), 16)
    return (1, bm, ks, cdiv(M, bm))


# --------------------------------------------------------------------------------------------------- rounding helpers
def rnd(v, dt):
    """T(): fp32 rounding first (a float64 value becomes the fp32 value the kernel would hold), then the model dtype."""
    return v.to(torch.float32).to(TDT[dt]).to(v.dtype)


def ulp(v, dt):
    _, e = torch.frexp(v.double().abs())
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - P_BITS[dt]).clamp_min(MIN_ULP[dt])


def cap(dt, K, n=1):
    return None if dt == "f32" else max(0.005, 8 * n * 2.0 ** -24 * math.sqrt(K) * 2.0 ** P_BITS[dt])


def silu64(v):
    return v / (1.0 + torch.exp(-v))


def gelu64(v):
    return 0.5 * v * (1.0 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v * v * v)))


# --------------------------------------------------------------------------------------------------- check 2: fp32 restatement
def rms_r32(v, eps=EPS):
    return 1.0 / torch.sqrt((v * v).sum(-1, keepdim=True) / v.shape[-1] + eps)


def rmsnorm32(x, w, dt, eps=EPS, r_scale=1.0):
    """rmsnorm_kernel / the gemv_small prologue in fp32: T(T(x r) w)."""
    xf = x.float()
    return rnd(rnd(xf * (rms_r32(xf, eps) * r_scale), dt) * w.float(), dt)


def restate(dt, epi, acc, h=None, norm_out=None, eps=EPS, mut=None):
    """The batched epilogue kernels in fp32 torch on the kernel's accumulator acc (f32 [M][N], [M][2N] for SwiGLU): {"h": ...,
    "out": ...}. mut names a deliberately wrong chain (test_linear_plan.py's self-check of checks 2 and 3)."""
    R = (lambda v: rnd(v, "bf16")) if mut == "bf16_in_f16" else (lambda v: rnd(v, dt))
    a = acc.float()
    if epi == 0:
        return {"out": a}
    if epi == 1:
        hn = R(h.float() + (a if mut == "residual_unrounded_branch" else R(a)))
        res = {"h": hn}
        if norm_out is not None:
            xr = hn * rms_r32(hn, eps)
            res["out"] = R((xr if mut == "norm_no_round" else R(xr)) * norm_out.float())
        return res
    if epi == 2:
        F = a.shape[-1] // 2
        av, bv = R(a[:, :F]), R(a[:, F:])
        s = av / (1.0 + torch.exp(-av))
        return {"out": R((s if mut == "silu_no_inner_round" else R(s)) * bv)}
    v = R(a)
    if epi == 4:
        v = 0.5 * v * (1.0 + torch.tanh(0.7978845608028654 * (v + 0.044715 * v * v * v)))
    return {"out": R(v)}


def restated_problem(dt, got, want, epi, acc):
    """None when every output is within one ulp of T of the restatement and >= 99.9 % are bit-equal, else what is wrong. In an fp32
    model T is fp32 itself, so an ulp of expf / tanhf or of the row's r (epi 1 with the next norm, 2, 4) reaches the output
    unrounded: those outputs are held to 64 fp32 ulps (2^-18 relative) instead, plus, for gelu, 2^-21 |acc| for tanhf's absolute
    error where 1 + tanh cancels."""
    for k, w in want.items():
        o, w = got[k].double(), w.double()
        loose = dt == "f32" and k == "out" and epi in (1, 2, 4)
        eq = (o == w).double().mean().item()
        tol = ulp(torch.maximum(o.abs(), w.abs()), dt) * (64 if loose else 1)
        if loose and epi == 4:
            tol = tol + FN_ABS * acc.double().abs()
        far = int(((o - w).abs() > tol).sum())
        if (eq < 0.999 and not loose) or far:
            return f"{k}: {eq:.5f} bit-equal to the restatement, {far} beyond {64 if loose else 1} ulp"
    return None


# --------------------------------------------------------------------------------------------------- check 3: float64 chain
def _fn_interval(f, lo, hi, cmin):
    """[min, max] of a function with one minimum (at cmin) over [lo, hi], widened for its fp32 evaluation."""
    flo, fhi = f(lo), f(hi)
    mn, mx = torch.minimum(flo, fhi), torch.maximum(flo, fhi)
    inside = (lo <= cmin) & (hi >= cmin)
    mn = torch.where(inside, torch.minimum(mn, f(torch.full_like(lo, cmin))), mn)
    w_lo = FN_REL * mn.abs() + FN_ABS * torch.maximum(lo.abs(), hi.abs())
    w_hi = FN_REL * mx.abs() + FN_ABS * torch.maximum(lo.abs(), hi.abs())
    return mn - w_lo, mx + w_hi


def _mul_interval(alo, ahi, blo, bhi):
    c = torch.stack([alo * blo, alo * bhi, ahi * blo, ahi * bhi])
    return c.min(0).values, c.max(0).values


def _rms_r_interval(lo, hi, eps):
    sq_hi = torch.maximum(lo * lo, hi * hi)
    sq_lo = torch.where((lo <= 0) & (hi >= 0), torch.zeros_like(lo), torch.minimum(lo * lo, hi * hi))
    return (1.0 / torch.sqrt(sq_hi.mean(-1, keepdim=True) + eps) * (1 - DR),
            1.0 / torch.sqrt(sq_lo.mean(-1, keepdim=True) + eps) * (1 + DR))


def _norm_interval(dt, vlo, vhi, w, eps):
    """T(T(v r) w) over v in [vlo, vhi] and the r interval of the row."""
    rlo, rhi = _rms_r_interval(vlo, vhi, eps)
    plo, phi = torch.minimum(vlo * rlo, vlo * rhi), torch.maximum(vhi * rlo, vhi * rhi)
    ylo, yhi = rnd(plo, dt) * w, rnd(phi, dt) * w
    return rnd(torch.minimum(ylo, yhi), dt), rnd(torch.maximum(ylo, yhi), dt)


def chain64(dt, epi, ref, E, h=None, norm_out=None, eps=EPS):
    """{"h" / "out": (point, lo, hi)}: the float64 chain at acc = ref and over acc in [ref - E, ref + E]."""
    R = lambda v: rnd(v, dt)
    lo, hi = ref - E, ref + E
    if epi == 0:
        return {"out": (ref, lo, hi)}
    if epi == 1:
        hd = h.double()
        hp, hl, hh = R(hd + R(ref)), R(hd + R(lo)), R(hd + R(hi))
        res = {"h": (hp, hl, hh)}
        if norm_out is not None:
            w = norm_out.double()
            r = 1.0 / torch.sqrt((hp * hp).mean(-1, keepdim=True) + eps)
            res["out"] = (R(R(hp * r) * w), *_norm_interval(dt, hl, hh, w, eps))
        return res
    if epi == 2:
        F = ref.shape[-1] // 2
        ap, alo, ahi = R(ref[:, :F]), R(lo[:, :F]), R(hi[:, :F])
        bp, blo, bhi = R(ref[:, F:]), R(lo[:, F:]), R(hi[:, F:])
        slo, shi = _fn_interval(silu64, alo, ahi, SILU_MIN_AT)
        olo, ohi = _mul_interval(R(slo), R(shi), blo, bhi)
        return {"out": (R(R(silu64(ap)) * bp), R(olo), R(ohi))}
    vp, vlo, vhi = R(ref), R(lo), R(hi)
    if epi == 3:
        return {"out": (vp, vlo, vhi)}
    glo, ghi = _fn_interval(gelu64, vlo, vhi, GELU_MIN_AT)
    return {"out": (R(gelu64(vp)), R(glo), R(ghi))}


def chain_problem(got, chain, cap_frac, skip=None):
    """None when every output lies in its interval and fewer than cap_frac differ from the point value (outputs in `skip` are not
    counted), else what is wrong."""
    for k, (pt, lo, hi) in chain.items():
        o = got[k].double()
        out = (o < lo) | (o > hi)
        if out.any():
            i = out.nonzero()[0].tolist()
            return f"{k}: {int(out.sum())} outside the float64 interval, e.g. {tuple(i)}: {o[tuple(i)].item()!r} not in " \
                   f"[{lo[tuple(i)].item()!r}, {hi[tuple(i)].item()!r}]"
        if cap_frac is not None:
            diff = o != pt
            if skip is not None and k in skip:
                diff = diff & ~skip[k]
            frac = diff.double().mean().item()
            if frac > cap_frac:
                return f"{k}: {frac:.4f} of the outputs differ from the float64 chain (cap {cap_frac:.4f})"
    return None


# --------------------------------------------------------------------------------------------------- the C-ABI call
def run_linear(dt, x, wa, wb, epi, small, norm_in=None, norm_out=None, h=None, eps=EPS):
    """lg_test_linear. Returns ({"h" / "out": output}, acc_out or None, path)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    M, K = x.shape
    N = wa.shape[0]
    dev = x.device
    NN = 2 * N if wb is not None else N
    out_f32 = torch.empty(M, N, dtype=torch.float32, device=dev) if epi == 0 else None
    out = torch.empty(M, N, dtype=TDT[dt], device=dev) if (epi >= 2 or norm_out is not None) else None
    hh = h.clone() if epi == 1 else None
    acc = None if small else torch.empty(M, NN, dtype=torch.float32, device=dev)
    nbytes = 0 if small else 16 * M * NN * 4 + 256 + (M * K * 4 if norm_in is not None else 0)
    scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    path = (ctypes.c_int * 4)(-9, -9, -9, -9)
    P = _lib.ptr
    _lib.check(lib.lg_test_linear(LG_DT[dt], M, N, K, P(x), P(norm_in), ctypes.c_float(eps), P(wa), P(wb), epi, P(norm_out), P(hh),
                                  P(out), P(out_f32), P(acc), int(small), P(scratch) if nbytes else None, ctypes.c_size_t(nbytes),
                                  path, _lib.current_stream(dev)), "lg_test_linear")
    torch.cuda.synchronize()
    got = {}
    if epi == 0:
        got["out"] = out_f32
    if epi == 1:
        got["h"] = hh
    if out is not None:
        got["out"] = out
    return got, acc, tuple(path)


# --------------------------------------------------------------------------------------------------- case matrix
class Case:
    """One linear layer: M rows, N outputs (F for SwiGLU, epi 2, whose GEMM has 2F columns), K inputs. want: the leading entries of
    the path the case is meant to reach, pinned against plan_model."""

    def __init__(self, cid, dt, M, N, K, epi=0, small=False, norm_in=False, norm_out=False, tc=True, want=None):
        self.id, self.dt, self.M, self.N, self.K, self.epi, self.small = cid, dt, M, N, K, epi, small
        self.norm_in, self.norm_out, self.tc = norm_in, norm_out, tc
        self.env = {} if tc else {"LG_GEMM_TC": "0"}
        self.expect = plan_model(dt, M, N, K, epi == 2, small, tc)
        assert want is None or self.expect[:len(want)] == tuple(want), (cid, self.expect, want)


CASES = [
    # gemm_skinny_kernel: fp32 at any M, 16-bit at M <= 8 without the wgmma kernel
    Case("skinny_f32_m1", "f32", 1, 512, 1024, want=(0, 8, 2)),
    Case("skinny_f32_m3_residual", "f32", 3, 512, 1024, epi=1),
    Case("skinny_f32_m8_store", "f32", 8, 512, 1024, epi=3),
    Case("skinny_f32_m9_gelu", "f32", 9, 512, 1024, epi=4, want=(0, 8, 2, 2)),
    Case("skinny_f32_m130_residual_norm", "f32", 130, 512, 1024, epi=1, norm_out=True, want=(0, 8, 1, 17)),
    Case("skinny_f32_k2816_empty_slice", "f32", 8, 512, 2816, want=(0, 8, 5)),      # kper 768: the fifth k-slice is empty
    Case("skinny_bf16_k2816_empty_slice", "bf16", 3, 512, 2816, epi=3, tc=False, want=(0, 8, 5)),
    Case("skinny_f32_n200", "f32", 5, 200, 512, norm_in=True, want=(0, 8)),          # N % 16 != 0: a half-populated CTA
    Case("skinny_bf16_n200", "bf16", 4, 200, 512, epi=3, want=(0, 8)),                # N % 128 != 0: skinny with LG_GEMM_TC on
    Case("skinny_bf16_m8_residual", "bf16", 8, 768, 1024, epi=1, tc=False, want=(0, 8)),
    Case("skinny_f16_m2_gelu", "f16", 2, 1024, 768, epi=4, tc=False, want=(0, 8)),
    Case("skinny_f32_swiglu", "f32", 6, 256, 512, epi=2, want=(0, 8)),
    # gemm_mma_kernel: N % 128 != 0, or LG_GEMM_TC=0; K % 64 != 0
    Case("mma_bf16_bm32_n200_k200", "bf16", 20, 200, 200, epi=3, want=(1, 32)),
    Case("mma_f16_bm64_n1000_k1032", "f16", 50, 1000, 1032, epi=4, want=(1, 64)),
    Case("mma_bf16_bm128_residual_norm", "bf16", 130, 640, 512, epi=1, norm_out=True, tc=False, want=(1, 128, 2, 2)),
    Case("mma_f16_bm32_norm_in", "f16", 9, 384, 1024, norm_in=True, tc=False, want=(1, 32, 4)),
    # gemm_tc_kernel: every row pad, partial last row blocks, ksplit 1 and 16, short and empty last k-slices, K % 64 != 0
    Case("tc_bf16_pad16_m2", "bf16", 2, 384, 1024, want=(2, 16)),
    Case("tc_bf16_pad16_m9_residual", "bf16", 9, 256, 512, epi=1, want=(2, 16)),
    Case("tc_f16_pad32_n128", "f16", 32, 128, 768, epi=3, want=(2, 32)),
    Case("tc_bf16_pad64_k1000", "bf16", 40, 512, 1000, epi=4, want=(2, 64)),
    Case("tc_f16_pad128_residual_norm", "f16", 100, 256, 2048, epi=1, norm_out=True, want=(2, 128)),
    Case("tc_bf16_pad256", "bf16", 256, 384, 512, epi=3, want=(2, 256, 4, 1)),
    Case("tc_bf16_m257", "bf16", 257, 256, 512, epi=1, want=(2, 256, 4, 2)),
    Case("tc_f16_m383", "f16", 383, 256, 256, epi=3, want=(2, 256, 2, 2)),
    Case("tc_bf16_m1921", "bf16", 1921, 256, 512, epi=4, want=(2, 256, 4, 8)),        # the eighth row block holds 129 rows
    Case("tc_bf16_ks1", "bf16", 64, 512, 128, want=(2, 64, 1)),
    Case("tc_bf16_ks16", "bf16", 16, 256, 4096, want=(2, 16, 16)),
    Case("tc_f16_ks16_short_tail", "f16", 24, 256, 2816, epi=3, want=(2, 32, 16)),    # 44 k-blocks by 3: short, then empty slice
    Case("tc_bf16_k1032_short_tail", "bf16", 12, 256, 1032, epi=3, want=(2, 16, 8)),  # 17 k-blocks by 3
    # the two-segment weight [w1; w3] on all three GEMM kernels (w3 at 4x the scale of w1)
    Case("pair_tc_bf16_f256", "bf16", 16, 256, 512, epi=2, norm_in=True, want=(2, 16)),
    Case("pair_tc_f16_f384_m300", "f16", 300, 384, 256, epi=2, want=(2, 256)),
    Case("pair_mma_bf16_f256", "bf16", 40, 256, 512, epi=2, tc=False, want=(1, 64)),
    Case("pair_skinny_bf16_f256", "bf16", 4, 256, 512, epi=2, tc=False, want=(0, 8)),
    Case("pair_f704_bf16_m64", "bf16", 64, 704, 256, epi=2, want=(1, 64)),            # 2F = 11 * 128, F not a tile edge
    Case("pair_f704_f16_m300", "f16", 300, 704, 256, epi=2, norm_in=True, want=(1, 128)),
    Case("pair_f704_bf16_m5", "bf16", 5, 704, 256, epi=2, want=(0, 8)),
    # gemv_small: every R, each instantiation, chunk counts below PF and off the 8 warps, the largest K at R = 5, a prologue that
    # reads more norm-weight pieces than it requests ahead
    *[Case(f"small_r{R}_{EPI_NAMES[(0, 1, 2)[R % 3]]}", "bf16" if R % 2 else "f16", R, 256, 512, epi=(0, 1, 2)[R % 3], small=True,
           norm_in=R % 2 == 0) for R in range(1, 9)],
    Case("small_rows8_n2048_k256", "bf16", 2, 2048, 256, small=True, norm_in=True, want=(3, 8, 1, 12)),
    Case("small_rows16_n4096", "f16", 3, 4096, 512, epi=1, small=True, want=(3, 16, 1, 4)),
    Case("small_rows32_n16384", "bf16", 2, 16384, 256, small=True, norm_in=True, want=(3, 32, 1, 4)),
    Case("small_paired_r8_k1280", "f16", 8, 512, 1280, epi=2, small=True, norm_in=True, want=(3, 32, 1, 4)),
    Case("small_k288", "bf16", 3, 512, 288, epi=1, small=True),
    Case("small_k288_norm", "f16", 7, 512, 288, epi=0, small=True, norm_in=True),
    Case("small_r5_k8704", "bf16", 5, 3200, 8704, epi=1, small=True),                 # GPT-3B w2
    Case("small_r5_k9184", "f16", 5, 256, 9184, small=True, norm_in=True),            # the largest K the 90 KiB rule admits at R = 5
    Case("small_r8_k1280_norm", "bf16", 8, 256, 1280, small=True, norm_in=True),
    # batched epilogues: residual with and without the next norm (D / 4 threads: 16, 256, 800, 1024), SwiGLU / store / gelu at ksplit > 1
    *[Case(f"resid_d{D}{'_norm' if nrm else ''}", "bf16" if nrm else "f16", 16, D, min(D, 512), epi=1, norm_out=nrm)
      for D in (64, 1024, 3200, 4096) for nrm in (False, True)],
    Case("epi_swiglu_ks", "f16", 64, 512, 1024, epi=2, norm_in=True, want=(2, 64, 8)),
    Case("epi_store_ks", "bf16", 64, 512, 2048, epi=3, want=(2, 64, 16)),
    Case("epi_gelu_ks", "f16", 64, 512, 2048, epi=4, want=(2, 64, 16)),
]

# registry layer GEMMs (dim D, ffn_dim F) at R = 2 on the small path and R = 128 batched, bf16; GPT-B also batched at R = 2
REGISTRY = {"GPT-B": (768, 2048), "GPT-L": (1024, 2816), "GPT-XL": (1280, 3584), "GPT-XXL": (1536, 4096), "GPT-3B": (3200, 8704),
            "GPT-7B": (4096, 11008)}
V = 16384


def layer_cases(name, R, small):
    D, F = REGISTRY[name]
    tag = f"{name}_r{R}_{'small' if small else 'batched'}"
    return [
        Case(f"{tag}_qkv", "bf16", R, 3 * D, D, small=small, norm_in=True),                      # layer 0: attention norm first
        Case(f"{tag}_wo", "bf16", R, D, D, epi=1, small=small, norm_out=not small),
        Case(f"{tag}_w13", "bf16", R, F, D, epi=2, small=small, norm_in=small),
        Case(f"{tag}_w2", "bf16", R, D, F, epi=1, small=small, norm_out=not small),
        Case(f"{tag}_head", "bf16", R, V, D, small=small, norm_in=small),
    ]


for _n in REGISTRY:
    CASES += layer_cases(_n, 2, True) + layer_cases(_n, 128, False)
CASES += layer_cases("GPT-B", 2, False)
CASES += [Case("t2i_caption_fc1", "bf16", 240, 1280, 2048, epi=4),                # CaptionEmbedder of GPT-XL t2i: fc2(gelu(fc1(x)))
          Case("t2i_caption_fc2", "bf16", 240, 1280, 1280, epi=3)]
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES)


# --------------------------------------------------------------------------------------------------- one case end to end
def operands(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = TDT[c.dt]
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    x = rn(c.M, c.K).to(dt)
    wa = (rn(c.N, c.K) / math.sqrt(c.K)).to(dt)
    wb = (rn(c.N, c.K) * 4 / math.sqrt(c.K)).to(dt) if c.epi == 2 else None
    nin = (1 + 0.1 * rn(c.K)).to(dt) if c.norm_in else None
    h = rn(c.M, c.N).to(dt) if c.epi == 1 else None
    nout = (1 + 0.1 * rn(c.N)).to(dt) if c.norm_out else None
    return x, wa, wb, nin, h, nout


def reference(c, x, w, nin):
    """(ref64, E, skip-predicate inputs): the float64 accumulator at the point activation and its bound (check 1)."""
    wd = w.double()
    if nin is None:
        xp = x.double()
        E = E_REL * (xp.abs() @ wd.abs().t())
        return xp @ wd.t(), E, [xp]
    xd, nd = x.double(), nin.double()
    r = 1.0 / torch.sqrt((xd * xd).mean(-1, keepdim=True) + EPS)
    plo, phi = torch.minimum(xd * r * (1 - DR), xd * r * (1 + DR)), torch.maximum(xd * r * (1 - DR), xd * r * (1 + DR))
    ylo, yhi = rnd(plo, c.dt) * nd, rnd(phi, c.dt) * nd
    xlo, xhi = rnd(torch.minimum(ylo, yhi), c.dt), rnd(torch.maximum(ylo, yhi), c.dt)
    xps = [rmsnorm32(x, nin, c.dt, r_scale=s).double() for s in (1.0, 1 - 2.0 ** -22, 1 + 2.0 ** -22)]
    xp = xps[0]
    assert ((xp >= xlo) & (xp <= xhi)).all()
    E = E_REL * (xp.abs() @ wd.abs().t()) + (xhi - xlo) @ wd.abs().t()
    return xp @ wd.t(), E, xps


def run_case(c, monkeypatch, seed=0):
    for k in ("LG_GEMM_TC",):
        monkeypatch.delenv(k, raising=False)
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    x, wa, wb, nin, h, nout = operands(c, seed)
    got, acc, path = run_linear(c.dt, x, wa, wb, c.epi, c.small, norm_in=nin, norm_out=nout, h=h)
    assert path == c.expect, f"{c.id}: ran {path}, expected {c.expect}"
    w = wa if wb is None else torch.cat([wa, wb])
    ref, E, xps = reference(c, x, w, nin)
    # 1. accumulator
    for name, a in (("acc_out", acc), ("out_f32", got.get("out") if c.epi == 0 else None)):
        if a is not None:
            bad = (a.double() - ref).abs() > E
            assert not bad.any(), f"{c.id} {name}: {int(bad.sum())} of {bad.numel()} beyond E, worst " \
                                  f"{((a.double() - ref).abs() / E).max().item():.2f} E"
    # 2. batched epilogues on the kernel's own accumulator
    if acc is not None:
        want = restate(c.dt, c.epi, acc, h=h, norm_out=nout)
        if c.epi == 0:
            assert torch.equal(got["out"], acc), f"{c.id}: out_f32 differs from the same slabs summed into acc_out"
        else:
            p = restated_problem(c.dt, got, want, c.epi, acc)
            assert p is None, f"{c.id}: {p}"
    # 3. the chain in float64
    ch = chain64(c.dt, c.epi, ref, E, h=h, norm_out=nout)
    skip = None
    if len(xps) > 1:        # outputs whose point value moves with the prologue's fp32 r
        wd = w.double()
        alts = [chain64(c.dt, c.epi, xa @ wd.t(), E, h=h, norm_out=nout) for xa in xps[1:]]
        skip = {k: (alts[0][k][0] != ch[k][0]) | (alts[1][k][0] != ch[k][0]) for k in ch}
    cap_frac = cap(c.dt, c.K, 2 if c.epi == 2 else 1) if c.epi != 0 else None
    p = chain_problem(got, ch, cap_frac, skip)
    assert p is None, f"{c.id}: {p}"


@pytest.mark.parametrize("cid", list(CASE_BY_ID))
def test_linear_layer(cid, monkeypatch):
    run_case(CASE_BY_ID[cid], monkeypatch)


def test_scratch_too_small_reports_its_size():
    from llamagen_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(16, 512, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(256, 512, dtype=torch.bfloat16, device="cuda")
    y = torch.zeros(16, 256, dtype=torch.float32, device="cuda")
    s = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    P = _lib.ptr
    rc = lib.lg_test_linear(1, 16, 256, 512, P(x), None, ctypes.c_float(EPS), P(w), None, 0, None, None, None, P(y), None, 0, P(s),
                            ctypes.c_size_t(1024), None, _lib.current_stream(x.device))
    err = lib.lg_last_error().decode()
    ks = plan_model("bf16", 16, 256, 512, False, False)[2]
    assert rc < 0 and f"scratch 1024 < {ks * 16 * 256 * 4}" in err, err


def test_ffn_dim_704_model_generates_and_scores():
    """ffn_dim 704 (dim 256 with multiple_of 64): 2F = 1408 is a multiple of 128 but the w1 | w3 boundary is not, so the batched
    w1 | w3 GEMM runs on gemm_mma_kernel. generate and score at B = 16 meet the bf16 oracle bounds of test_gpt_gpu / test_score_gpu."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    from test_gpt_gpu import _bf16_parity
    from test_score_gpu import _parity_16
    torch.manual_seed(7)
    m = Transformer(ModelArgs(n_layer=2, n_head=4, dim=256, multiple_of=64, block_size=64, vocab_size=1024))
    assert m.config.ffn_dim == 704
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    cond = torch.randint(0, 1000, (16,))
    _bf16_parity(m, cond, 6)
    _parity_16(m, cond, torch.randint(0, 1024, (16, 64)), 4.0)
