"""Call-level parity of every transformer attention kernel path against a float64 reference.

lg_test_attention runs one attention call through the engine's own dispatch (launch_attention) over a KV buffer of several layers,
with tensor maps built as lg_engine_set_workspace builds them, and reports the kernel that ran: (kernel, ring depth, fused), kernel
0 = attention_kernel (CUDA cores), 1 = attn_tma_kernel, 3 = attn_prefill_tc_kernel. Every case asserts the triple it must run on.

Reference: plain torch in float64 from the operands exactly as the kernel reads them (q, K and V in the model dtype T, or the decoded
e4m3 codes times the layer's K / V scale). Key j is visible to the query at position qpos iff
j <= qpos and (j >= Tc or mask[r % B, j] != 0 or j == qpos).

Bounds follow from the kernels' arithmetic, not from the spread between models. absO = sum p |v| / sum p bounds every term a kernel
adds; dmax = max over the visible keys of |q|.|k| / sqrt(hd):
  |out - ref| <= delta + ulp_T(|ref| + delta) / 2,  delta = (u_P + 2 eps_dot + 2^-20 + (n + 2) 2^-23) absO [+ n 2^-25 vmax]
  * u_P: P (<= 1 after the running max is subtracted) is rounded to T before P.V on the tensor cores: the unit roundoff of T,
    2^-8 for bf16 (8 significant bits), 2^-11 for fp16; 0 on the CUDA-core kernel and for fp32. sum p is taken from the unrounded
    fp32 p, so the rounding enters the numerator only. fp16 rounds p < 2^-14 to a subnormal with an absolute error of at most
    2^-25: the bracketed term, vmax the largest visible |v|, since sum p >= 1.
  * eps_dot = (hd + 1) 2^-23 dmax: fp32 accumulation of q.k with one ulp per step (truncating tensor-core adds included) and the
    scaling; a score error e moves p by a factor e^e in the numerator and denominator, hence the 2.
  * 2^-20 = 2 x 2^-21: __expf (ex2.approx) on the scores. The running-max corrections multiply O and L alike and cancel.
  * (n + 2) 2^-23: fp32 sums of p v and p over the n visible keys, the division O / L.
  * ulp_T / 2: the final rounding to T; fp32 outputs are held to the same formula with ulp_fp32 and u_P = 0.
  On the CUDA-core kernel a 16-bit output must also equal T(ref) for all but 1 % of the elements (at least one is allowed).

The inputs make a wrong kernel miss by O(|v|), not by a rounding error:
  * needles: one key per (row, head) scores about 24 against N(0, 2) for the rest (the margin of 12 is asserted), with a distinct V
    row; its position sweeps the 16-row box, 32-key chunk, deep-ring refill, condition and diagonal edges.
  * poison: every key past the query position, every emb-masked condition key and every other layer of the buffer would have the top
    score and carries V of about 2^12 (bf16 / fp32), 2^14 (fp16) or e4m3 codes of 256..448.
  * wide: scores from -60 to 60 rising along the context, so the maximum arrives last and the running max rescales at every chunk.
  * hd 100 in 112-wide rows: garbage in dims 100..111 must give bit-identical outputs.
  * guard bands: `out`, `q_out` and every cache byte outside the rows the call writes must be unchanged.
With the QKV slabs as input, the K / V rows written at the query position (and, unfused, q) are bit-equal to an fp32 torch
restatement of the epilogue, and the fused and unfused writers store identical bytes.
"""
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from kv_fp8_oracle import e4m3_bytes

TORCH_DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
LG_DT = {"f32": 0, "bf16": 1, "f16": 2}
LG_E4M3 = 3
MANT = {"f32": 24, "bf16": 8, "f16": 11}
U_P = {"f32": 0.0, "bf16": 2.0 ** -8, "f16": 2.0 ** -11}   # unit roundoff of T
DEV = "cuda"
C0 = 0.125           # score = C0 (u + z / 4) . kappa: kappa (K in code units) has about 8 per dim of noise


# ---------------------------------------------------------------------------------------------------------------- references
def e4m3_decode(codes):
    """float64 value of e4m3 codes (uint8): sign, 4-bit exponent (bias 7), 3-bit mantissa; exponent 0 is subnormal (m 2^-9)."""
    c = codes.long()
    sign = 1.0 - 2.0 * ((c >> 7) & 1).double()
    e = (c >> 3) & 15
    m = (c & 7).double()
    normal = (1.0 + m / 8.0) * torch.pow(2.0, (e - 7).double())
    return sign * torch.where(e == 0, m * 2.0 ** -9, normal)


def visibility(qpos, mask, B, Tc, S):
    """[R, Tq, S] bool: key j visible to the query at qpos[r, t]."""
    j = torch.arange(S, device=qpos.device)
    vis = j <= qpos[..., None]
    if mask is not None:
        R = qpos.shape[0]
        cond = torch.ones(R, S, dtype=torch.bool, device=qpos.device)
        cond[:, :Tc] = mask[torch.arange(R, device=qpos.device) % B] != 0
        vis = vis & (cond[:, None, :] | (j == qpos[..., None]))
    return vis


def attention_ref(q, k, v, qpos, mask=None, B=1, Tc=0):
    """q [R, Tq, H, hd], k / v [R, H, S, hd] (float64, the values the kernel reads), qpos [R, Tq].
    Returns out, absO [R, Tq, H, hd], dmax [R, Tq, H], the visible-key count [R, Tq] and the largest visible |v| [R, Tq, H]."""
    hd, S = q.shape[-1], k.shape[2]
    vis = visibility(qpos, mask, B, Tc, S)[:, None]                         # [R, 1, Tq, S]
    s = torch.einsum("rthd,rhsd->rhts", q, k) / math.sqrt(hd)
    p = torch.softmax(s.masked_fill(~vis, float("-inf")), dim=-1)
    out = torch.einsum("rhts,rhsd->rthd", p, v)
    abs_o = torch.einsum("rhts,rhsd->rthd", p, v.abs())
    dots = (torch.einsum("rthd,rhsd->rhts", q.abs(), k.abs()) / math.sqrt(hd)).masked_fill(~vis, 0.0)
    vmax = v.abs().amax(-1)[:, :, None, :].masked_fill(~vis, 0.0).amax(-1).permute(0, 2, 1)
    return out, abs_o, dots.amax(-1).permute(0, 2, 1), vis[:, 0].sum(-1), vmax


def epilogue_ref(partial, freqs, qpos, dt, H, hd, kv_scales=None):
    """The QKV epilogue in fp32 torch: sequential slab sum, round to T, RoPE with separately rounded products, round to T; fp8:
    e4m3_satfinite(x / s). partial [ks, M, 3 H hd], qpos [M]. Returns q, k, v [M, H, hd] (k / v as uint8 codes for fp8)."""
    T = TORCH_DT[dt]
    s = partial[0].clone()
    for i in range(1, partial.shape[0]):
        s = s + partial[i]
    x = s.to(T).float().view(-1, 3, H, hd // 2, 2)
    cs = freqs[qpos.long()][:, None, None]                                   # [M, 1, 1, hd / 2, 2]
    c, sn = cs[..., 0], cs[..., 1]
    x0, x1 = x[:, :2, ..., 0], x[:, :2, ..., 1]
    y = torch.stack([x0 * c - x1 * sn, x1 * c + x0 * sn], dim=-1).to(T)
    q, k = y[:, 0].reshape(-1, H, hd), y[:, 1].reshape(-1, H, hd)
    v = x[:, 2].reshape(-1, H, hd).to(T)
    if kv_scales is not None:
        k, v = e4m3_bytes(k, kv_scales[0]), e4m3_bytes(v, kv_scales[1])
    return q, k, v


def ulp(x, dt):
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), e - MANT[dt])
    return u.clamp(min=2.0 ** -24) if dt == "f16" else u


# ------------------------------------------------------------------------------------------------------ CPU self-checks
def test_reference_matches_sdpa_with_explicit_mask():
    torch.manual_seed(0)
    R, Tq, H, hd, S, B, Tc = 4, 5, 3, 16, 23, 2, 9
    q = torch.randn(R, Tq, H, hd, dtype=torch.float64)
    k, v = torch.randn(R, H, S, hd, dtype=torch.float64), torch.randn(R, H, S, hd, dtype=torch.float64)
    qpos = torch.tensor([[0, 1, 2, 3, 4], [3, 4, 5, 6, 7], [8, 9, 10, 11, 12], [17, 18, 19, 20, 21]])
    mask = torch.tensor([[0, 0, 0, 1, 1, 0, 1, 1, 1], [0] * 9], dtype=torch.float32)
    allowed = torch.zeros(R, H, Tq, S, dtype=torch.bool)
    for r in range(R):
        for t in range(Tq):
            p = int(qpos[r, t])
            for j in range(S):
                allowed[r, :, t, j] = j <= p and (j >= Tc or mask[r % B, j] != 0 or j == p)
    want = F.scaled_dot_product_attention(q.permute(0, 2, 1, 3), k, v, attn_mask=allowed).permute(0, 2, 1, 3)
    got, abs_o, dmax, nvis, vmax = attention_ref(q, k, v, qpos, mask, B, Tc)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    assert torch.equal(nvis, allowed[:, 0].sum(-1))
    assert (abs_o >= got.abs() - 1e-12).all() and (dmax > 0).all() and (vmax[..., None] >= abs_o - 1e-12).all()


def test_e4m3_decode_of_every_finite_code():
    codes = torch.tensor([c for c in range(256) if c not in (0x7F, 0xFF)], dtype=torch.uint8)
    want = codes.view(torch.float8_e4m3fn).double()
    assert codes.numel() == 254 and torch.equal(e4m3_decode(codes), want)
    assert torch.equal(e4m3_bytes(e4m3_decode(codes).float()), codes)


def test_epilogue_rope_is_a_rotation():
    torch.manual_seed(1)
    M, H, hd = 3, 2, 8
    part = torch.randn(2, M, 3 * H * hd)
    ang = torch.rand(5, hd // 2) * 6.28
    freqs = torch.stack([ang.cos(), ang.sin()], -1)
    qpos = torch.tensor([0, 2, 4])
    q, k, v = epilogue_ref(part, freqs, qpos, "f32", H, hd)
    x = (part[0] + part[1]).double().view(M, 3, H, hd // 2, 2)
    rot = torch.view_as_complex(x[:, 1].contiguous()) * torch.polar(torch.ones_like(ang), ang).to(torch.complex128)[qpos][:, None]
    assert torch.allclose(k.double(), torch.view_as_real(rot).reshape(M, H, hd), atol=1e-5)
    assert torch.equal(v, (part[0] + part[1]).view(M, 3, H, hd)[:, 2])


# ------------------------------------------------------------------------------------------------------ case matrix
class Case:
    """One attention call. pos: ("scalar", p) | ("dev", p) | ("rows", [p_r]) for the query's first position; mask: ("ragged", B, Tc)
    or None; inp: "q", "slab" (QKV epilogue kernel, then attention) or "fused"; expect: (kernel, stages, fused)."""

    def __init__(self, cid, dt, kv, hd, R, H, S, expect, hdp=None, Tq=1, pos=None, mask=None, inp="q", ks=2, layers=(2, 1),
                 scales=(1.0, 1.0), env=None, needles=True):
        self.id, self.dt, self.kv, self.hd, self.R, self.H, self.S, self.expect = cid, dt, kv, hd, R, H, S, expect
        self.hdp = hdp or hd
        self.Tq, self.pos, self.mask, self.inp, self.ks, self.layers = Tq, pos or ("scalar", S - Tq), mask, inp, ks, layers
        self.scales, self.env, self.needles = scales, env or {}, needles

    @property
    def combo(self):
        return (*self.expect, self.dt, self.kv, self.hd, self.hdp)

    def positions(self):
        kind, val = self.pos
        return torch.tensor(val) if kind == "rows" else torch.full((self.R,), val)


def dispatchable():
    """Every (kernel, stages, fused, dtype, kv, hd, hdp) launch_attention can select: fp32 rows are hd wide, bf16 / fp16 store hd 100
    in 112-wide rows."""
    out = {(0, 0, 0, "f32", "auto", hd, hd) for hd in (64, 128, 100)}
    for dt in ("bf16", "f16"):
        for kv in ("auto", "fp8"):
            for hd, hdp in ((64, 64), (128, 128), (100, 112)):
                out |= {(1, 2, 0, dt, kv, hd, hdp), (1, 2, 1, dt, kv, hd, hdp), (0, 0, 0, dt, kv, hd, hdp)}
            out.add((3, 1, 0, dt, kv, 64, 64))
            out |= {(1, st, 1, dt, kv, 64, 64) for st in (3, 8)}
    return out


FP8_SCALES = [(2.0 ** -8, 2.0 ** 7), (1.0, 1.0), (2.0 ** 7, 2.0 ** -8)]
LENGTHS = [1, 2, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 255, 256, 257, 289, 376, 377, 1144]
MASK4 = ("ragged", 2, 120)      # decode, R = 4
MASK_PF = ("ragged", 3, 120)    # prefill, R = 6


def _cases():
    cs = []
    # one case per dispatchable combination at a context with a tail chunk
    i = 0
    for dt in ("bf16", "f16"):
        for kv in ("auto", "fp8"):
            for hd, hdp in ((64, 64), (128, 128), (100, 112)):
                sc = FP8_SCALES[i % 3] if kv == "fp8" else (1.0, 1.0)
                i += 1
                pos = ("dev", 203) if i % 2 else ("scalar", 203)
                tag = f"{dt}_{kv}_{hd}_{hdp}"
                cs.append(Case(f"tma_{tag}", dt, kv, hd, 3, 2, 230, (1, 2, 0), hdp=hdp, pos=pos, scales=sc))
                cs.append(Case(f"fused_{tag}", dt, kv, hd, 17 if hd == 64 else 2, 16 if hd == 64 else 3, 230, (1, 2, 1), hdp=hdp,
                               pos=pos, inp="fused", scales=sc))
                cs.append(Case(f"cc_notma_{tag}", dt, kv, hd, 3, 2, 230, (0, 0, 0), hdp=hdp, pos=pos, scales=sc,
                               env={"LG_ATTN_TMA": "0"}))
            sc = FP8_SCALES[i % 3] if kv == "fp8" else (1.0, 1.0)
            cs.append(Case(f"fused_nst3_{dt}_{kv}", dt, kv, 64, 17, 16, 300, (1, 3, 1), pos=("dev", 290), inp="fused",
                           scales=sc, env={"LG_ATTN_NST": "3"}))
            cs.append(Case(f"fused_s300_{dt}_{kv}", dt, kv, 64, 17, 16, 300, (1, 2, 1), pos=("dev", 290), inp="fused", scales=sc))
            cs.append(Case(f"deep_{dt}_{kv}", dt, kv, 64, 2, 4, 300, (1, 8, 1), pos=("scalar", 290), inp="fused", scales=sc))
            cs.append(Case(f"prefill_tc_{dt}_{kv}", dt, kv, 64, 6, 2, 377, (3, 1, 0), Tq=120, pos=("scalar", 0), mask=MASK_PF,
                           scales=sc, env={"LG_ATTN_PREFILL_TC": "1"}))
    for hd in (64, 128, 100):
        cs.append(Case(f"cc_f32_{hd}", "f32", "auto", hd, 3, 2, 230, (0, 0, 0), pos=("dev", 203)))
    # "wide": many (row, head) items (R * H >= 528) on the unfused 2-stage kernel, as a large decode batch runs it
    cs.append(Case("wide_bf16", "bf16", "auto", 64, 33, 16, 300, (1, 2, 0), pos=("scalar", 290)))
    # context lengths (nkeys = position + 1) on the main kernels
    for n in LENGTHS:
        S = n + 23
        cs.append(Case(f"len{n}_tma_bf16", "bf16", "auto", 64, 2, 3, S, (1, 2, 0), pos=("scalar", n - 1)))
        cs.append(Case(f"len{n}_tma_f16_fp8_128", "f16", "fp8", 128, 2, 2, S, (1, 2, 0), pos=("dev", n - 1), scales=FP8_SCALES[n % 3]))
        cs.append(Case(f"len{n}_deep_bf16_fp8", "bf16", "fp8", 64, 1, 4, S, (1, 8, 1), pos=("scalar", n - 1), inp="fused",
                       scales=FP8_SCALES[n % 3]))
        cs.append(Case(f"len{n}_fused_f16", "f16", "auto", 64, 17, 16, S, (1, 2, 1), pos=("dev", n - 1), inp="fused", needles=n < 300))
        cs.append(Case(f"len{n}_cc_f32", "f32", "auto", 64, 2, 2, S, (0, 0, 0), pos=("scalar", n - 1)))
        if n in (16, 17, 33, 256, 257, 377, 1144):
            cs.append(Case(f"len{n}_wide", "bf16", "auto", 64, 33, 16, S, (1, 2, 0), pos=("scalar", n - 1), needles=False))
            cs.append(Case(f"len{n}_fused_hd112", "bf16", "auto", 100, 2, 2, S, (1, 2, 1), hdp=112, pos=("scalar", n - 1),
                           inp="fused"))
    # the last (row, head) of the last layer at max_seq - 1, max_seq 257 / 377 (c2i / t2i): the tail boxes cross the map's end
    for S in (257, 377):
        end = ("scalar", S - 1)
        cs += [Case(f"end{S}_tma_bf16", "bf16", "auto", 64, 2, 3, S, (1, 2, 0), pos=end, layers=(3, 2)),
               Case(f"end{S}_tma_f16_fp8_112", "f16", "fp8", 100, 2, 3, S, (1, 2, 0), hdp=112, pos=end, layers=(3, 2)),
               Case(f"end{S}_deep_bf16", "bf16", "auto", 64, 2, 3, S, (1, 8, 1), pos=end, inp="fused", layers=(3, 2)),
               Case(f"end{S}_fused_f16_fp8", "f16", "fp8", 64, 17, 16, S, (1, 2, 1), pos=end, inp="fused", layers=(3, 2)),
               Case(f"end{S}_wide", "bf16", "auto", 64, 33, 16, S, (1, 2, 0), pos=end, layers=(3, 2), needles=False)]
    # per-row positions: rows at 0, chunk edges and max_seq - 1 in one call (as lg_decode_rows passes them)
    rows = [0, 15, 16, 31, 32, 33, 63, 64, 255, 256, 299, 300]
    cs += [Case("rows_tma_bf16", "bf16", "auto", 64, 12, 2, 301, (1, 2, 0), pos=("rows", rows)),
           Case("rows_slab_f16_fp8", "f16", "fp8", 128, 12, 2, 301, (1, 2, 0), pos=("rows", rows), inp="slab", scales=FP8_SCALES[0]),
           Case("rows_deep_bf16", "bf16", "auto", 64, 12, 2, 301, (1, 8, 1), pos=("rows", rows), inp="fused"),
           Case("rows_fused_f16_112", "f16", "auto", 100, 12, 2, 301, (1, 2, 1), hdp=112, pos=("rows", rows), inp="fused"),
           Case("rows_cc_f32", "f32", "auto", 128, 12, 2, 301, (0, 0, 0), pos=("rows", rows)),
           Case("rows_cc_bf16_fp8_112", "bf16", "fp8", 100, 12, 2, 301, (0, 0, 0), hdp=112, pos=("rows", rows), scales=FP8_SCALES[2],
                env={"LG_ATTN_TMA": "0"})]
    # decode with an emb-mask, query positions inside and past the condition (the j == qpos exemption)
    mrows = [50, 119, 120, 300]
    cs += [Case("mask_tma_bf16", "bf16", "auto", 64, 4, 2, 301, (1, 2, 0), pos=("rows", mrows), mask=MASK4),
           Case("mask_tma_f16_fp8", "f16", "fp8", 128, 4, 2, 301, (1, 2, 0), pos=("rows", mrows), mask=MASK4, scales=FP8_SCALES[1]),
           Case("mask_deep_bf16", "bf16", "auto", 64, 4, 2, 301, (1, 8, 1), pos=("rows", mrows), mask=MASK4, inp="fused"),
           Case("mask_wide_bf16", "bf16", "auto", 64, 66, 8, 377, (1, 2, 0), pos=("scalar", 300), mask=("ragged", 33, 120),
                needles=False),
           Case("mask_cc_f32", "f32", "auto", 64, 4, 2, 301, (0, 0, 0), pos=("rows", mrows), mask=MASK4),
           Case("mask_cc_f16_fp8", "f16", "fp8", 64, 4, 2, 301, (0, 0, 0), pos=("rows", mrows), mask=MASK4, scales=FP8_SCALES[2],
                env={"LG_ATTN_TMA": "0"})]
    # t2i condition prefill: Tq query rows at positions 0.., ragged / all-zero / all-one mask rows, R = 2B (CFG twins share rows)
    for Tq in (2, 15, 16, 17, 120, 127, 128):
        m = ("ragged", 3, min(Tq, 120))
        cs += [Case(f"prefill{Tq}_tc_bf16", "bf16", "auto", 64, 6, 2, 377, (3, 1, 0), Tq=Tq, pos=("scalar", 0), mask=m),
               Case(f"prefill{Tq}_tc_f16_fp8", "f16", "fp8", 64, 6, 2, 377, (3, 1, 0), Tq=Tq, pos=("scalar", 0), mask=m,
                    scales=FP8_SCALES[Tq % 3]),
               Case(f"prefill{Tq}_cc_bf16_notc", "bf16", "auto", 64, 6, 2, 377, (0, 0, 0), Tq=Tq, pos=("scalar", 0), mask=m,
                    env={"LG_ATTN_PREFILL_TC": "0"}),
               Case(f"prefill{Tq}_cc_f16_128", "f16", "auto", 128, 6, 2, 377, (0, 0, 0), Tq=Tq, pos=("scalar", 0), mask=m)]
    cs += [Case("prefill120_slab_tc_bf16_fp8", "bf16", "fp8", 64, 6, 2, 377, (3, 1, 0), Tq=120, pos=("scalar", 0), mask=MASK_PF,
                inp="slab", scales=FP8_SCALES[2], ks=3),
           Case("prefill120_slab_cc_f32", "f32", "auto", 64, 6, 2, 377, (0, 0, 0), Tq=120, pos=("scalar", 0), mask=MASK_PF, inp="slab"),
           Case("prefill120_cc_bf16_fp8_112", "bf16", "fp8", 100, 6, 2, 377, (0, 0, 0), hdp=112, Tq=120, pos=("scalar", 0), mask=MASK_PF,
                scales=FP8_SCALES[0]),
           Case("decode_past_prefill_cc_f16_2tq", "f16", "auto", 64, 2, 2, 200, (0, 0, 0), Tq=3, pos=("dev", 150))]
    # unfused slab writers next to the fused ones (same bytes), fused at position 0 (no cached key)
    cs += [Case("slab_bf16_64", "bf16", "auto", 64, 3, 2, 230, (1, 2, 0), pos=("dev", 203), inp="slab", ks=3),
           Case("slab_f16_fp8_112", "f16", "fp8", 100, 3, 2, 230, (1, 2, 0), hdp=112, pos=("scalar", 203), inp="slab",
                scales=FP8_SCALES[1]),
           Case("slab_cc_f32_100", "f32", "auto", 100, 3, 2, 230, (0, 0, 0), pos=("scalar", 203), inp="slab", ks=1)]
    return cs


CASES = _cases()
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES)


def test_case_matrix_covers_every_dispatchable_kernel():
    """The cases' (kernel, stages, fused) annotations, which the GPU run asserts, cover every combination the dispatch selects."""
    have = {c.combo for c in CASES}
    assert dispatchable() <= have, sorted(dispatchable() - have)
    assert have <= dispatchable(), sorted(have - dispatchable())
    for c in CASES:
        assert c.kv == "auto" or c.dt != "f32"
        assert c.expect[2] == (c.inp == "fused")
        k = c.expect[0]
        rh = c.R * c.H
        if c.expect == (1, 8, 1):
            assert rh <= 264 and c.hd == 64
        elif c.expect[:2] == (1, 2) and c.expect[2] and c.hd == 64:
            assert rh > 264
        if k == 3:
            assert 1 < c.Tq <= 128 and c.S >= 128 and c.pos == ("scalar", 0)
    nkeys = {p + 1 for c in CASES if c.Tq == 1 for p in c.positions().tolist()}
    assert set(LENGTHS) <= nkeys
    assert {c.Tq for c in CASES if c.expect[0] == 3} >= {2, 15, 16, 17, 120, 127, 128}
    assert {s for c in CASES if c.kv == "fp8" for s in c.scales} == {2.0 ** -8, 1.0, 2.0 ** 7}
    assert "3" in {c.env.get("LG_ATTN_NST") for c in CASES} and any(c.env.get("LG_ATTN_TMA") == "0" for c in CASES)
    assert {c.env.get("LG_ATTN_PREFILL_TC") for c in CASES} >= {"0", "1"}


# ------------------------------------------------------------------------------------------------------ inputs
def _mask(c, dev):
    """[B, Tc] left-padded masks: row 0 ragged, row 1 all zero, row 2 all one, further rows ragged."""
    if c.mask is None:
        return None, 1, 0
    _, B, Tc = c.mask
    pads = [min(60, Tc // 2), Tc, 0] + [(7 * b + 3) % Tc for b in range(3, B)]
    return torch.stack([(torch.arange(Tc) >= p).float() for p in pads[:B]]).to(dev), B, Tc


def _needle_specs(c, Tc):
    specs = [("abs", j) for j in (0, 15, 16, 31, 32, 33)] + [("rel", d) for d in (16, 15, 1, 0)]
    if Tc:
        specs += [("abs", Tc - 1), ("abs", Tc)]
    if c.expect[1] == 8:
        specs += [("abs", 32 * g) for g in range(8)] + [("abs", 32 * (8 + g)) for g in range(8)]
    return list(dict.fromkeys(specs))


def _poison_v(shape, c, gen, dev):
    sign = torch.randint(0, 2, shape, generator=gen, device=dev) * 2.0 - 1.0
    if c.kv == "fp8":                                             # codes 0x70..0x7E: 256 .. 448
        codes = torch.randint(0x70, 0x7F, shape, generator=gen, device=dev)
        return sign * e4m3_decode(codes.to(torch.uint8))
    mag = 2.0 ** 14 if c.dt == "f16" else 2.0 ** 12
    return sign * mag * (1 + torch.rand(shape, generator=gen, device=dev, dtype=torch.float64))


def _design(c, scen, needle, seed, dev):
    """Scores, query and cache contents in code units (K = k_scale kappa, V = v_scale nu). Returns a dict of float64 tensors."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=gen, device=dev, dtype=torch.float64)
    R, H, S, hd, Tq = c.R, c.H, c.S, c.hd, c.Tq
    L, layer = c.layers
    ks, vs = c.scales
    pos = c.positions().to(dev)
    qpos = pos[:, None] + torch.arange(Tq, device=dev)
    qmax = qpos[:, -1]
    j = torch.arange(S, device=dev)
    if scen == "needle":
        s, top = rnd(R, H, S), 34.0
    else:
        frac = j[None, :].double() / qmax.clamp(min=1)[:, None].double()
        s, top = ((-60.0 + 100.0 * frac)[:, None, :] + 5.0 * rnd(R, H, S)).clamp(-60.0, 60.0), 70.0
    vmag = 16.0 if c.kv == "fp8" else 1.0
    nu = vmag * rnd(R, H, S, hd)
    has_needle = torch.zeros(R, dtype=torch.bool, device=dev)
    jn = torch.zeros(R, dtype=torch.long, device=dev)
    if needle is not None:
        kind, val = needle
        jn = torch.full_like(qmax, val) if kind == "abs" else qmax - val
        has_needle = (jn >= 0) & (jn <= qmax)
        for r in has_needle.nonzero().flatten().tolist():
            j_r = int(jn[r])
            s[r, :, j_r] = 24.0
            nu[r, :, j_r] = 4.0 * vmag * (torch.randint(0, 2, (H, hd), generator=gen, device=dev) * 2.0 - 1.0)
    mask, B, Tc = _mask(c, dev)
    poison = j[None, :] > qmax[:, None]
    if mask is not None:
        cond = torch.zeros(R, S, dtype=torch.bool, device=dev)
        cond[:, :Tc] = mask[torch.arange(R, device=dev) % B] == 0
        poison |= cond
    s = torch.where(poison[:, None], torch.full_like(s, top), s)
    nu = torch.where(poison[:, None, :, None], _poison_v((R, H, S, hd), c, gen, dev), nu)
    u = rnd(R, H, hd)
    u = u / u.norm(dim=-1, keepdim=True)
    kappa = (s[..., None] * u[:, :, None, :] + rnd(R, H, S, hd)) / C0
    q = (C0 * math.sqrt(hd) / ks) * (u[:, None] + 0.25 * rnd(R, Tq, H, hd) / math.sqrt(hd))
    # the other layers: every key would win, every value is poison
    kap_o = (top * u[:, :, None, :] + rnd(R, H, S, hd)) / C0
    nu_o = _poison_v((R, H, S, hd), c, gen, dev)
    return dict(qpos=qpos, q=q, kappa=kappa, nu=nu, kap_o=kap_o, nu_o=nu_o, mask=mask, B=B, Tc=Tc, poison=poison,
                has_needle=has_needle, jn=jn, gen=gen, L=L, layer=layer)


def _store(x, c, scale):
    """Code-unit values -> the cache's storage (T, or e4m3 codes of x) and the float64 values the kernel reads (times the scale)."""
    if c.kv == "fp8":
        codes = e4m3_bytes(x.float())
        return codes, e4m3_decode(codes) * scale
    t = (x * scale).to(TORCH_DT[c.dt])
    return t, t.double()


def _cache(c, d, which, pad):
    """[L, R, H, S, hdp] storage of K ("k") or V ("v"); pad: "zero" or "garbage" in dims hd..hdp."""
    x, xo, scale = (d["kappa"], d["kap_o"], c.scales[0]) if which == "k" else (d["nu"], d["nu_o"], c.scales[1])
    L, layer = d["L"], d["layer"]
    st, _ = _store(xo, c, scale)
    buf = st.unsqueeze(0).repeat(L, 1, 1, 1, 1)
    buf[layer] = _store(x, c, scale)[0]
    if c.hdp > c.hd:
        buf = torch.cat([buf, torch.zeros(*buf.shape[:-1], c.hdp - c.hd, dtype=buf.dtype, device=buf.device)], dim=-1)
        if pad == "garbage":
            g = torch.Generator(device=buf.device).manual_seed(99)
            if c.kv == "fp8":
                gb = torch.randint(0, 0x7F, buf[..., c.hd:].shape, generator=g, device=buf.device).to(torch.uint8)
            else:
                gb = (100.0 * torch.randn(buf[..., c.hd:].shape, generator=g, device=buf.device)).to(buf.dtype)
            buf[..., c.hd:] = gb
    return buf.contiguous()


def _slabs(c, d, dev):
    """QKV split-K slabs whose epilogue reproduces the designed q, K and V rows at the query positions, and a RoPE table."""
    gen = d["gen"]
    R, H, S, hd, Tq = c.R, c.H, c.S, c.hd, c.Tq
    ang = torch.rand(S, hd // 2, generator=gen, device=dev) * (2 * math.pi)
    freqs = torch.stack([ang.cos(), ang.sin()], dim=-1).float().contiguous()
    qp = d["qpos"].reshape(-1)
    rr = torch.arange(R, device=dev).repeat_interleave(Tq)
    kk = d["kappa"][rr, :, qp] * c.scales[0]                           # [M, H, hd]
    vv = d["nu"][rr, :, qp] * c.scales[1]
    qq = d["q"].reshape(R * Tq, H, hd)
    cs = freqs[qp].double()[:, None]                                    # [M, 1, hd / 2, 2]
    def unrope(y):
        y = y.view(*y.shape[:-1], hd // 2, 2)
        c_, s_ = cs[..., 0], cs[..., 1]
        return torch.stack([y[..., 0] * c_ + y[..., 1] * s_, y[..., 1] * c_ - y[..., 0] * s_], -1).flatten(-2)
    x = torch.stack([unrope(qq), unrope(kk), vv], dim=1).reshape(R * Tq, 3 * H * hd)
    parts = [0.05 * torch.randn(R * Tq, 3 * H * hd, generator=gen, device=dev, dtype=torch.float64) for _ in range(c.ks - 1)]
    p0 = x - sum(parts) if parts else x
    return torch.stack([p0] + parts).float().contiguous(), freqs


def _run(c, kbuf, vbuf, d, q=None, partial=None, freqs=None, fuse=0, dev="cuda"):
    from llamagen_b200 import _lib
    lib = _lib.load()
    T = TORCH_DT[c.dt]
    R, H, hd, Tq, S = c.R, c.H, c.hd, c.Tq, c.S
    n, G = R * Tq * H * hd, 64
    out_buf = torch.full((n + 2 * G,), -12345.0, dtype=T, device=dev)
    qo_buf = torch.full((n + 2 * G,), -4321.0, dtype=T, device=dev) if (partial is not None and not fuse) else None
    kind, val = c.pos
    pos_dev = pos_rows = None
    pos_value = 0
    if kind == "rows":
        pos_rows = torch.tensor(val, dtype=torch.int32, device=dev)
    elif kind == "dev":
        off = min(val, 7)
        pos_dev, pos_value = torch.tensor([val - off], dtype=torch.int32, device=dev), off
    else:
        pos_value = val
    mask, B, Tc = d["mask"], d["B"], d["Tc"]
    path = (ctypes.c_int * 3)(-1, -1, -1)
    P = _lib.ptr
    out = out_buf[G:G + n]
    q_out = qo_buf[G:G + n] if qo_buf is not None else None
    L, layer = d["L"], d["layer"]
    _lib.check(lib.lg_test_attention(LG_DT[c.dt], LG_E4M3 if c.kv == "fp8" else LG_DT[c.dt], c.scales[0], c.scales[1], R, Tq, H, hd,
                                     c.hdp, S, P(kbuf), P(vbuf), L, layer, pos_value, P(pos_dev), P(pos_rows), P(mask), B, Tc, P(q),
                                     P(partial), c.ks, P(freqs), fuse, P(q_out), P(out), path, _lib.current_stream(dev)),
               f"lg_test_attention {c.id}")
    torch.cuda.synchronize()
    for buf, fill in ((out_buf, -12345.0), (qo_buf, -4321.0)):
        if buf is not None:
            guard = torch.cat([buf[:G], buf[G + n:]])
            assert torch.equal(guard, torch.full_like(guard, fill)), f"{c.id}: write outside out / q_out"
    return out.view(R, Tq, H, hd), (q_out.view(R * Tq, H, hd) if q_out is not None else None), tuple(path)


def _check(c, out, ref, abs_o, dmax, nvis, vmax, kernel, what):
    o = out.double()
    rel = U_P[c.dt] * (kernel != 0) + 2 * (c.hd + 1) * 2.0 ** -23 * dmax[..., None] + 2.0 ** -20 \
        + (nvis[:, :, None, None] + 2) * 2.0 ** -23
    delta = rel * abs_o
    if kernel != 0 and c.dt == "f16":
        delta = delta + (nvis[:, :, None, None] * 2.0 ** -25) * vmax[..., None]
    bound = delta + 0.5 * ulp(ref.abs() + delta, c.dt)
    err = (o - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; worst err {err[bad].max().item():.4g} "
                           f"bound {bound[bad].min().item():.4g} absO {abs_o[bad].max().item():.4g}")
    if kernel == 0 and c.dt != "f32":
        wrong = int((o != ref.to(TORCH_DT[c.dt]).double()).sum())
        assert wrong <= max(1, 0.01 * o.numel()), f"{what}: {wrong} of {o.numel()} outputs not T(ref)"
    return (err / abs_o.clamp(min=1e-300)).max().item()


def _one(c, scen, needle, seed, pad="zero"):
    """Runs one call; returns the output and the written cache rows (for the fused / unfused comparison)."""
    dev = DEV
    d = _design(c, scen, needle, seed, dev)
    kbuf, vbuf = _cache(c, d, "k", pad), _cache(c, d, "v", pad)
    L, layer = d["L"], d["layer"]
    R, H, hd, Tq = c.R, c.H, c.hd, c.Tq
    rr = torch.arange(R, device=dev).repeat_interleave(Tq)
    qp = d["qpos"].reshape(-1)
    inp_q = partial = freqs = None
    if c.inp == "q":
        inp_q = d["q"].to(TORCH_DT[c.dt]).reshape(R * Tq, H * hd).contiguous()
        qref = inp_q.view(R, Tq, H, hd).double()
    else:
        partial, freqs = _slabs(c, d, dev)
        for buf in (kbuf, vbuf):      # the rows this call writes hold poison until the writer replaces them
            buf[layer, rr, :, qp] = buf[(layer + 1) % L, rr, :, qp]
    k0, v0 = kbuf.clone(), vbuf.clone()
    out, q_out, path = _run(c, kbuf, vbuf, d, q=inp_q, partial=partial, freqs=freqs, fuse=int(c.inp == "fused"), dev=dev)
    assert path == c.expect, f"{c.id}: ran {path}, expected {c.expect}"
    written = None
    if partial is not None:
        f8 = c.scales if c.kv == "fp8" else None
        qr, kr, vr = epilogue_ref(partial, freqs, qp, c.dt, H, hd, f8)
        got_k, got_v = kbuf[layer, rr, :, qp, :hd], vbuf[layer, rr, :, qp, :hd]
        assert torch.equal(got_k, kr), f"{c.id}: K row bytes differ from the epilogue restatement"
        assert torch.equal(got_v, vr), f"{c.id}: V row bytes differ from the epilogue restatement"
        if q_out is not None:
            assert torch.equal(q_out, qr), f"{c.id}: q differs from the epilogue restatement"
        for buf, ref_buf, new in ((kbuf, k0, kr), (vbuf, v0, vr)):
            ref_buf[layer, rr, :, qp, :hd] = new
        written = (got_k.clone(), got_v.clone())
        qref = qr.to(TORCH_DT[c.dt]).view(R, Tq, H, hd).double()
    assert torch.equal(kbuf, k0) and torch.equal(vbuf, v0), f"{c.id}: cache bytes changed outside the written rows"
    if c.kv == "fp8":
        kref = e4m3_decode(kbuf[layer, ..., :hd]) * c.scales[0]
        vref = e4m3_decode(vbuf[layer, ..., :hd]) * c.scales[1]
    else:
        kref, vref = kbuf[layer, ..., :hd].double(), vbuf[layer, ..., :hd].double()
    ref, abs_o, dmax, nvis, vmax = attention_ref(qref, kref, vref, d["qpos"], d["mask"], d["B"], d["Tc"])
    if scen == "needle" and needle is not None and c.inp == "q":
        _assert_margin(c, d, qref, kref)
    rel = _check(c, out, ref, abs_o, dmax, nvis, vmax, path[0], f"{c.id}/{scen}/{needle}")
    return out, written, rel


def _assert_margin(c, d, qref, kref):
    """The needle beats every other visible key by at least 12 wherever it is visible and no poison key is."""
    vis = visibility(d["qpos"], d["mask"], d["B"], d["Tc"], c.S)                  # [R, Tq, S]
    s = torch.einsum("rthd,rhsd->rhts", qref, kref) / math.sqrt(c.hd)             # [R, H, Tq, S]
    R, H, Tq = c.R, c.H, c.Tq
    jn = d["jn"].clamp(0, c.S - 1)
    at = jn[:, None, None].expand(R, Tq, 1)
    seen = vis.gather(2, at)[..., 0] & d["has_needle"][:, None] & ~(vis & d["poison"][:, None, :]).any(-1)    # [R, Tq]
    others = vis.scatter(2, at, False)
    s_needle = s.gather(3, jn[:, None, None, None].expand(R, H, Tq, 1))[..., 0]
    s_other = s.masked_fill(~others[:, None], float("-inf")).amax(-1)
    margin = (s_needle - s_other).permute(0, 2, 1)[seen]
    assert margin.numel() == 0 or margin.min().item() >= 12, f"{c.id}: needle margin {margin.min().item():.2f}"


# ------------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASE_BY_ID))
def test_attention_call(cid, monkeypatch):
    c = CASE_BY_ID[cid]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    seed = zlib.crc32(cid.encode())
    worst = _one(c, "wide", None, seed)[2]
    _, Tc = (c.mask[1], c.mask[2]) if c.mask else (1, 0)
    if c.needles:
        for i, nd in enumerate(_needle_specs(c, Tc)):
            worst = max(worst, _one(c, "needle", nd, seed + 1 + i)[2])
    else:
        for nd in (("rel", 0), ("rel", 1), ("abs", 0)):
            worst = max(worst, _one(c, "needle", nd, seed + 7)[2])
    if c.hdp > c.hd:
        a = _one(c, "needle", ("rel", 1), seed + 99, pad="zero")[0]
        b = _one(c, "needle", ("rel", 1), seed + 99, pad="garbage")[0]
        assert torch.equal(a, b), f"{cid}: dims {c.hd}..{c.hdp - 1} of the cache rows change the output"
    print(f"[{cid}] path {c.expect} max |out - ref| / absO {worst:.3g}")


FUSE_PAIRS = [c.id for c in CASES if c.inp == "fused" and c.pos[0] != "rows"]


@pytest.mark.gpu
@pytest.mark.parametrize("cid", FUSE_PAIRS)
def test_fused_and_unfused_writers_store_the_same_bytes(cid, monkeypatch):
    c = CASE_BY_ID[cid]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    seed = zlib.crc32(cid.encode()) + 5
    _, wf, _ = _one(c, "needle", ("rel", 0), seed)
    u = Case(c.id + "_unfused", c.dt, c.kv, c.hd, c.R, c.H, c.S, (1, 2, 0), hdp=c.hdp, pos=c.pos, mask=c.mask, inp="slab", ks=c.ks,
             layers=c.layers, scales=c.scales)
    _, wu, _ = _one(u, "needle", ("rel", 0), seed)
    assert torch.equal(wf[0], wu[0]) and torch.equal(wf[1], wu[1])


@pytest.mark.gpu
def test_argument_validation():
    """Host-side rejections only: every buffer is large enough that no call could address outside it."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    dev = "cuda"
    R, H, hd, S, L = 2, 2, 64, 64, 2
    kv = torch.zeros(L * R * H * S * 112 * 4, dtype=torch.uint8, device=dev)
    q = torch.zeros(4 * R * H * 128, dtype=torch.float32, device=dev)
    out = torch.zeros_like(q)
    part = torch.zeros(3 * 4 * R * H * 128, dtype=torch.float32, device=dev)
    freqs = torch.zeros(S * 64 * 2, dtype=torch.float32, device=dev)
    P = _lib.ptr
    st = _lib.current_stream(dev)

    def call(dt=1, kvdt=1, ks=1.0, vs=1.0, Tq=1, hd_=hd, hdp=hd, layer=1, pos=0, qq=q, pp=None, fuse=0, qo=None, n_layer=L):
        path = (ctypes.c_int * 3)(-1, -1, -1)
        rc = lib.lg_test_attention(dt, kvdt, ks, vs, R, Tq, H, hd_, hdp, S, P(kv), P(kv), n_layer, layer, pos, None, None, None, 1, 0,
                                   P(qq), P(pp), 1, P(freqs), fuse, P(qo), P(out), path, st)
        return rc, lib.lg_last_error().decode()

    for kw, msg in [(dict(dt=0, kvdt=LG_E4M3), "KV dtype"), (dict(kvdt=LG_E4M3, ks=3.0), "scales"), (dict(ks=0.5), "scales"),
                    (dict(pos=S), "exceeds max_seq"), (dict(pos=S - 1, Tq=2), "exceeds max_seq"), (dict(hd_=96, hdp=96), "head_dim"),
                    (dict(dt=0, kvdt=0, hd_=100, hdp=112), "row width"), (dict(hd_=100, hdp=100), "row width"),
                    (dict(dt=2, kvdt=2, hd_=100, hdp=100), "row width"), (dict(layer=2), "bad shape"), (dict(qq=None), "exactly one"),
                    (dict(pp=part), "exactly one"), (dict(qq=None, pp=part), "fuse"), (dict(fuse=1), "fuse"),
                    (dict(qq=None, pp=part, fuse=1, Tq=2), "fused QKV"), (dict(qq=None, pp=part, fuse=1, dt=0, kvdt=0), "fused QKV")]:
        rc, err = call(**kw)
        assert rc < 0 and msg in err, (kw, rc, err)
    torch.cuda.synchronize()
