"""Layer-level parity of every VQ convolution and GroupNorm kernel path against a float64 reference.

lg_test_vq_conv runs one convolution through the decoder's own dispatch (run_conv) and reports which kernel ran
(0 = mma.sync gather, 1 = conv_tc_kernel, 2 = conv_tcw_kernel) and how many GroupNorm partial-statistics splits its drain wrote;
lg_test_group_norm runs the stand-alone GroupNorm. The references are plain torch in float64 on the GPU, from the operands exactly
as the kernel sees them (bf16 activations, bf16(W), and for the tensor-core upsample the bf16 2x2 phase weights summed in fp32).

Bounds follow from fp32 accumulation, not from the spread between models. `absconv` is the same float64 convolution of |x| and
|W| plus |bias| and |residual|: it bounds every term the kernel adds.
  * f32 outputs: |y - ref| <= 2^-13 absconv. Serial fp32 accumulation over <= ~300 k16 steps stays below ~2^-14.8 absconv even with
    truncating tensor cores, while one missing 64-channel k-block or tap moves the result by ~(64 / K) absconv (2^-6 at K = 4608).
  * bf16 outputs: |y - ref| <= ulp(ref) / 2 + 2^-13 absconv (correctly rounded unless the float64 value lies within the accumulation
    error of a rounding midpoint), and fewer than 1 % of elements differ from bf16(ref).
  * uint8 outputs: bit-equal to torch's clamp(127.5 f + 128, 0, 255).to(uint8) of the same call's f32 output, and within 1 LSB of
    the same finishing applied to the float64 reference.
  * GroupNorm: one bf16 ulp of the float64 result plus 2^-16 |gamma_c| (1 + |mu_g| / sigma_g) for outputs near zero; fewer than 1 %
    of elements off the correctly rounded value.
"""
import ctypes
import zlib

import pytest
import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------------------------------------------- references
# Taps of the 3x3 kernel that land on input offset a of a 2x2 phase kernel, per output parity p (rows and columns alike):
# p = 0 reads input rows (y - 1, y), p = 1 reads (y, y + 1).
_PHASE_TAPS = {(0, 0): (0,), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2,)}


def phase_weights(w):
    """[2, 2, Cout, Cin, 2, 2] sums of the 3x3 taps per (py, px, a, b), accumulated in w's dtype in the kernel's order (ky outer,
    kx inner, starting from zero)."""
    co, ci = w.shape[:2]
    out = w.new_zeros(2, 2, co, ci, 2, 2)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    s = w.new_zeros(co, ci)
                    for ky in _PHASE_TAPS[py, a]:
                        for kx in _PHASE_TAPS[px, b]:
                            s = s + w[:, :, ky, kx]
                    out[py, px, :, :, a, b] = s
    return out


def phase_conv(x, wp):
    """nearest-2x upsample + 3x3 conv (pad 1) evaluated as four 2x2 convolutions of the low-resolution NCHW input."""
    B, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros(B, wp.shape[2], 2 * H, 2 * W)
    for py in range(2):
        for px in range(2):
            out[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + H + 1, px:px + W + 1], wp[py, px])
    return out


def conv_ref(x, w, k, up, phase=False):
    """float64 NCHW convolution of NCHW x by w. up: 0 = same size (pad k // 2), 1 = nearest-2x upsample first (phase: through
    the 2x2 phase weights w, shaped like phase_weights()), 2 = Downsample (zero pad right/bottom by one, stride 2)."""
    if up == 1:
        return phase_conv(x, w) if phase else F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, padding=1)
    if up == 2:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)
    return F.conv2d(x, w, padding=k // 2)


def group_norm_ref(x, gamma, beta, swish):
    """float64 GroupNorm(32, eps 1e-6) [+ swish] of NHWC x [B, HW, C]; also the per-(image, group) mean and std, [B, 32]."""
    B, HW, C = x.shape
    xd = x.double().permute(0, 2, 1)
    y = F.group_norm(xd, 32, gamma.double(), beta.double(), eps=1e-6)
    if swish:
        y = y * torch.sigmoid(y)
    g = xd.reshape(B, 32, -1)
    mu = g.mean(-1)
    sd = (g.var(-1, unbiased=False) + 1e-6).sqrt()
    return y.permute(0, 2, 1), mu, sd


def ulp_bf16(r):
    _, e = torch.frexp(r)                    # |r| in [2^(e-1), 2^e): 8 significant bits -> spacing 2^(e-8)
    return torch.ldexp(torch.ones_like(r), e - 8)


def u8_finish(f):
    return torch.clamp(127.5 * f + 128.0, 0, 255).to(torch.uint8)


# ------------------------------------------------------------------------------------------------------ CPU self-checks
def test_phase_reference_equals_upsample_conv():
    torch.manual_seed(0)
    x = torch.randn(2, 16, 5, 7, dtype=torch.float64)
    w = torch.randn(8, 16, 3, 3, dtype=torch.float64)
    want = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w, padding=1)
    got = conv_ref(x, phase_weights(w), 3, 1, phase=True)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)


def test_downsample_reference_equals_tap_sum():
    """Downsample (pad right/bottom by one, 3x3 stride 2) as the oracle writes it, against an explicit sum over the nine taps."""
    torch.manual_seed(1)
    x = torch.randn(2, 8, 10, 6, dtype=torch.float64)
    w = torch.randn(4, 8, 3, 3, dtype=torch.float64)
    b = torch.randn(4, dtype=torch.float64)
    got = conv_ref(x, w, 3, 2) + b[None, :, None, None]
    xp = torch.zeros(2, 8, 12, 8, dtype=torch.float64)
    xp[:, :, :10, :6] = x
    want = b[None, :, None, None].expand(2, 4, 5, 3).clone()
    for ky in range(3):
        for kx in range(3):
            want += torch.einsum("bchw,oc->bohw", xp[:, :, ky:ky + 10:2, kx:kx + 6:2], w[:, :, ky, kx])
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    orc = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2, padding=0)       # oracle/vq_oracle.py encode_z
    assert torch.allclose(got, orc, rtol=0, atol=1e-12)


def test_group_norm_reference_matches_torch():
    torch.manual_seed(2)
    x = torch.randn(2, 36, 64, dtype=torch.float64) * 3 + 5
    gamma, beta = torch.randn(64, dtype=torch.float64), torch.randn(64, dtype=torch.float64)
    for swish in (0, 1):
        got, mu, sd = group_norm_ref(x, gamma, beta, swish)
        g = x.reshape(2, 36, 32, 2)
        m = g.mean(dim=(1, 3), keepdim=True)
        v = ((g - m) ** 2).mean(dim=(1, 3), keepdim=True)
        want = ((g - m) / (v + 1e-6).sqrt()).reshape(2, 36, 64) * gamma + beta
        if swish:
            want = F.silu(want)
        assert torch.allclose(got, want, rtol=0, atol=1e-12)
        assert torch.allclose(mu, m.reshape(2, 32), rtol=0, atol=1e-12)
        assert torch.allclose(sd, (v + 1e-6).sqrt().reshape(2, 32), rtol=0, atol=1e-12)
    tg = torch.nn.GroupNorm(32, 64, eps=1e-6).double()
    tg.weight.data.copy_(gamma)
    tg.bias.data.copy_(beta)
    want = tg(x.permute(0, 2, 1)).permute(0, 2, 1)
    assert torch.allclose(group_norm_ref(x, gamma, beta, 0)[0], want, rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ C-ABI wrappers
def _out_hw(H, W, up):
    return (2 * H, 2 * W) if up == 1 else ((H // 2, W // 2) if up == 2 else (H, W))


def vq_conv(x, w, bias, k, up, out="bf", residual=None, inplace=False, gn=None):
    """lg_test_vq_conv. x bf16 NHWC, w f32 [Cout, Cin, k, k]; out: "bf" (bf16 NHWC), "f32" (NCHW) or "u8" (NHWC).
    inplace: the output buffer starts as a copy of `residual` and is passed as both. gn: (gamma, beta, swish) or None.
    Returns (y, path, gn_splits, partials [B, splits, 32, (sum, sum of squares)] or None, gn_out or None)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, Hin, Win, Cin = x.shape
    Cout = w.shape[0]
    Ho, Wo = _out_hw(Hin, Win, up)
    dev = x.device
    out_bf = out_nchw = out_u8 = None
    if out == "bf":
        out_bf = residual.clone() if inplace else torch.empty(B, Ho, Wo, Cout, dtype=torch.bfloat16, device=dev)
    elif out == "f32":
        out_nchw = torch.empty(B, Cout, Ho, Wo, dtype=torch.float32, device=dev)
    else:
        out_u8 = torch.empty(B, Ho, Wo, Cout, dtype=torch.uint8, device=dev)
    res = out_bf if inplace else residual
    a256 = lambda n: (n + 255) // 256 * 256
    max_splits = max(64, -(-Hin // 16) * -(-Win // 16) * 4)
    scratch_bytes = a256(Cout * Cin * k * k * 2) + a256(16 * Cout * Cin * 2) + B * max_splits * 64 * 4
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    part = torch.zeros(B * max_splits * 64, dtype=torch.float32, device=dev)
    gn_out = torch.empty(B, Ho, Wo, Cout, dtype=torch.bfloat16, device=dev) if gn is not None else None
    path, splits = ctypes.c_int(-1), ctypes.c_int(-1)
    P = _lib.ptr
    _lib.check(lib.lg_test_vq_conv(P(x), B, Hin, Win, Cin, P(w), P(bias), Cout, k, up, P(res), P(out_bf), P(out_nchw), P(out_u8),
                                   P(gn[0]) if gn else None, P(gn[1]) if gn else None, int(gn[2]) if gn else 0, P(gn_out),
                                   P(part), ctypes.c_size_t(part.numel()), P(scratch), ctypes.c_size_t(scratch_bytes),
                                   ctypes.byref(path), ctypes.byref(splits), _lib.current_stream(dev)), "lg_test_vq_conv")
    torch.cuda.synchronize()
    y = out_bf if out == "bf" else (out_nchw if out == "f32" else out_u8)
    p = part[:B * splits.value * 64].view(B, splits.value, 32, 2).clone() if splits.value > 0 else None
    return y, path.value, splits.value, p, gn_out


def group_norm(x, gamma, beta, swish):
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, HW, C = x.shape
    y = torch.empty_like(x)
    scratch = torch.empty(B * 64 * 64, dtype=torch.float32, device=x.device)
    _lib.check(lib.lg_test_group_norm(_lib.ptr(x), B, HW, C, _lib.ptr(gamma), _lib.ptr(beta), int(swish), _lib.ptr(y),
                                      _lib.ptr(scratch), ctypes.c_size_t(scratch.numel() * 4), _lib.current_stream(x.device)),
               "lg_test_group_norm")
    torch.cuda.synchronize()
    return y


# ------------------------------------------------------------------------------------------------------ case matrix
class Case:
    """One convolution. path: the kernel the tensor-core dispatch must pick (LG_CONV_TC=1); the mma.sync path (0) is also run when
    it accepts the case (every output but uint8). gn: the GroupNorm of a ResnetBlock follows (with and without drain statistics)."""

    def __init__(self, cid, B, H, W, cin, cout, k=3, up=0, out="bf", res=None, path=2, gn=False, wscale=1.0, boff=0.0, env=None):
        self.id, self.B, self.H, self.W, self.cin, self.cout, self.k, self.up = cid, B, H, W, cin, cout, k, up
        self.out, self.res, self.path, self.gn, self.wscale, self.boff, self.env = out, res, path, gn, wscale, boff, env or {}

    @property
    def mode(self):
        return 2 if self.up == 1 else (3 if self.up == 2 else (1 if self.k == 1 else 0))

    @property
    def bn(self):                            # conv_tc_kernel's Cout tile
        bn = 16
        while bn < 128 and bn < self.cout:
            bn *= 2
        return bn if self.path == 1 else 256

    def fused_splits(self, fuse=True):
        """Partial-statistics splits conv_tcw_kernel's drain writes: one per 16x16 tile (and upsample phase) of the tiled grid."""
        if self.path != 2 or self.out != "bf" or not fuse or self.cout % 32 or 128 % (self.cout // 32):
            return 0
        ht, wt = (self.H // 2, self.W // 2) if self.up == 2 else (self.H, self.W)
        return -(-ht // 16) * -(-wt // 16) * (4 if self.up == 1 else 1)


CASES = [
    # registry decoder layers (VQ-16 at 16x16 / 24x24 grids, VQ-8)
    Case("conv_in_256_512_16", 3, 16, 16, 256, 512, gn=True),
    Case("conv_in_256_512_24", 1, 24, 24, 256, 512),
    Case("res_512_16", 3, 16, 16, 512, 512, gn=True),
    Case("res_512_24", 1, 24, 24, 512, 512, res="sep", gn=True),
    Case("res_256_32", 1, 32, 32, 256, 256, res="sep", gn=True),
    Case("res_128_64", 1, 64, 64, 128, 128, res="inplace", gn=True),
    Case("nin_512_256", 1, 32, 32, 512, 256, k=1),
    Case("nin_256_128", 1, 64, 64, 256, 128, k=1),
    Case("attn_proj_512_inplace", 3, 16, 16, 512, 512, k=1, res="inplace", gn=True),
    Case("up_512_16", 1, 16, 16, 512, 512, up=1, gn=True),
    Case("up_512_24", 1, 24, 24, 512, 512, up=1),
    Case("up_256_32", 1, 32, 32, 256, 256, up=1, gn=True),
    Case("up_128_64", 1, 64, 64, 128, 128, up=1),
    Case("conv_out_128", 1, 128, 128, 128, 3, out="f32", path=1, wscale=0.4),
    Case("conv_out_256", 1, 256, 256, 128, 3, out="f32", path=1, wscale=0.4),
    Case("conv_out_128_u8", 1, 128, 128, 128, 3, out="u8", path=1, wscale=0.4),
    Case("conv_out_256_u8", 1, 256, 256, 128, 3, out="u8", path=1, wscale=0.4),
    # registry encoder layers
    Case("down_128_256", 1, 256, 256, 128, 128, up=2),
    Case("down_256_32", 3, 32, 32, 256, 256, up=2, gn=True),
    Case("enc_conv_out_512_256", 3, 16, 16, 512, 256),
    Case("quant_conv_256_8", 3, 16, 16, 256, 8, k=1, out="f32", path=1),   # f32 output: Cout = 8 is a masked BN = 16 tile
    # conv_tc_kernel: every BN, masked Cout tails, odd k-chunk count, 1x1 with a single k-block
    *[Case(f"tc_cout{c}", 3, 16, 16, 64, c, path=1, res="sep" if c in (48, 160) else None, gn=c in (32, 64))
      for c in (16, 32, 48, 64, 96, 160, 192)],
    Case("tc_cin192", 3, 16, 16, 192, 64, path=1),
    Case("tc_1x1_64_128", 3, 16, 16, 64, 128, k=1, path=1),
    # conv_tcw_kernel edges
    Case("tcw_1x1_nkb2", 3, 16, 16, 128, 128, k=1, gn=True),
    Case("tcw_cout384", 1, 16, 16, 128, 384),                               # 128 % (384 / 32) != 0: no drain statistics
    Case("tcw_swap0", 3, 16, 16, 512, 512, path=1, env={"LG_CONV_SWAP": "0"}, gn=True),
    # patch shapes: the 8-wide patch, overhanging patches, non-square images, small upsample / Downsample
    Case("bw8_16x8", 3, 16, 8, 64, 64, path=1),
    Case("bw8_12x12", 3, 12, 12, 128, 128, path=1, gn=True),
    Case("overhang_40", 1, 40, 40, 128, 128, gn=True),
    Case("tc_overhang_24", 3, 24, 24, 64, 64, path=1),
    # outputs whose |mean| / std is about 100: drain statistics and stand-alone statistics must keep the variance
    Case("tcw_bias100", 1, 24, 24, 128, 128, gn=True, boff=100.0),
    Case("tc_bias100", 3, 16, 16, 64, 64, path=1, gn=True, boff=-100.0),
    *[Case(f"nonsq_{h}x{w}_{name}", 1, h * (2 if up == 2 else 1), w * (2 if up == 2 else 1), 128, cout, k=k, up=up, path=path,
           gn=path == 2 and up != 2)
      for h, w in ((16, 40), (40, 16))
      for name, cout, k, up, path in (("m0_tcw", 128, 3, 0, 2), ("m0_tc", 64, 3, 0, 1), ("m1", 128, 1, 0, 2), ("m2", 128, 3, 1, 2),
                                      ("m3", 128, 3, 2, 2))],
    Case("up_hin8", 3, 8, 8, 128, 128, up=1, path=1),
    Case("up_hin12", 3, 12, 12, 128, 128, up=1, path=1, gn=True),
    Case("down_to_8", 3, 16, 16, 128, 128, up=2, path=1),
    Case("down_to_12", 3, 24, 24, 128, 128, up=2, path=1),
]
CASE_BY_ID = {c.id: c for c in CASES}
assert len(CASE_BY_ID) == len(CASES)


def test_case_matrix_covers_every_kernel_path():
    """Every case asserts the kernel it ran on, so the table's expectations are what the GPU run covered."""
    assert {c.path for c in CASES} == {1, 2} and any(c.out != "u8" for c in CASES)          # + path 0 for every non-uint8 case
    assert {c.bn for c in CASES if c.path == 1} == {16, 32, 64, 128}
    for p in (1, 2):
        assert {c.mode for c in CASES if c.path == p} == {0, 1, 2, 3}, p
    assert {c.mode for c in CASES if c.out != "u8"} == {0, 1, 2, 3}                      # the mma.sync path
    assert {c.B for c in CASES} == {1, 3}
    assert any(c.fused_splits() for c in CASES) and any(c.path == 2 and not c.fused_splits() for c in CASES)


# ------------------------------------------------------------------------------------------------------ GPU tests
def _operands(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(c.B, c.H, c.W, c.cin, device="cuda", generator=g).bfloat16()
    w = torch.randn(c.cout, c.cin, c.k, c.k, device="cuda", generator=g) * (c.wscale / (c.cin * c.k * c.k) ** 0.5)
    bias = 0.5 * torch.randn(c.cout, device="cuda", generator=g) + c.boff
    Ho, Wo = _out_hw(c.H, c.W, c.up)
    res = torch.randn(c.B, Ho, Wo, c.cout, device="cuda", generator=g).bfloat16() if c.res else None
    gamma = 1.0 + 0.5 * torch.randn(c.cout, device="cuda", generator=g)
    beta = 0.5 * torch.randn(c.cout, device="cuda", generator=g)
    return x, w, bias, res, gamma, beta


def _reference(c, x, w, bias, res, phase):
    """(ref, absconv), float64 NCHW."""
    xd = x.double().permute(0, 3, 1, 2)
    if phase:
        wq = phase_weights(w).bfloat16().double()             # fp32 tap sums, then bf16: the kernel's phase weights
    else:
        wq = w.bfloat16().double()
    ref = conv_ref(xd, wq, c.k, c.up, phase) + bias.double()[None, :, None, None]
    absconv = conv_ref(xd.abs(), wq.abs(), c.k, c.up, phase) + bias.double().abs()[None, :, None, None]
    if res is not None:
        rd = res.double().permute(0, 3, 1, 2)
        ref, absconv = ref + rd, absconv + rd.abs()
    return ref, absconv


def _check_bf16(y, ref, absconv, what):
    yd = y.double().permute(0, 3, 1, 2)
    err = (yd - ref).abs()
    bound = 0.5 * ulp_bf16(ref) + 2.0 ** -13 * absconv
    bad = err > bound
    assert not bad.any(), f"{what}: {bad.sum().item()} elements outside the bound, worst excess {(err - bound).max().item():.3g}"
    wrong = (yd != ref.bfloat16().double()).double().mean().item()
    assert wrong < 0.01, f"{what}: {wrong:.2%} of elements not correctly rounded"
    return (err / absconv).max().item(), wrong


def _check_f32(y, ref, absconv, what):
    err = (y.double() - ref).abs()
    rel = (err / absconv).max().item()
    assert rel <= 2.0 ** -13, f"{what}: max |y - ref| / absconv = 2^{torch.log2(torch.tensor(rel)).item():.2f}"
    return rel


def _check_partials(part, y, cout):
    """The drain's per-split (sum, sum of squares) summed over splits == float64 group sums of the stored bf16 output, so
    overhanging patch pixels contribute nothing."""
    B = y.shape[0]
    v = y.double().reshape(B, -1, 32, cout // 32)
    s_ref, q_ref, a_ref = v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3)), v.abs().sum(dim=(1, 3))
    s, q = part.double().sum(1).unbind(-1)
    assert ((s - s_ref).abs() <= 1e-5 * a_ref).all(), (s - s_ref).abs().max().item()
    assert ((q - q_ref).abs() <= 1e-5 * q_ref).all(), ((q - q_ref).abs() / q_ref).max().item()


def _check_gn(y, x, gamma, beta, swish, what):
    ref, mu, sd = group_norm_ref(x.reshape(x.shape[0], -1, x.shape[-1]), gamma, beta, swish)
    C = x.shape[-1]
    yd = y.double().reshape(ref.shape)
    floor = 2.0 ** -16 * gamma.double().abs()[None, None, :] * (1 + (mu / sd).abs()).repeat_interleave(C // 32, dim=1)[:, None, :]
    err = (yd - ref).abs()
    bound = ulp_bf16(ref) + floor
    bad = err > bound
    assert not bad.any(), f"{what}: {bad.sum().item()} of {bad.numel()} outside the bound, worst err {err.max().item():.3g}"
    wrong = (yd != ref.bfloat16().double()).double().mean().item()
    assert wrong < 0.01, f"{what}: {wrong:.2%} of elements not correctly rounded"
    return err.max().item(), wrong


def _run_case(c, x, w, bias, res, gn=None):
    return vq_conv(x, w, bias, c.k, c.up, out=c.out, residual=res, inplace=c.res == "inplace", gn=gn)


@pytest.mark.gpu
@pytest.mark.parametrize("conv", ["tc", "mma"])
@pytest.mark.parametrize("cid", list(CASE_BY_ID))
def test_vq_conv_layer(cid, conv, monkeypatch):
    c = CASE_BY_ID[cid]
    if conv == "mma" and c.out == "u8":
        pytest.skip("uint8 output is written by the wgmma drain only")
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("LG_CONV_TC", "1" if conv == "tc" else "0")
    x, w, bias, res, _, _ = _operands(c, zlib.crc32(cid.encode()))
    phase = conv == "tc" and c.up == 1
    ref, absconv = _reference(c, x, w, bias, res, phase)
    want_path = c.path if conv == "tc" else 0
    y, path, splits, part, _ = _run_case(c, x, w, bias, res)
    assert path == want_path, (path, want_path)
    assert splits == (c.fused_splits() if conv == "tc" else 0), splits
    what = f"{cid}/{conv}"
    wrong = 0.0
    if c.out == "bf":
        rel, wrong = _check_bf16(y, ref, absconv, what)
        if part is not None:
            _check_partials(part, y, c.cout)
    elif c.out == "f32":
        rel = _check_f32(y, ref, absconv, what)
    else:
        yf, pf, _, _, _ = vq_conv(x, w, bias, c.k, c.up, out="f32")
        assert pf == path
        assert torch.equal(y.cpu(), u8_finish(yf.cpu()).permute(0, 2, 3, 1)), "uint8 drain != torch finishing of the f32 output"
        rel = _check_f32(yf, ref, absconv, what)
        fin = torch.clamp(127.5 * ref + 128.0, 0, 255).floor().permute(0, 2, 3, 1)
        assert (y.double() - fin).abs().max().item() <= 1
    if phase:
        # the mma path runs the real 3x3 bf16(W) on the upsampled input: it rounds different weights
        monkeypatch.setenv("LG_CONV_TC", "0")
        ym, pm, _, _, _ = _run_case(c, x, w, bias, res)
        assert pm == 0
        ref_m, abs_m = _reference(c, x, w, bias, res, False)
        d = (y.double() - ym.double()).abs().permute(0, 3, 1, 2)
        assert (d <= ulp_bf16(ref_m) + 2.0 ** -8 * abs_m).all(), d.max().item()
    print(f"[{what}] path {path} gn_splits {splits} max|y-ref|/absconv 2^{torch.log2(torch.tensor(max(rel, 1e-30))).item():.2f} "
          f"not correctly rounded {wrong:.3%}")


GN_CASES = [c.id for c in CASES if c.gn]


@pytest.mark.gpu
@pytest.mark.parametrize("fuse", [1, 0])
@pytest.mark.parametrize("cid", GN_CASES)
def test_vq_conv_then_group_norm(cid, fuse, monkeypatch):
    """conv -> GroupNorm(32) + swish as run_res hands it over: with LG_GN_FUSE=1 the statistics come from the conv's drain."""
    c = CASE_BY_ID[cid]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("LG_GN_FUSE", str(fuse))
    x, w, bias, res, gamma, beta = _operands(c, zlib.crc32(cid.encode()) + 1)
    y, path, splits, part, yn = _run_case(c, x, w, bias, res, gn=(gamma, beta, 1))
    assert path == c.path and splits == c.fused_splits(bool(fuse)), (path, splits)
    err, wrong = _check_gn(yn, y, gamma, beta, 1, f"{cid}/fuse{fuse}")
    print(f"[{cid}/fuse{fuse}] path {path} gn_splits {splits} gn max err {err:.3g} not correctly rounded {wrong:.3%}")


@pytest.mark.gpu
@pytest.mark.parametrize("budget", [1, 2, 5, 131])
@pytest.mark.parametrize("cid", ["res_256_32", "tcw_1x1_nkb2", "up_512_16", "down_256_32", "tc_cout16"])
def test_conv_cta_budget_is_bit_identical(cid, budget):
    """Persistent CTAs (lg_vq_set_cta_budget) loop over many tiles with the stage ring carried across them: output and drain
    statistics must be bit-identical to one CTA per tile."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    c = CASE_BY_ID[cid]
    x, w, bias, res, _, _ = _operands(c, 7)
    try:
        lib.lg_vq_set_cta_budget(0)
        y0, p0, s0, part0, _ = _run_case(c, x, w, bias, res)
        lib.lg_vq_set_cta_budget(budget)
        y1, p1, s1, part1, _ = _run_case(c, x, w, bias, res)
    finally:
        lib.lg_vq_set_cta_budget(0)
    assert p0 == p1 == c.path and s0 == s1
    assert torch.equal(y0, y1)
    assert (part0 is None and part1 is None) or torch.equal(part0, part1)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 10, 100])
@pytest.mark.parametrize("swish", [1, 0])
@pytest.mark.parametrize("C,HW", [(32, 128 * 128), (64, 64 * 64), (128, 8 * 8), (128, 128 * 128), (256, 32 * 32), (512, 16 * 16),
                                  (512, 8 * 8)])
def test_group_norm_stand_alone(C, HW, swish, offset):
    """|mean| / std of about 0, 10 and 100 per group: the statistics must not lose the variance to cancellation."""
    g = torch.Generator(device="cuda").manual_seed(C * 7 + HW + offset)
    B = 3 if HW <= 32 * 32 else 1
    cpg = C // 32
    sign = torch.randint(0, 2, (32,), device="cuda", generator=g) * 2.0 - 1.0
    mean = (offset * sign).repeat_interleave(cpg)
    scale = torch.exp(0.5 * torch.randn(32, device="cuda", generator=g)).repeat_interleave(cpg)
    x = ((mean + torch.randn(B, HW, C, device="cuda", generator=g)) * scale).bfloat16()
    gamma = 1.0 + 0.5 * torch.randn(C, device="cuda", generator=g)
    beta = 0.5 * torch.randn(C, device="cuda", generator=g)
    y = group_norm(x, gamma, beta, swish)
    err, wrong = _check_gn(y, x, gamma, beta, swish, f"gn C{C} HW{HW} swish{swish} offset{offset}")
    print(f"[gn C{C} HW{HW} swish{swish} offset{offset}] max err {err:.3g} not correctly rounded {wrong:.3%}")
