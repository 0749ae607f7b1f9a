"""One-call parity of the VQ tokenizer's remaining kernels against a float64 reference: the AttnBlock stage by stage, the codebook
lookup + post_quant_conv, the encoder's fp32 conv_in, and the codebook argmin / straight-through output at every codebook_embed_dim.

lg_test_vq_attn runs the decoder's own run_attn on weights packed by its own make_attn; lg_test_vq_lookup and lg_test_vq_conv_in_rgb
run the launchers lg_vq_decode and lg_vq_encode call. The argmin and quant_out kernels are reached through VQModel.quantize_indices and
VQModel.encode on tiny models. Every reference is plain torch in float64 on the GPU, computed from the operands exactly as the kernel
sees them: bf16 activations, bf16(W), and the kernel's own upstream intermediates for each later stage. The bf16 rule ("ulp/2 +
2^-13 absdot, fewer than 1 % off bf16(ref)") and the GroupNorm bound are those of tests/test_vq_layers_gpu.py.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from test_vq_gpu import _check_pixels
from test_vq_layers_gpu import _check_bf16, _check_gn, ulp_bf16

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24     # fp32 unit roundoff


def _a256(n):
    return (n + 255) // 256 * 256


def _check_rows(y, ref, absdot, what):
    """_check_bf16 on row-major [R, Ccol] tensors (y bf16, ref / absdot float64)."""
    return _check_bf16(y.reshape(1, -1, 1, y.shape[-1]), ref.reshape(-1, ref.shape[-1]).t()[None, :, :, None],
                       absdot.reshape(-1, absdot.shape[-1]).t()[None, :, :, None], what)


# ---------------------------------------------------------------------------------------------------------------- AttnBlock
def attn_chunk_images(B, N):
    """The engine's images per score chunk: fp32 S of one chunk stays <= 256 MiB."""
    return max(1, min(B, (256 << 20) // (N * N * 4)))


def vq_attn(x, p, attn_bc=0):
    """lg_test_vq_attn. x bf16 NHWC [B,H,W,C]; p: the checkpoint tensors of one AttnBlock. Returns dict of x (out), hn, qk, vt,
    o, s, p (s / p: the last chunk) and bc (images per chunk)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, H, W, C = x.shape
    N = H * W
    bc = min(attn_bc, B) if attn_bc > 0 else attn_chunk_images(B, N)
    last = B - (B - 1) // bc * bc
    dev = x.device
    out = dict(x=x.clone(), hn=torch.empty(B, N, C, dtype=torch.bfloat16, device=dev),
               qk=torch.empty(B, N, 2 * C, dtype=torch.bfloat16, device=dev), vt=torch.empty(B, C, N, dtype=torch.bfloat16, device=dev),
               o=torch.empty(B, N, C, dtype=torch.bfloat16, device=dev), s=torch.empty(last, N, N, dtype=torch.float32, device=dev),
               p=torch.empty(last, N, N, dtype=torch.bfloat16, device=dev))
    gn_floats = B * max(64, -(-H // 16) * -(-W // 16) * 4) * 64
    nbytes = (_a256(B * N * C * 2) + _a256(B * N * 2 * C * 2) + _a256(B * C * N * 2) + _a256(bc * N * N * 4) + _a256(bc * N * N * 2)
              + _a256(gn_floats * 4))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    P = _lib.ptr
    _lib.check(lib.lg_test_vq_attn(P(out["x"]), B, H, W, C, P(p["norm.weight"]), P(p["norm.bias"]), P(p["q.weight"]), P(p["q.bias"]),
                                   P(p["k.weight"]), P(p["k.bias"]), P(p["v.weight"]), P(p["v.bias"]), P(p["proj_out.weight"]),
                                   P(p["proj_out.bias"]), attn_bc, P(out["hn"]), P(out["qk"]), P(out["vt"]), P(out["o"]), P(out["s"]),
                                   P(out["p"]), P(scratch), ctypes.c_size_t(nbytes), _lib.current_stream(dev)), "lg_test_vq_attn")
    out["bc"] = bc
    return out


# (B, H, W, C, attn_bc)
ATTN_SHAPES = [
    (2, 4, 4, 64, 0),       # N = 16: the tiny golden's shape; P.V K-tail below BK = 64; N < 128 tiles
    (3, 8, 8, 32, 0),       # C = 32: the O GEMM has N = 32
    (2, 12, 12, 128, 0),    # N = 144: M and K tails
    (2, 16, 16, 512, 0),    # VQ-16 decoder mid at 256 px
    (1, 24, 24, 512, 0),    # 384 px
    (2, 32, 32, 512, 0),    # VQ-8 mid at 256 px
    (3, 16, 16, 512, 1),    # chunk loop, one image per chunk
    (3, 16, 16, 512, 2),    # chunk loop with a partial last chunk
    (5, 64, 64, 128, 0),    # the engine's own rule splits 4 + 1
]


def test_attn_chunk_rule_splits_the_largest_case():
    assert attn_chunk_images(5, 64 * 64) == 4 and attn_chunk_images(3, 16 * 16) == 3


def _attn_operands(B, H, W, C, peaky, seed):
    """Scores of std ~3 (peaky) or ~0.3, and one query row (the last image's token 0) whose own key scores ~120: above
    ln(FLT_MAX) = 88.7, so a softmax without its max subtraction overflows. The score comes from a rank-one term a u h*^T / |h*|^2
    added to the q and k weights, h* the float64 GroupNorm output of that token and u a unit vector orthogonal to its q and k without
    the term: q*.k* grows by a^2 = 120 sqrt(C) while other scores move by ~120 / C."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    x = rn(B, H, W, C).bfloat16()
    gamma, beta = 1.0 + 0.2 * rn(C), 0.2 * rn(C)
    sig = (3.0 if peaky else 0.3) ** 0.5           # q, k entries ~ N(0, sig^2) -> q.k / sqrt(C) has std sig^2
    wq, wk = rn(C, C) * sig / C ** 0.5, rn(C, C) * sig / C ** 0.5
    bq, bk = 0.1 * rn(C), 0.1 * rn(C)
    xd = x.double().reshape(B, H * W, C)
    grp = xd[-1].reshape(H * W, 32, C // 32)
    mu, sd = grp.mean(dim=(0, 2)), (grp.var(dim=(0, 2), unbiased=False) + 1e-6).sqrt()
    hstar = ((xd[-1, 0].reshape(32, -1) - mu[:, None]) / sd[:, None]).reshape(C) * gamma.double() + beta.double()
    basis = []
    for t in (wq.double() @ hstar + bq.double(), wk.double() @ hstar + bk.double(), rn(C).double()):
        for e in basis:
            t = t - t.dot(e) * e
        basis.append(F.normalize(t, dim=0))
    u = basis[-1]
    a = (120.0 * C ** 0.5) ** 0.5
    r1 = (a * u[:, None] * hstar[None, :] / hstar.dot(hstar)).float()
    p = {"norm.weight": gamma, "norm.bias": beta, "q.weight": wq + r1, "k.weight": wk + r1, "v.weight": rn(C, C) / C ** 0.5,
         "proj_out.weight": rn(C, C) / C ** 0.5, "q.bias": bq, "k.bias": bk, "v.bias": 0.5 * rn(C), "proj_out.bias": 0.5 * rn(C)}
    return x, {k: (v.reshape(C, C, 1, 1) if v.dim() == 2 else v).contiguous() for k, v in p.items()}


def _bfw(w):
    return w.reshape(w.shape[0], -1).bfloat16().double()


@pytest.mark.parametrize("peaky", [True, False], ids=["std3", "std0.3"])
@pytest.mark.parametrize("B,H,W,C,bc", ATTN_SHAPES, ids=[f"B{b}_{h}x{w}_C{c}_bc{k}" for b, h, w, c, k in ATTN_SHAPES])
def test_vq_attn_block_stage_by_stage(B, H, W, C, bc, peaky):
    N = H * W
    x, p = _attn_operands(B, H, W, C, peaky, seed=B * 1000 + N + C + bc + peaky)
    r = vq_attn(x, p, bc)
    what = f"attn B{B} {H}x{W} C{C} bc{bc} {'peaky' if peaky else 'flat'}"
    # hn: the GroupNorm bound of test_vq_layers_gpu (one bf16 ulp + 2^-16 |gamma| (1 + |mu| / sigma))
    _check_gn(r["hn"], x, p["norm.weight"], p["norm.bias"], 0, what + " hn")
    hn = r["hn"].double().reshape(B * N, C)
    # q | k: bf16 GEMM bound against hn @ bf16(W)^T + b; the halves are checked against their own weights
    for half, name in ((0, "q"), (1, "k")):
        w, b = _bfw(p[f"{name}.weight"]), p[f"{name}.bias"].double()
        ref, absdot = hn @ w.t() + b, hn.abs() @ w.abs().t() + b.abs()
        _check_rows(r["qk"].reshape(B * N, 2 * C)[:, half * C:(half + 1) * C], ref, absdot, f"{what} {name}")
    # V^T [B, C, N]: bias added per row (channel)
    wv, bv = _bfw(p["v.weight"]), p["v.bias"].double()
    hb = r["hn"].double()
    ref = torch.einsum("cd,bnd->bcn", wv, hb) + bv[None, :, None]
    absdot = torch.einsum("cd,bnd->bcn", wv.abs(), hb.abs()) + bv.abs()[None, :, None]
    _check_rows(r["vt"].reshape(B * C, N), ref.reshape(B * C, N), absdot.reshape(B * C, N), what + " vt")
    q = r["qk"].double()[..., :C]
    k = r["qk"].double()[..., C:]
    v = r["vt"].double()
    scale = C ** -0.5
    # s (last chunk): fp32 accumulation of a bf16 dot product, |s - C^-1/2 q.k| <= 2^-13 C^-1/2 |q|.|k|
    last = r["s"].shape[0]
    ql, kl = q[B - last:], k[B - last:]
    s_ref = scale * ql @ kl.transpose(1, 2)
    s_abs = scale * ql.abs() @ kl.abs().transpose(1, 2)
    err = (r["s"].double() - s_ref).abs()
    assert (err <= 2.0 ** -13 * s_abs).all(), f"{what} s: max err / bound {(err / (2.0 ** -13 * s_abs)).max().item():.3g}"
    assert r["s"][-1, 0].max().item() > 89.0, "operand design: the planted score must exceed ln(FLT_MAX)"
    # p (last chunk): softmax of the kernel's own fp32 scores, rounded to bf16; __expf is within 2^-17 relative at |s| <= 128, and
    # results below 2^-126 flush to zero
    p_ref = torch.softmax(r["s"].double(), dim=-1)
    pk = r["p"].double()
    perr = (pk - p_ref.bfloat16().double()).abs()
    pbound = ulp_bf16(torch.maximum(p_ref, pk)) + 2.0 ** -126
    assert (perr <= pbound).all(), f"{what} p: {(perr > pbound).sum().item()} elements off by more than one bf16 ulp"
    same = (pk == p_ref.bfloat16().double()).double().mean().item()
    assert same >= 0.99, f"{what} p: {same:.2%} bit-equal to bf16(softmax)"
    rows = pk.sum(-1)
    assert ((rows - 1).abs() <= N * 2.0 ** -9).all(), (rows - 1).abs().max().item()
    # o (every image, every chunk): float64 softmax(C^-1/2 q k^T) v from the kernel's q, k, v. P rounded to bf16 plus __expf moves
    # each weight by < 2^-8 relative; the fp32 P.V accumulation adds 2^-13 (p.|v|); the bf16 store ulp(o) / 2
    pr = torch.softmax(scale * q @ k.transpose(1, 2), dim=-1)
    o_ref = pr @ v.transpose(1, 2)
    pv = pr @ v.abs().transpose(1, 2)
    oerr = (r["o"].double() - o_ref).abs()
    obound = (2.0 ** -8 + 2.0 ** -13) * pv + 0.5 * ulp_bf16(o_ref)
    assert (oerr <= obound).all(), (f"{what} o: {(oerr > obound).sum().item()} of {oerr.numel()} outside the bound, "
                                    f"worst image {(oerr - obound).amax(dim=(1, 2)).argmax().item()}")
    # x out = x + proj_out(o): the 1x1 conv + residual bound against the kernel's own o
    o = r["o"].double().reshape(B * N, C)
    wp, bp = _bfw(p["proj_out.weight"]), p["proj_out.bias"].double()
    xd = x.double().reshape(B * N, C)
    ref = xd + o @ wp.t() + bp
    absdot = xd.abs() + o.abs() @ wp.abs().t() + bp.abs()
    _check_rows(r["x"].reshape(B * N, C), ref, absdot, what + " x")


@pytest.mark.parametrize("B,H,W,C,chunks", [(3, 16, 16, 512, (1, 2)), (5, 64, 64, 128, (1, 5))])
def test_vq_attn_chunking_is_bit_identical(B, H, W, C, chunks):
    """Every image runs the same tiles and K loop whatever chunk it falls in: any difference between chunkings is a bug."""
    x, p = _attn_operands(B, H, W, C, True, seed=77)
    base = vq_attn(x, p, 0)
    for bc in chunks:
        r = vq_attn(x, p, bc)
        assert r["bc"] == bc != base["bc"]
        for key in ("x", "hn", "qk", "vt", "o"):
            assert torch.equal(r[key], base[key]), (bc, key)
        last = min(r["s"].shape[0], base["s"].shape[0])     # both hold the scores of the last `last` images
        assert torch.equal(r["s"][-last:], base["s"][-last:]) and torch.equal(r["p"][-last:], base["p"][-last:]), bc


# ----------------------------------------------------------------------------------------------------- lookup + post_quant_conv
def vq_lookup(codes, cb, l2, w, b):
    from llamagen_b200 import _lib
    lib = _lib.load()
    n_e, ed = cb.shape
    Z = w.shape[0]
    cb_out = torch.empty_like(cb)
    sq = torch.empty(n_e, dtype=torch.float32, device=cb.device)
    out = torch.empty(codes.numel(), Z, dtype=torch.bfloat16, device=cb.device)
    P = _lib.ptr
    _lib.check(lib.lg_test_vq_lookup(P(codes), codes.numel(), P(cb), n_e, ed, int(l2), P(w), P(b), Z, P(cb_out), P(sq), P(out),
                                     _lib.current_stream(cb.device)), "lg_test_vq_lookup")
    torch.cuda.synchronize()
    return cb_out, sq, out


@pytest.mark.parametrize("Z", [32, 256])
@pytest.mark.parametrize("l2", [0, 1])
@pytest.mark.parametrize("ed", [4, 8, 16, 32])
def test_vq_lookup_postquant(ed, l2, Z):
    g = torch.Generator(device="cuda").manual_seed(ed * 10 + l2 * 3 + Z)
    n_e = 1000
    cb = torch.randn(n_e, ed, device="cuda", generator=g) * 0.7
    cb[3] = 0.0                                              # F.normalize's eps path: stays zero
    codes = torch.randint(0, n_e, (300,), device="cuda", generator=g, dtype=torch.int32)
    codes[:3] = torch.tensor([0, n_e - 1, 3], dtype=torch.int32)
    w = (torch.randn(Z, ed, 1, 1, device="cuda", generator=g) / ed ** 0.5).contiguous()
    b = 0.5 * torch.randn(Z, device="cuda", generator=g)
    cb_out, sq, out = vq_lookup(codes, cb, l2, w, b)
    # normalised rows: the fp32 sum of ed squares is off by <= ed u, its square root by half that, the division by u more:
    # (ed / 2 + 2) u relative, and sq (a sum of ed squares of those) by (2 ed + 4) u; never looser than 2^-21 is needed below ed = 8
    cd = cb.double()
    if l2:
        ref = F.normalize(cd, dim=-1)
        assert ((cb_out.double() - ref).abs() <= max(2.0 ** -21, (ed / 2 + 2) * U32) * ref.abs()).all()
        sq_tol = max(2.0 ** -21, (2 * ed + 4) * U32)
    else:
        ref = cd
        assert torch.equal(cb_out, cb)
        sq_tol = max(2.0 ** -21, ed * U32)
    sq_ref = (ref * ref).sum(-1)
    assert ((sq.double() - sq_ref).abs() <= sq_tol * sq_ref).all(), ((sq.double() - sq_ref).abs() / sq_ref.clamp_min(1e-30)).max()
    assert cb_out[3].abs().max().item() == 0 and sq[3].item() == 0
    # rows through post_quant_conv in fp32: the bf16 rule with absdot = |b| + sum |e| |w|
    e = cb_out.double()[codes.long()]
    wd = w.double().reshape(Z, ed)
    _check_rows(out, e @ wd.t() + b.double(), e.abs() @ wd.abs().t() + b.double().abs(), f"lookup ed{ed} l2{l2} Z{Z}")


# --------------------------------------------------------------------------------------------------------------- conv_in_rgb
def vq_conv_in_rgb(x, w, b):
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, _, H, W = x.shape
    ch = w.shape[0]
    out = torch.empty(B, H, W, ch, dtype=torch.bfloat16, device=x.device)
    _lib.check(lib.lg_test_vq_conv_in_rgb(_lib.ptr(x), B, H, W, _lib.ptr(w), _lib.ptr(b), ch, _lib.ptr(out),
                                          _lib.current_stream(x.device)), "lg_test_vq_conv_in_rgb")
    torch.cuda.synchronize()
    return out


CONV_IN_CASES = [(2, h, w, ch) for ch in (32, 64, 128) for h, w in ((4, 4), (8, 12), (256, 256))] + [
    (2, 384, 384, 128),     # 1.18 M items over a grid capped at 132 * 8 CTAs (270,336 threads): several grid-stride passes
]


@pytest.mark.parametrize("B,H,W,ch", CONV_IN_CASES, ids=[f"B{b}_{h}x{w}_ch{c}" for b, h, w, c in CONV_IN_CASES])
def test_vq_conv_in_rgb(B, H, W, ch):
    g = torch.Generator(device="cuda").manual_seed(H * 7 + W + ch)
    x = torch.rand(B, 3, H, W, device="cuda", generator=g) * 2 - 1
    big = 20.0 * torch.randn(B, 3, H, W, device="cuda", generator=g)   # border rows and columns: a padding or edge error shows
    for sl in ((slice(None), slice(None), 0), (slice(None), slice(None), -1),
               (slice(None), slice(None), slice(None), 0), (slice(None), slice(None), slice(None), -1)):
        x[sl] = big[sl]
    w = torch.randn(ch, 3, 3, 3, device="cuda", generator=g) / 27 ** 0.5
    b = 0.5 * torch.randn(ch, device="cuda", generator=g)
    y = vq_conv_in_rgb(x.contiguous(), w, b)
    wd = w.double()
    ref = F.conv2d(x.double(), wd, b.double(), padding=1)
    absconv = F.conv2d(x.double().abs(), wd.abs(), b.double().abs(), padding=1)
    # 27 fp32 FMAs after the bias: |y - ref| <= 27 u absconv < 2^-18 absconv before the bf16 store (ulp / 2)
    err = (y.double().permute(0, 3, 1, 2) - ref).abs()
    bound = 0.5 * ulp_bf16(ref) + 2.0 ** -18 * absconv
    assert (err <= bound).all(), f"{(err > bound).sum().item()} outside the bound at {(err > bound).nonzero()[:4].tolist()}"
    wrong = (y.double().permute(0, 3, 1, 2) != ref.bfloat16().double()).double().mean().item()
    assert wrong < 0.01, f"{wrong:.2%} of elements not correctly rounded"


# ------------------------------------------------------------------------------------------------------------------ argmin
def _tiny_vq(ed, l2, n_e, cb):
    from llamagen_b200.vq_model import ModelArgs, VQModel
    torch.manual_seed(ed * 100 + n_e + l2)
    m = VQModel(ModelArgs(codebook_size=n_e, codebook_embed_dim=ed, codebook_l2_norm=bool(l2), encoder_ch_mult=[1, 2],
                          decoder_ch_mult=[1, 2], z_channels=32), ch=32)
    m.quantize.embedding.weight.data.copy_(cb)
    return m.cuda().eval()


ARGMIN_TILES = (1024, 2048)     # codebook rows per shared-memory tile: 1024 at ED = 32, 2048 below
ARGMIN_NE = sorted({1, 100, 16384} | {t + d for t in ARGMIN_TILES for d in (-1, 0, 1)})


def _dup_pairs(n_e):
    """(a, b), a < b: row b is made a bitwise copy of row a. One pair ends near the top; one straddles each tile boundary below it."""
    if n_e < 4:
        return []
    return [(1, n_e - 2)] + [(t - 1, t) for t in ARGMIN_TILES if t + 1 < n_e - 2]


@pytest.mark.parametrize("n_e", ARGMIN_NE)
@pytest.mark.parametrize("l2", [0, 1])
@pytest.mark.parametrize("ed", [4, 8, 16, 32])
def test_vq_argmin(ed, l2, n_e):
    g = torch.Generator().manual_seed(ed * 7 + l2 + n_e)
    cb = torch.randn(n_e, ed, generator=g)
    pairs = _dup_pairs(n_e)
    for a, b in pairs:
        cb[b] = cb[a]
    B, gs = 3, 7                                   # 147 latents: not a multiple of the 128-thread block
    z = torch.randn(B, gs * gs, ed, generator=g)
    # planted latents (l2: the row scaled by 2, the same direction): the last row, the first row, and every duplicated row
    plant = [n_e - 1, 0] + [a for a, _ in pairs]
    for i, row in enumerate(plant):
        z[0, i] = cb[row] * (2.0 if l2 else 1.0)
    z = z.reshape(B, gs, gs, ed).permute(0, 3, 1, 2).contiguous()
    m = _tiny_vq(ed, l2, n_e, cb)
    idx = m.quantize_indices(z.cuda())
    zf = z.cuda().double().permute(0, 2, 3, 1).reshape(-1, ed)
    e = cb.cuda().double()
    if l2:
        zf, e = F.normalize(zf, dim=-1), F.normalize(e, dim=-1)
    d = (zf * zf).sum(1, keepdim=True) + (e * e).sum(1) - 2 * zf @ e.t()
    # fp32 error of (|z|^2 + |e|^2) - 2 z.e with z, e normalised in fp32 (each within (ed/2 + 2) u relative) and ed-term fp32 sums:
    # below (4 ed + 8) u (|z| + |e|)^2 for every pair; eps takes the largest |e| of the codebook
    eps = (4 * ed + 8) * U32 * (zf.norm(dim=1) + e.norm(dim=1).max()) ** 2
    chosen = d.gather(1, idx[:, None]).squeeze(1)
    top = d.topk(min(2, n_e), dim=1, largest=False).values
    assert ((chosen - top[:, 0]) <= 2 * eps).all(), f"ED{ed} l2{l2} n_e{n_e}: a chosen code is not within 2 eps of the minimum"
    clear = (top[:, 1] - top[:, 0] > 2 * eps) if n_e > 1 else torch.ones_like(eps, dtype=torch.bool)
    assert torch.equal(idx[clear], d.argmin(1)[clear]), f"ED{ed} l2{l2} n_e{n_e}: {(idx[clear] != d.argmin(1)[clear]).sum()} wrong"
    assert clear.double().mean().item() > 0.5
    # duplicated rows tie bitwise: the lowest index wins, like torch.argmin
    want = torch.tensor(plant, device=idx.device)
    assert torch.equal(idx[:len(plant)], want), (idx[:len(plant)].tolist(), plant)


# --------------------------------------------------------------------------------------- quant_out and whole models at every ED
@pytest.mark.parametrize("l2", [0, 1])
@pytest.mark.parametrize("ed", [4, 16, 32])
def test_tiny_model_encode_and_decode_at_embed_dim(ed, l2):
    from oracle import VQOracle
    g = torch.Generator().manual_seed(ed + l2)
    n_e = 64
    cb = torch.randn(n_e, ed, generator=g) * 0.2
    m = _tiny_vq(ed, l2, n_e, F.normalize(cb, dim=-1) if l2 else cb)
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    orc = VQOracle(sd, ch_mult=(1, 2), l2_norm=bool(l2))
    x = torch.rand(2, 3, 16, 16, generator=g) * 2 - 1
    quant, _, (_, _, idx), z = m.encode(x.cuda(), return_z=True)
    q_own, idx_own = orc.quantize(z.cpu())
    assert torch.equal(idx.cpu(), idx_own)
    assert torch.allclose(quant.cpu(), q_own, atol=2e-6, rtol=0), (quant.cpu() - q_own).abs().max().item()
    codes = idx.reshape(2, 64)
    out = m.decode_code(codes, [2, ed, 8, 8]).cpu()
    ref = orc.decode_code(codes.cpu(), [2, ed, 8, 8])
    assert tuple(out.shape) == tuple(ref.shape)
    _check_pixels(out, ref)
