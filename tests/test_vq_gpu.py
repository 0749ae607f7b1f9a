"""GPU parity of the VQ decode path (lg_vq_decode) and the codebook argmin (lg_vq_argmin).

Tolerance (stated, SURVEY §8c): the sm_90a decoder feeds bf16 operands to the tensor cores with fp32
accumulation and keeps activations in bf16; the oracle's own bf16-vs-fp32 spread on this decoder is
max-abs 0.146 / mean-abs 0.010 at output std 0.39, so we require max-abs <= 0.2 and mean-abs <= 0.02
against the fp32 oracle, and <= 1 LSB mean error after the uint8 conversion of sample_c2i_ddp.py:143."""
import pytest
import torch

from oracle import VQOracle
from util import load_golden

pytestmark = pytest.mark.gpu


def _check_pixels(out, ref):
    scale = max(1.0, ref.std().item() / 0.39)
    err = (out - ref).abs()
    assert err.max().item() <= 0.2 * scale, err.max().item()
    assert err.mean().item() <= 0.02 * scale, err.mean().item()
    u8 = lambda x: torch.clamp(127.5 * x + 128.0, 0, 255).to(torch.uint8).float()
    assert (u8(out) - u8(ref)).abs().mean().item() <= 1.0 * scale


def _tiny_model(g):
    from llamagen_b200.vq_model import ModelArgs, VQModel
    m = VQModel(ModelArgs(codebook_size=64, codebook_embed_dim=8, encoder_ch_mult=g["ch_mult"], decoder_ch_mult=g["ch_mult"],
                          z_channels=g["z_channels"]), ch=g["ch"])
    missing, unexpected = m.load_state_dict(g["state_dict"], strict=False)
    assert not unexpected and all(k.startswith(("encoder.", "quant_conv.", "quantize.codebook_used")) for k in missing)
    return m.cuda().eval()


def test_tiny_decoder_matches_reference_golden():
    g = load_golden("vq_tiny.pt")
    m = _tiny_model(g)
    out = m.decode_code(g["codes"].cuda(), [2, 8, 4, 4]).cpu()
    assert tuple(out.shape) == tuple(g["pixels"].shape)
    _check_pixels(out, g["pixels"])


def test_tiny_argmin_matches_reference_golden():
    g = load_golden("vq_tiny.pt")
    m = _tiny_model(g)
    idx = m.quantize_indices(g["z"].cuda()).cpu()
    assert torch.equal(idx, g["argmin"])


@pytest.mark.parametrize("conv", ["tcgen05", "mma"])
@pytest.mark.parametrize("name,g,B", [("VQ-16", 16, 3), ("VQ-16", 24, 1), ("VQ-8", 16, 2)])
def test_full_decoder_vs_oracle(name, g, B, conv, monkeypatch):
    """conv=tcgen05 (test id kept stable): TMA 4-D box + wgmma implicit GEMM (conv_tc.cu, incl. the 2x2 phase form of upsample+conv and
    24x24 grids whose 8x16 patches overhang the image); conv=mma: the mma.sync + cp.async gather path."""
    monkeypatch.setenv("LG_CONV_TC", "1" if conv == "tcgen05" else "0")
    from llamagen_b200 import VQ_models
    torch.manual_seed(g + B)
    m = VQ_models[name](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    codes = torch.randint(0, 16384, (B, g * g))
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    ref = VQOracle(sd, ch_mult=m.config.decoder_ch_mult).decode_code(codes, [B, 8, g, g])
    out = m.decode_code(codes.cuda(), [B, 8, g, g]).cpu()
    assert tuple(out.shape) == tuple(ref.shape)
    _check_pixels(out, ref)


@pytest.mark.parametrize("variant", ["n128_tiles", "persistent_8_ctas", "no_gn_fuse", "cta_budget_api"])
def test_conv_kernel_variants_agree(variant, monkeypatch):
    """The shipped decoder = weights-as-A convs (wgmma N = 256, conv_tcw_kernel) with the GroupNorm statistics in their drain. It must
    agree with: the pixels-as-A kernel (N <= 128), the same kernels looping as 8 or 5 persistent CTAs (C-ABI CTA budget; many tiles per
    CTA: ring / accumulator phases carried across tiles) and the stand-alone statistics pass. Same bf16 rounding points everywhere;
    only fp32 summation orders differ."""
    from llamagen_b200 import VQ_models, _lib
    torch.manual_seed(5)
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    codes = torch.randint(0, 16384, (2, 256), device="cuda")
    base = m.decode_code(codes, [2, 8, 16, 16]).cpu()
    if variant == "n128_tiles":
        monkeypatch.setenv("LG_CONV_SWAP", "0")
    elif variant == "persistent_8_ctas":
        _lib.load().lg_vq_set_cta_budget(8)
    elif variant == "no_gn_fuse":
        monkeypatch.setenv("LG_GN_FUSE", "0")
    else:
        _lib.load().lg_vq_set_cta_budget(5)
    try:
        out = m.decode_code(codes, [2, 8, 16, 16]).cpu()
    finally:
        _lib.load().lg_vq_set_cta_budget(0)
    err = (out - base).abs()
    if variant in ("persistent_8_ctas", "cta_budget_api"):
        assert torch.equal(out, base)                        # same tiles, same arithmetic, only the CTA -> tile map changes
    else:
        # two bf16 decoders that differ in fp32 summation order: bounded like the oracle's own bf16-vs-fp32 spread (0.146 / 0.010);
        # measured 0.116 / 0.0073 between the N = 128 and N = 256 kernels
        assert err.max().item() <= 0.2 and err.mean().item() <= 0.015, (err.max().item(), err.mean().item())


def test_decode_is_batch_invariant():
    """Images are independent (replica sharding relies on it): decoding a batch == decoding its halves."""
    from llamagen_b200 import VQ_models
    torch.manual_seed(0)
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    codes = torch.randint(0, 16384, (4, 256), device="cuda")
    full = m.decode_code(codes, [4, 8, 16, 16])
    a = m.decode_code(codes[:2], [2, 8, 16, 16])
    b = m.decode_code(codes[2:], [2, 8, 16, 16])
    assert torch.equal(full, torch.cat([a, b]))


def test_argmin_full_codebook_vs_oracle():
    from llamagen_b200 import VQ_models
    torch.manual_seed(1)
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    m.quantize.embedding.weight.data.copy_(torch.nn.functional.normalize(torch.randn(16384, 8), dim=-1))
    z = torch.randn(4, 8, 16, 16)
    orc = VQOracle({k: v.cpu() for k, v in m.state_dict().items()}, ch_mult=m.config.decoder_ch_mult)
    ref = orc.argmin_indices(z)
    idx = m.quantize_indices(z.cuda()).cpu()
    if not torch.equal(idx, ref):
        # a mismatch is only acceptable on an fp32 near-tie of the two distances
        e = torch.nn.functional.normalize(m.quantize.embedding.weight.data.cpu(), dim=-1)
        zf = torch.nn.functional.normalize(z.permute(0, 2, 3, 1).reshape(-1, 8), dim=-1)
        bad = (idx != ref).nonzero().view(-1)
        assert bad.numel() <= 4
        d = ((zf[bad, None, :] - e[None, :, :]) ** 2).sum(-1)
        gap = (d.gather(1, idx[bad, None]) - d.gather(1, ref[bad, None])).abs().max().item()
        assert gap <= 1e-6, gap


# ------------------------------------------------------------------------------------------------ encode (SURVEY §8 f-2)
# Tolerance (stated): the oracle's own bf16-vs-fp32 spread on the VQ-16 encoder output z (random init, z std 0.185) is
# max-abs 0.0145 / mean-abs 0.0029 and its argmin indices agree on 92 % of positions. We require max-abs <= 0.02 and
# mean-abs <= 0.004 (scaled by z std / 0.185) against the fp32 oracle, >= 85 % identical indices, every differing index
# to be a near-tie under the ORACLE's distances, and bit-exact indices given our own z (the integer part of the path).
def _check_encode(m, x, orc):
    quant, losses, info, z = m.encode(x.cuda(), return_z=True)
    idx = info[2].cpu()
    z = z.cpu()
    assert losses == (None, None, None, 0) and info[0] is None and info[1] is None
    z_ref = orc.encode_z(x)
    q_ref, idx_ref = orc.quantize(z_ref)
    scale = max(1e-3, z_ref.std().item() / 0.185)
    err = (z - z_ref).abs()
    assert err.max().item() <= 0.02 * scale, (err.max().item(), scale)
    assert err.mean().item() <= 0.004 * scale, (err.mean().item(), scale)
    # integer part: argmin of OUR z through the oracle must be bit-identical, and the returned tensor must be its quantisation
    q_own, idx_own = orc.quantize(z)
    assert torch.equal(idx, idx_own)
    assert torch.allclose(quant.cpu(), q_own, atol=2e-6, rtol=0)
    assert tuple(quant.shape) == tuple(q_ref.shape) and idx.dtype == torch.int64
    agree = (idx == idx_ref).float().mean().item()
    assert agree >= 0.85, agree
    # every disagreement is a near-tie in the oracle's own distance matrix
    e = orc.codebook()
    zf = torch.nn.functional.normalize(z_ref.permute(0, 2, 3, 1).reshape(-1, z_ref.shape[1]), dim=-1) if orc.l2_norm \
        else z_ref.permute(0, 2, 3, 1).reshape(-1, z_ref.shape[1])
    d = (zf ** 2).sum(1, keepdim=True) + (e ** 2).sum(1) - 2 * zf @ e.t()
    gap = d.gather(1, idx[:, None]) - d.gather(1, idx_ref[:, None])
    assert gap.max().item() <= 0.2 * scale, gap.max().item()
    return agree


def test_tiny_encoder_matches_reference_golden():
    g = load_golden("vq_enc_tiny.pt")
    from llamagen_b200.vq_model import ModelArgs, VQModel
    m = VQModel(ModelArgs(codebook_size=64, codebook_embed_dim=8, encoder_ch_mult=g["ch_mult"], decoder_ch_mult=g["ch_mult"],
                          z_channels=g["z_channels"]), ch=g["ch"])
    missing, unexpected = m.load_state_dict(g["state_dict"], strict=False)
    assert not unexpected
    m = m.cuda().eval()
    orc = VQOracle(g["state_dict"], ch_mult=g["ch_mult"])
    assert torch.equal(orc.encode_z(g["x"]), g["z"])            # the checker itself is pinned to the reference output
    _check_encode(m, g["x"], orc)


@pytest.mark.parametrize("conv", ["tcgen05", "mma"])
@pytest.mark.parametrize("name,size,B", [("VQ-16", 256, 2), ("VQ-8", 128, 1), ("VQ-16", 384, 1)])
def test_full_encoder_vs_oracle(name, size, B, conv, monkeypatch):
    monkeypatch.setenv("LG_CONV_TC", "1" if conv == "tcgen05" else "0")
    from llamagen_b200 import VQ_models
    torch.manual_seed(size + B)
    m = VQ_models[name](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    x = torch.rand(B, 3, size, size) * 2 - 1
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    _check_encode(m, x, VQOracle(sd, ch_mult=m.config.encoder_ch_mult))


def test_encode_is_batch_invariant_and_feeds_decode():
    """extract_codes_c2i.py:103 / vq_demo.py:59-61: encode -> indices -> decode_code; images are independent."""
    from llamagen_b200 import VQ_models
    torch.manual_seed(3)
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    x = torch.rand(4, 3, 256, 256, device="cuda") * 2 - 1
    _, _, (_, _, idx) = m.encode(x)
    _, _, (_, _, a) = m.encode(x[:2])
    _, _, (_, _, b) = m.encode(x[2:])
    assert torch.equal(idx, torch.cat([a, b]))
    pix = m.decode_code(idx.reshape(4, -1), [4, 8, 16, 16])
    assert tuple(pix.shape) == (4, 3, 256, 256) and torch.isfinite(pix).all()


def test_encode_rejects_bad_shapes():
    from llamagen_b200 import VQ_models
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    with pytest.raises(ValueError):
        m.encode(torch.zeros(1, 3, 250, 250))
    with pytest.raises(ValueError):
        m.encode(torch.zeros(1, 3, 256, 128))


# ------------------------------------------------------------------------------------------------ pixel finishing (§8 f-1)
@pytest.mark.parametrize("w", [48, 50])      # 4-pixel vector path / scalar fallback
def test_pixels_to_uint8_is_bit_exact(w):
    from llamagen_b200.postprocess import to_uint8_nhwc
    torch.manual_seed(0)
    x = torch.randn(3, 3, 64, w) * 0.8
    x[0, 0, 0, :4] = torch.tensor([-1.0, 1.0, -1.0039216, 0.99607843])
    ref = torch.clamp(127.5 * x + 128.0, 0, 255).permute(0, 2, 3, 1).to(torch.uint8)      # sample_c2i_ddp.py:143
    out = to_uint8_nhwc(x.cuda()).cpu()
    assert out.dtype == torch.uint8 and torch.equal(out, ref)


@pytest.mark.parametrize("src,dst", [(384, 256), (512, 256), (96, 128), (40, 30)])
def test_pixels_bicubic_resize_matches_torch(src, dst):
    """F.interpolate(mode='bicubic') of sample_c2i_ddp.py:141-142 fused with the uint8 conversion. Float tolerance: the
    tap sums are fp32 in a different association order than ATen's, so a pixel may land on the other side of an integer
    boundary: require |diff| <= 1 LSB everywhere and < 0.5 % of values off by one."""
    import torch.nn.functional as F
    from llamagen_b200.postprocess import to_uint8_nhwc
    torch.manual_seed(src)
    x = torch.randn(2, 3, src, src) * 0.7
    ref = torch.clamp(127.5 * F.interpolate(x, size=(dst, dst), mode="bicubic") + 128.0, 0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    out = to_uint8_nhwc(x.cuda(), size=dst).cpu()
    diff = (out.int() - ref.int()).abs()
    assert diff.max().item() <= 1
    assert (diff != 0).float().mean().item() < 5e-3


@pytest.mark.parametrize("name,g", [("VQ-16", 16), ("VQ-8", 16)])
def test_decode_code_uint8_equals_decode_then_finishing(name, g):
    """SURVEY §8 f-1: the uint8/NHWC conversion inside conv_out's accumulator drain (lg_vq_decode_u8) must give the same BYTES as
    decode_code followed by the reference's finishing `clamp(127.5*x+128, 0, 255).permute(0,2,3,1).to(uint8)`
    (sample_c2i_ddp.py:141-143) applied to our own fp32 pixels — the arithmetic per pixel is identical."""
    from llamagen_b200 import VQ_models
    torch.manual_seed(3)
    vq = VQ_models[name](codebook_size=16384, codebook_embed_dim=8).to("cuda").eval()
    codes = torch.randint(0, 16384, (3, g * g), device="cuda")
    shape = [3, 8, g, g]
    pix = vq.decode_code(codes, shape)
    want = torch.clamp(127.5 * pix + 128.0, 0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    got = vq.decode_code_uint8(codes, shape)
    assert got.dtype == torch.uint8 and tuple(got.shape) == tuple(want.shape)
    assert torch.equal(got, want)
