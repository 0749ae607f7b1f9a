"""Host-side mirror of the reference VQ tokenizer interface (tokenizer/tokenizer_image/vq_model.py).

A parameter container with the reference's state_dict names/shapes (so `load_state_dict(ckpt["model"])`
of a LlamaGen tokenizer checkpoint works unchanged, strict=True included), the `VQ_models` registry
(vq_model.py:418-424) and `decode_code` (vq_model.py:52-55) executed by the sm_90a implicit-GEMM
decoder behind the C-ABI (lg_vq_decode).  The encode-side argmin-L2 (vq_model.py:215-233) is exposed
as `quantize_indices` (lg_vq_argmin).  The conv encoder itself is the next-tier row of SURVEY §8(f).
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, field
from typing import List

import torch
import torch.nn as nn

from . import _lib


@dataclass
class ModelArgs:
    # same fields / defaults as vq_model.py:12-24
    codebook_size: int = 16384
    codebook_embed_dim: int = 8
    codebook_l2_norm: bool = True
    codebook_show_usage: bool = True
    commit_loss_beta: float = 0.25
    entropy_loss_ratio: float = 0.0
    encoder_ch_mult: List[int] = field(default_factory=lambda: [1, 1, 2, 2, 4])
    decoder_ch_mult: List[int] = field(default_factory=lambda: [1, 1, 2, 2, 4])
    z_channels: int = 256
    dropout_p: float = 0.0


def _conv(cout, cin, k):
    return [("weight", (cout, cin, k, k)), ("bias", (cout,))]


def _norm(c):
    return [("weight", (c,)), ("bias", (c,))]


def _res_spec(prefix, cin, cout):
    out = []
    for sub, spec in (("norm1", _norm(cin)), ("conv1", _conv(cout, cin, 3)), ("norm2", _norm(cout)),
                      ("conv2", _conv(cout, cout, 3))):
        out += [(f"{prefix}.{sub}.{n}", s) for n, s in spec]
    if cin != cout:
        out += [(f"{prefix}.nin_shortcut.{n}", s) for n, s in _conv(cout, cin, 1)]
    return out


def _attn_spec(prefix, c):
    out = [(f"{prefix}.norm.{n}", s) for n, s in _norm(c)]
    for sub in ("q", "k", "v", "proj_out"):
        out += [(f"{prefix}.{sub}.{n}", s) for n, s in _conv(c, c, 1)]
    return out


def decoder_spec(ch, ch_mult, z_channels, num_res_blocks=2, out_channels=3):
    """(name, shape) list of Decoder parameters in the reference's order (vq_model.py:128-171)."""
    n = len(ch_mult)
    block_in = ch * ch_mult[-1]
    spec = [(f"conv_in.{k}", s) for k, s in _conv(block_in, z_channels, 3)]
    spec += _res_spec("mid.0", block_in, block_in) + _attn_spec("mid.1", block_in) + _res_spec("mid.2", block_in, block_in)
    for bi, i_level in enumerate(reversed(range(n))):
        block_out = ch * ch_mult[i_level]
        for j in range(num_res_blocks + 1):
            spec += _res_spec(f"conv_blocks.{bi}.res.{j}", block_in, block_out)
            block_in = block_out
            if i_level == n - 1:
                spec += _attn_spec(f"conv_blocks.{bi}.attn.{j}", block_in)
        if i_level != 0:
            spec += [(f"conv_blocks.{bi}.upsample.conv.{k}", s) for k, s in _conv(block_in, block_in, 3)]
    spec += [(f"norm_out.{k}", s) for k, s in _norm(block_in)]
    spec += [(f"conv_out.{k}", s) for k, s in _conv(out_channels, block_in, 3)]
    return spec


def encoder_spec(ch, ch_mult, z_channels, num_res_blocks=2, in_channels=3):
    """(name, shape) list of Encoder parameters (vq_model.py:64-104) — held for checkpoint compatibility."""
    n = len(ch_mult)
    in_mult = (1,) + tuple(ch_mult)
    spec = [(f"conv_in.{k}", s) for k, s in _conv(ch, in_channels, 3)]
    block_in = ch
    for i in range(n):
        block_in, block_out = ch * in_mult[i], ch * ch_mult[i]
        for j in range(num_res_blocks):
            spec += _res_spec(f"conv_blocks.{i}.res.{j}", block_in, block_out)
            block_in = block_out
            if i == n - 1:
                spec += _attn_spec(f"conv_blocks.{i}.attn.{j}", block_in)
        if i != n - 1:
            spec += [(f"conv_blocks.{i}.downsample.conv.{k}", s) for k, s in _conv(block_in, block_in, 3)]
    spec += _res_spec("mid.0", block_in, block_in) + _attn_spec("mid.1", block_in) + _res_spec("mid.2", block_in, block_in)
    spec += [(f"norm_out.{k}", s) for k, s in _norm(block_in)]
    spec += [(f"conv_out.{k}", s) for k, s in _conv(z_channels, block_in, 3)]
    return spec


class _Group(nn.Module):
    pass


def _install(root: nn.Module, dotted: str, tensor: torch.Tensor):
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            setattr(mod, p, _Group())
        mod = getattr(mod, p)
    setattr(mod, parts[-1], nn.Parameter(tensor, requires_grad=False))


def _init_tensor(name, shape):
    if len(shape) == 4:                       # torch Conv2d default: U(-1/sqrt(fan_in), 1/sqrt(fan_in))
        bound = 1.0 / math.sqrt(shape[1] * shape[2] * shape[3])
        return torch.empty(shape).uniform_(-bound, bound)
    if ".norm" in name or name.startswith("norm"):
        return torch.ones(shape) if name.endswith("weight") else torch.zeros(shape)
    return torch.empty(shape).uniform_(-0.05, 0.05)   # conv bias


class VQModel(nn.Module):
    CH = 128                                   # Encoder/Decoder default ch (vq_model.py:65,129)

    def __init__(self, config: ModelArgs, ch: int = 128):
        super().__init__()
        self.config = config
        self.ch = ch
        self.encoder, self.decoder, self.quantize = _Group(), _Group(), _Group()
        for name, shape in encoder_spec(ch, config.encoder_ch_mult, config.z_channels):
            _install(self.encoder, name, _init_tensor(name, shape))
        for name, shape in decoder_spec(ch, config.decoder_ch_mult, config.z_channels):
            _install(self.decoder, name, _init_tensor(name, shape))
        emb = torch.empty(config.codebook_size, config.codebook_embed_dim).uniform_(
            -1.0 / config.codebook_size, 1.0 / config.codebook_size)              # vq_model.py:207
        if config.codebook_l2_norm:
            emb = torch.nn.functional.normalize(emb, p=2, dim=-1)                  # vq_model.py:208-209
        self.quantize.embedding = _Group()
        self.quantize.embedding.weight = nn.Parameter(emb, requires_grad=False)
        if config.codebook_show_usage:
            self.quantize.register_buffer("codebook_used", torch.zeros(65536))
        self.quant_conv, self.post_quant_conv = _Group(), _Group()
        for g, (co, ci) in ((self.quant_conv, (config.codebook_embed_dim, config.z_channels)),
                            (self.post_quant_conv, (config.z_channels, config.codebook_embed_dim))):
            g.weight = nn.Parameter(_init_tensor("w", (co, ci, 1, 1)), requires_grad=False)
            g.bias = nn.Parameter(_init_tensor("b", (co,)), requires_grad=False)
        self._handle = None
        self._sig = None
        self._ws = None

    # ------------------------------------------------------------------ engine plumbing
    def _has_encoder_path(self):
        # the engine builds the encoder with the cfg's single ch_mult; both registry entries use equal lists (vq_model.py:418-422)
        return list(self.config.encoder_ch_mult) == list(self.config.decoder_ch_mult)

    def _decode_tensors(self):
        sd = self.state_dict()
        keep = ("decoder.", "post_quant_conv.") + (("encoder.", "quant_conv.") if self._has_encoder_path() else ())
        return {k: v for k, v in sd.items() if k.startswith(keep) or k == "quantize.embedding.weight"}

    def engine(self):
        tensors = self._decode_tensors()
        first = tensors["quantize.embedding.weight"]
        _lib.require_cuda(first, "VQModel.engine")
        if first.dtype != torch.float32:
            raise _lib.LgError("the VQ tokenizer is kept in fp32 like the reference (sample_c2i.py:30); "
                               "weights are repacked to bf16 operands inside the engine")
        # lg_vq_finalize repacks the conv weights and the normalised codebook into engine-owned copies, so an in-place
        # update (load_state_dict, broadcast_module's copy_) must rebuild them: the version counters are part of the key
        sig = (first.device, tuple((t.data_ptr(), t._version) for t in tensors.values()))
        if self._handle is not None and sig == self._sig:
            return self._handle
        self._drop()
        lib = _lib.load()
        c = self.config
        mult = (ctypes.c_int32 * 8)(*list(c.decoder_ch_mult) + [0] * (8 - len(c.decoder_ch_mult)))
        cfg = _lib.VqCfg(c.codebook_size, c.codebook_embed_dim, c.z_channels, self.ch, 2, len(c.decoder_ch_mult), mult,
                         1 if c.codebook_l2_norm else 0)
        h = ctypes.c_void_p()
        dev = first.device.index if first.device.index is not None else torch.cuda.current_device()
        _lib.check(lib.lg_vq_create(ctypes.byref(cfg), dev, ctypes.byref(h)), "lg_vq_create")
        for name, t in tensors.items():
            if not t.is_contiguous():          # a .contiguous() temporary would leave the engine with a dangling pointer
                raise _lib.LgError(f"parameter {name} must be contiguous")
            _lib.check(lib.lg_vq_bind_weight(h, name.encode(), _lib.ptr(t), _lib.shape_array(t.shape), t.dim()),
                       f"bind {name}")
        _lib.check(lib.lg_vq_finalize(h, _lib.current_stream(first.device)), "lg_vq_finalize")
        self._handle, self._sig = h, sig
        return h

    def _drop(self):
        if self._handle is not None:
            _lib.load().lg_vq_destroy(self._handle)
        self._handle = None

    def __del__(self):
        try:
            self._drop()
        except Exception:
            pass

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def decode_code(self, code_b, shape=None, channel_first=True):
        """vq_model.py:52-55. code_b: int tensor [B, g*g] (or flat), shape = [B, embed_dim, g, g].
        Returns fp32 NCHW [B, 3, H, W] on the model's device."""
        if shape is None or not channel_first:
            raise NotImplementedError("decode_code needs shape=[B, C, g, g] with channel_first=True (the only form the samplers use)")
        h = self.engine()
        lib = _lib.load()
        dev = self.quantize.embedding.weight.device
        B, g = int(shape[0]), int(shape[2])
        if int(shape[3]) != g or int(shape[1]) != self.config.codebook_embed_dim:
            raise ValueError(f"bad latent shape {shape}")
        codes = code_b.to(device=dev, dtype=torch.int32).reshape(B, g * g).contiguous()
        up = 2 ** (len(self.config.decoder_ch_mult) - 1)
        out = torch.empty(B, 3, g * up, g * up, dtype=torch.float32, device=dev)
        base, nbytes = self._workspace(h, B, g, dev)
        _lib.check(lib.lg_vq_decode(h, _lib.ptr(codes), B, g, ctypes.c_void_p(base), nbytes, _lib.ptr(out),
                                    _lib.current_stream(dev)), "lg_vq_decode")
        return out

    @torch.no_grad()
    def decode_code_uint8(self, code_b, shape):
        """decode_code + the samplers' pixel finishing without a resize (sample_c2i_ddp.py:141-143:
        `clamp(127.5 * x + 128, 0, 255).permute(0, 2, 3, 1).to(uint8)`) in ONE pass: conv_out's accumulator drain writes
        the uint8 NHWC bytes, the fp32 image never exists in HBM. Returns uint8 [B, H, W, 3]."""
        h = self.engine()
        lib = _lib.load()
        dev = self.quantize.embedding.weight.device
        B, g = int(shape[0]), int(shape[2])
        if int(shape[3]) != g or int(shape[1]) != self.config.codebook_embed_dim:
            raise ValueError(f"bad latent shape {shape}")
        codes = code_b.to(device=dev, dtype=torch.int32).reshape(B, g * g).contiguous()
        up = 2 ** (len(self.config.decoder_ch_mult) - 1)
        out = torch.empty(B, g * up, g * up, 3, dtype=torch.uint8, device=dev)
        base, nbytes = self._workspace(h, B, g, dev)
        _lib.check(lib.lg_vq_decode_u8(h, _lib.ptr(codes), B, g, ctypes.c_void_p(base), nbytes, _lib.ptr(out),
                                       _lib.current_stream(dev)), "lg_vq_decode_u8")
        return out

    @torch.no_grad()
    def quantize_indices(self, z):
        """Index path of VectorQuantizer.forward (vq_model.py:215-233): z fp32 NCHW [B, e_dim, g, g] -> int64 [B*g*g]."""
        h = self.engine()
        dev = self.quantize.embedding.weight.device
        z = z.to(device=dev, dtype=torch.float32).contiguous()
        B, C, g, g2 = z.shape
        if g != g2 or C != self.config.codebook_embed_dim:
            raise ValueError(f"bad latent shape {tuple(z.shape)}")
        out = torch.empty(B * g * g, dtype=torch.int64, device=dev)
        _lib.check(_lib.load().lg_vq_argmin(h, _lib.ptr(z), B, g, _lib.ptr(out), _lib.current_stream(dev)), "lg_vq_argmin")
        return out

    def _workspace(self, h, B, g, dev):
        nbytes = ctypes.c_size_t()
        _lib.check(_lib.load().lg_vq_workspace_bytes(h, B, g, ctypes.byref(nbytes)), "lg_vq_workspace_bytes")
        if self._ws is None or self._ws.numel() < nbytes.value + 256:
            self._ws = None
            self._ws = torch.empty(nbytes.value + 256, dtype=torch.uint8, device=dev)
        return (self._ws.data_ptr() + 255) // 256 * 256, nbytes.value

    @torch.no_grad()
    def encode(self, x, return_z=False):
        """VQModel.encode (vq_model.py:41-45) in eval mode: x fp32 NCHW [B,3,H,H] in [-1,1] ->
        (quant fp32 [B,e_dim,g,g], (None, None, None, 0), (None, None, indices int64 [B*g*g])), the tuple layout of
        VectorQuantizer.forward :255 (`_, _, [_, _, indices] = vq_model.encode(x)`, extract_codes_c2i.py:103).
        `return_z=True` appends the pre-quantisation quant_conv output (test hook)."""
        if not self._has_encoder_path():
            raise NotImplementedError("encode needs encoder_ch_mult == decoder_ch_mult (true for VQ-8 and VQ-16)")
        h = self.engine()
        dev = self.quantize.embedding.weight.device
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        B, C, H, W = x.shape
        down = 2 ** (len(self.config.encoder_ch_mult) - 1)
        if C != 3 or H != W or H % down:
            raise ValueError(f"bad image shape {tuple(x.shape)}: need [B,3,H,H] with H a multiple of {down}")
        g, ed = H // down, self.config.codebook_embed_dim
        idx = torch.empty(B * g * g, dtype=torch.int64, device=dev)
        quant = torch.empty(B, ed, g, g, dtype=torch.float32, device=dev)
        z = torch.empty(B, ed, g, g, dtype=torch.float32, device=dev) if return_z else None
        base, nbytes = self._workspace(h, B, g, dev)
        _lib.check(_lib.load().lg_vq_encode(h, _lib.ptr(x), B, H, W, ctypes.c_void_p(base), nbytes, _lib.ptr(idx), _lib.ptr(quant),
                                            _lib.ptr(z) if return_z else None, _lib.current_stream(dev)), "lg_vq_encode")
        out = (quant, (None, None, None, 0), (None, None, idx))
        return out + (z,) if return_z else out

    def decode(self, quant):
        raise NotImplementedError("use decode_code (the sampling path never calls decode on raw latents)")


def VQ_8(**kwargs):
    return VQModel(ModelArgs(encoder_ch_mult=[1, 2, 2, 4], decoder_ch_mult=[1, 2, 2, 4], **kwargs))


def VQ_16(**kwargs):
    return VQModel(ModelArgs(encoder_ch_mult=[1, 1, 2, 2, 4], decoder_ch_mult=[1, 1, 2, 2, 4], **kwargs))


VQ_models = {"VQ-16": VQ_16, "VQ-8": VQ_8}
