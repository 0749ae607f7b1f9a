"""Host-side mirror of the reference AR transformer interface (autoregressive/models/gpt.py).

Only the *interface* lives here: a parameter container whose state_dict names/shapes equal the
reference's (SURVEY §5: `layers.{i}.attention.wqkv.weight`, `cls_embedding.embedding_table.weight`, ...),
the `GPT_models` registry (gpt.py:438-467) and the `ModelArgs` fields the inference path reads
(gpt.py:23-50).  All compute is done by the sm_90a kernels behind the C-ABI engine
(include/llamagen_b200.h); there is no PyTorch forward and no CPU path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn

from . import _lib


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


@dataclass
class ModelArgs:
    # same field names / defaults as the reference dataclass (gpt.py:23-50)
    dim: int = 4096
    n_layer: int = 32
    n_head: int = 32
    n_kv_head: Optional[int] = None
    multiple_of: int = 256
    ffn_dim_multiplier: Optional[float] = None
    rope_base: float = 10000
    norm_eps: float = 1e-5
    initializer_range: float = 0.02
    token_dropout_p: float = 0.1
    attn_dropout_p: float = 0.0
    resid_dropout_p: float = 0.1
    ffn_dropout_p: float = 0.1
    drop_path_rate: float = 0.0
    num_classes: int = 1000
    caption_dim: int = 2048
    class_dropout_prob: float = 0.1
    model_type: str = "c2i"
    vocab_size: int = 16384
    cls_token_num: int = 1
    block_size: int = 256
    max_batch_size: int = 32
    max_seq_len: int = 2048

    @property
    def ffn_dim(self) -> int:
        # FeedForward.__init__ (gpt.py:154-159)
        hidden = int(2 * (4 * self.dim) / 3)
        if self.ffn_dim_multiplier is not None:
            hidden = int(self.ffn_dim_multiplier * hidden)
        return find_multiple(hidden, self.multiple_of)

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_head


def rope_table_2d(grid_size: int, head_dim: int, base: float, cls_token_num: int) -> torch.Tensor:
    """fp32 [cls_token_num + grid^2, head_dim/2, 2] (cos, sin) table — the same torch fp32 expression as
    precompute_freqs_cis_2d (gpt.py:404-417) so the uploaded table is bit-identical to the reference's:
    first head_dim/4 pairs rotate with the row index, the next head_dim/4 with the column index, and the
    condition positions get all-zero (cos, sin) rows (SURVEY G2/G3)."""
    half = head_dim // 2
    inv = 1.0 / (base ** (torch.arange(0, half, 2)[: half // 2].float() / half))
    ang = torch.outer(torch.arange(grid_size), inv)                       # [g, hd/4]
    rows = ang[:, None, :].expand(grid_size, grid_size, ang.shape[-1])
    cols = ang[None, :, :].expand(grid_size, grid_size, ang.shape[-1])
    both = torch.cat([rows, cols], dim=-1).reshape(grid_size * grid_size, -1)   # [g*g, hd/2]
    table = torch.stack([torch.cos(both), torch.sin(both)], dim=-1)
    return torch.cat([torch.zeros(cls_token_num, head_dim // 2, 2), table]).contiguous()


class _Group(nn.Module):
    """Bare namespace so parameters get the reference's dotted names."""


def _weight(out_f: int, in_f: int, std: float) -> nn.Parameter:
    return nn.Parameter(torch.empty(out_f, in_f).normal_(mean=0.0, std=std))


class Transformer(nn.Module):
    """Parameter container + engine handle. Drop-in for `GPT_models[name](**kwargs)` objects:
    supports .to(device, dtype), .eval(), .load_state_dict(sd, strict=False) and the attributes
    generate() reads (model_type, num_classes, cls_token_num, tok_embeddings, cls_embedding)."""

    def __init__(self, config: ModelArgs):
        super().__init__()
        if config.model_type not in ("c2i", "t2i"):
            raise Exception("please check model type")          # gpt.py:275
        if config.n_kv_head not in (None, config.n_head):
            raise NotImplementedError("grouped KV heads are not used by any LlamaGen registry model")
        if config.dim % config.n_head:
            raise ValueError("dim must be divisible by n_head")
        grid = int(config.block_size ** 0.5)
        if grid * grid != config.block_size:
            raise AssertionError("block_size must be a square")  # gpt.py:291
        self.config = config
        self.vocab_size = config.vocab_size
        self.n_layer = config.n_layer
        self.block_size = config.block_size
        self.num_classes = config.num_classes
        self.model_type = config.model_type
        self.cls_token_num = config.cls_token_num
        std, D, F = config.initializer_range, config.dim, config.ffn_dim

        self.cls_embedding = _Group()
        if config.model_type == "c2i":
            rows = config.num_classes + (1 if config.class_dropout_prob > 0 else 0)   # gpt.py:60-62
            self.cls_embedding.embedding_table = _Group()
            self.cls_embedding.embedding_table.weight = _weight(rows, D, std)
        else:
            self.cls_embedding.cap_proj = _Group()
            self.cls_embedding.cap_proj.fc1 = _Group()
            self.cls_embedding.cap_proj.fc1.weight = _weight(D, config.caption_dim, std)
            self.cls_embedding.cap_proj.fc2 = _Group()
            self.cls_embedding.cap_proj.fc2.weight = _weight(D, D, std)
            self.cls_embedding.register_buffer(
                "uncond_embedding", torch.randn(config.cls_token_num, config.caption_dim) / config.caption_dim ** 0.5)
        self.tok_embeddings = _Group()
        self.tok_embeddings.weight = _weight(config.vocab_size, D, std)

        self.layers = nn.ModuleList()
        for _ in range(config.n_layer):
            blk = _Group()
            blk.attention = _Group()
            blk.attention.wqkv = _Group()
            blk.attention.wqkv.weight = _weight(3 * D, D, std)
            blk.attention.wo = _Group()
            blk.attention.wo.weight = _weight(D, D, std)
            blk.feed_forward = _Group()
            for name, (o, i) in (("w1", (F, D)), ("w3", (F, D)), ("w2", (D, F))):
                g = _Group()
                g.weight = _weight(o, i, std)
                setattr(blk.feed_forward, name, g)
            blk.attention_norm = _Group()
            blk.attention_norm.weight = nn.Parameter(torch.ones(D))
            blk.ffn_norm = _Group()
            blk.ffn_norm.weight = nn.Parameter(torch.ones(D))
            self.layers.append(blk)
        self.norm = _Group()
        self.norm.weight = nn.Parameter(torch.ones(D))
        self.output = _Group()
        # the reference zero-initialises the head (gpt.py:305); kept for init parity (SURVEY G1)
        self.output.weight = nn.Parameter(torch.zeros(config.vocab_size, D))

        self.freqs_cis = rope_table_2d(grid, config.head_dim, config.rope_base, config.cls_token_num)
        self.max_batch_size = -1
        self.max_seq_length = -1
        self._engine = None
        self._engine_sig = None
        self._workspace = None
        self._ws_shape = (0, 0)
        self._kv_cache = ("auto", None)
        self.requires_grad_(False)

    # ------------------------------------------------------------------ engine plumbing
    def set_kv_cache(self, dtype: str = "auto", scales=None):
        """KV-cache storage of a bf16 / fp16 model: "auto" (the model dtype) or "fp8" (e4m3, half the cache bytes).
        scales: [n_layer, 2] per-layer (k, v) scales for fp8, each a power of two in [2^-8, 2^7]; None = all 1.0. K and V are
        stored as e4m3(x / s) and read back as e4m3 * s. Takes effect at the next setup_caches(), which re-creates the workspace."""
        if dtype not in ("auto", "fp8"):
            raise ValueError(f"kv cache dtype must be 'auto' or 'fp8', got {dtype!r}")
        if scales is not None:
            if dtype != "fp8":
                raise ValueError("KV-cache scales apply to the fp8 cache only")
            s = torch.as_tensor(scales, dtype=torch.float32).detach().cpu()
            if tuple(s.shape) != (self.n_layer, 2):
                raise ValueError(f"KV-cache scales must have shape [{self.n_layer}, 2], got {tuple(s.shape)}")
            scales = tuple(float(x) for x in s.reshape(-1))
        self._kv_cache = (dtype, scales)

    def _signature(self):
        p = self.tok_embeddings.weight
        return (p.device, p.dtype, tuple(t.data_ptr() for t in self.state_dict().values()), self._kv_cache)

    def engine(self):
        """Create / refresh the C engine for the parameters' current device + dtype."""
        p = self.tok_embeddings.weight
        _lib.require_cuda(p, "Transformer.engine")
        dt = _lib.dtype_code(p.dtype)   # fp32, bf16 or fp16; raises for anything else
        sig = self._signature()
        if self._engine is not None and sig == self._engine_sig:
            return self._engine
        self._drop_engine()
        lib = _lib.load()
        c = self.config
        cfg = _lib.ModelCfg(c.n_layer, c.n_head, c.dim, c.ffn_dim, c.vocab_size, c.cls_token_num, c.block_size,
                            c.num_classes, c.caption_dim,
                            _lib.LG_MODEL_C2I if c.model_type == "c2i" else _lib.LG_MODEL_T2I, dt, c.norm_eps)
        handle = ctypes.c_void_p()
        dev_index = p.device.index if p.device.index is not None else torch.cuda.current_device()
        _lib.check(lib.lg_engine_create(ctypes.byref(cfg), dev_index, ctypes.byref(handle)), "lg_engine_create")
        self._keepalive = []
        for name, t in self.state_dict().items():
            if not t.is_contiguous():
                raise _lib.LgError(f"parameter {name} must be contiguous")
            t_dt = _lib.dtype_code(t.dtype)
            _lib.check(lib.lg_engine_bind_weight(handle, name.encode(), _lib.ptr(t), _lib.shape_array(t.shape),
                                                 t.dim(), t_dt), f"bind {name}")
        self.freqs_cis = self.freqs_cis.to(device=p.device, dtype=torch.float32).contiguous()
        _lib.check(lib.lg_engine_bind_weight(handle, b"freqs_cis", _lib.ptr(self.freqs_cis),
                                             _lib.shape_array(self.freqs_cis.shape), 3, _lib.LG_DTYPE_F32),
                   "bind freqs_cis")
        _lib.check(lib.lg_engine_finalize(handle), "lg_engine_finalize")
        kv_dtype, kv_scales = self._kv_cache
        if kv_dtype == "fp8":
            arr = (ctypes.c_float * len(kv_scales))(*kv_scales) if kv_scales is not None else None
            status = lib.lg_engine_set_kv_cache(handle, _lib.LG_DTYPE_E4M3, arr)
            if status < 0:
                msg = lib.lg_last_error()
                lib.lg_engine_destroy(handle)
                raise _lib.LgError(f"lg_engine_set_kv_cache: {msg.decode() if msg else 'unknown error'}")
        self._engine, self._engine_sig = handle, sig
        self._workspace, self._ws_shape = None, (0, 0)
        return handle

    def _drop_engine(self):
        if self._engine is not None:
            _lib.load().lg_engine_destroy(self._engine)
        self._engine = None
        self._engine_sig = None

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    def setup_caches(self, max_batch_size, max_seq_length, dtype=None):
        """gpt.py:316-330 — allocate the KV cache + scratch (one torch byte buffer handed to the engine).
        max_seq_length is rounded up to a multiple of 8 like the reference (SURVEY G10)."""
        handle = self.engine()
        max_seq_length = find_multiple(max_seq_length, 8)
        rows, seq = self._ws_shape
        if self._workspace is None or rows < max_batch_size or seq < max_seq_length:
            lib = _lib.load()
            nbytes = ctypes.c_size_t()
            _lib.check(lib.lg_engine_workspace_bytes(handle, max_batch_size, max_seq_length, ctypes.byref(nbytes)),
                       "lg_engine_workspace_bytes")
            dev = self.tok_embeddings.weight.device
            self._workspace = None
            self._workspace = torch.empty(nbytes.value + 256, dtype=torch.uint8, device=dev)
            base = (self._workspace.data_ptr() + 255) // 256 * 256
            _lib.check(lib.lg_engine_set_workspace(handle, ctypes.c_void_p(base), nbytes.value, max_batch_size,
                                                   max_seq_length), "lg_engine_set_workspace")
            self._ws_shape = (max_batch_size, max_seq_length)
        self.max_batch_size = max_batch_size
        self.max_seq_length = max_seq_length

    # ------------------------------------------------------------------ reference-style forward
    def forward(self, idx, cond_idx, input_pos=None, targets=None, mask=None, valid=None, emb_masks=None):
        """Inference branches of Transformer.forward (gpt.py:348-368) through the engine.

        prefill: idx=None, cond_idx given  -> fp32 logits [rows, 1, V] of the LAST condition position
                 (the only one generate() reads, generate.py:58; the reference materialises all T).
        decode : idx [rows, 1], cond_idx=None, input_pos=[p] -> fp32 logits [rows, 1, V].
        rows are taken as given (the caller has already doubled them for CFG, as in the reference)."""
        if targets is not None or (idx is not None and cond_idx is not None):
            raise NotImplementedError("training / teacher-forced full-sequence forward is outside the sampling hot path")
        if self.max_batch_size < 0:
            raise _lib.LgError("call setup_caches() before forward() (as generate() does)")
        lib, handle = _lib.load(), self.engine()
        dev = self.tok_embeddings.weight.device
        V = self.vocab_size
        if cond_idx is not None:
            rows = cond_idx.shape[0]
            out = torch.empty(rows, 1, V, dtype=torch.float32, device=dev)
            if self.model_type == "c2i":
                cond = cond_idx.to(device=dev, dtype=torch.int32).contiguous()
                T = 1
            else:
                cond = cond_idx.to(device=dev, dtype=self.tok_embeddings.weight.dtype).contiguous()
                T = cond.shape[1]
            em = emb_masks.to(device=dev, dtype=torch.float32).contiguous() if emb_masks is not None else None
            _lib.check(lib.lg_prefill(handle, _lib.ptr(cond), _lib.ptr(em), rows, T, 0, _lib.ptr(out),
                                      _lib.current_stream(dev)), "lg_prefill")
            return out, None
        rows = idx.shape[0]
        pos = int(input_pos.reshape(-1)[0].item())
        tok = idx.reshape(-1).to(device=dev, dtype=torch.int32).contiguous()
        out = torch.empty(rows, 1, V, dtype=torch.float32, device=dev)
        _lib.check(lib.lg_decode_step(handle, _lib.ptr(tok), rows, pos, 0, _lib.ptr(out), _lib.current_stream(dev)),
                   "lg_decode_step")
        return out, None


# ---------------------------------------------------------------------------- registry (gpt.py:438-467)
_SHAPES = {
    # name: (n_layer, n_head, dim)
    "GPT-B": (12, 12, 768), "GPT-L": (24, 16, 1024), "GPT-XL": (36, 20, 1280), "GPT-XXL": (48, 24, 1536),
    "GPT-XXXL": (48, 40, 2560), "GPT-1B": (22, 32, 2048), "GPT-3B": (24, 32, 3200), "GPT-7B": (32, 32, 4096),
}


def _factory(name):
    n_layer, n_head, dim = _SHAPES[name]

    def make(**kwargs):
        return Transformer(ModelArgs(n_layer=n_layer, n_head=n_head, dim=dim, **kwargs))

    make.__name__ = name.replace("-", "_")
    return make


GPT_models = {name: _factory(name) for name in _SHAPES}
