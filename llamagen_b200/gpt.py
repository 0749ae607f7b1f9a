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


# the per-layer GEMM weights `set_weight_dtype("fp8")` stores as e4m3 codes ("output.weight" joins them with head=True)
FP8_LAYER_WEIGHTS = ("attention.wqkv.weight", "attention.wo.weight", "feed_forward.w1.weight", "feed_forward.w3.weight",
                     "feed_forward.w2.weight")

SCORE_SCRATCH_CAP = 4 << 30   # bytes of lg_score scratch a model keeps; a batch that needs more is scored in image chunks
PREFIX_SCRATCH_CAP = 4 << 30  # bytes of prefix-prefill scratch (generate(prefix=...)); a batch that needs more is prefilled in chunks


def t2i_attn_mask(emb_masks: torch.Tensor, seq: int) -> torch.Tensor:
    """bool [B, seq, seq]: the attention mask dataset/t2i.py:123-128 builds from emb_masks [B, T] (tril, condition columns times
    emb_mask, unit diagonal); slicing the dataset's [:-1, :-1] gives the same matrix at seq = max_seq_length - 1."""
    B, T = emb_masks.shape
    m = torch.tril(torch.ones(seq, seq, device=emb_masks.device)).repeat(B, 1, 1)
    m[:, :, :T] = m[:, :, :T] * emb_masks.float()[:, None, :]
    eye = torch.eye(seq, device=emb_masks.device)
    return (m * (1 - eye) + eye).bool()


def emb_mask_from_attn_mask(mask: torch.Tensor, T: int) -> torch.Tensor:
    """emb_masks [B, T] (float) of a dataset-style t2i attention mask ([B, 1, seq, seq] or [B, seq, seq], any dtype, nonzero =
    visible): read from the last query row, then checked on the mask's device against the mask rebuilt from them. Any other
    mask raises ValueError: the engine's attention implements only this rule."""
    m = mask
    if m.dim() == 4:
        if m.shape[1] != 1:
            raise ValueError(f"the attention mask must be [B, 1, seq, seq] (one mask for every head), got {tuple(m.shape)}")
        m = m[:, 0]
    if m.dim() != 3 or m.shape[1] != m.shape[2] or m.shape[1] < T:
        raise ValueError(f"the attention mask must be [B, seq, seq] with seq >= {T}, got {tuple(mask.shape)}")
    m = m != 0
    seq = m.shape[1]
    emb = m[:, -1, :T].float()
    if seq == T:
        emb[:, T - 1] = 1.0     # the last condition column is then only seen from its own row, through the unit diagonal
    if not torch.equal(t2i_attn_mask(emb, seq), m):
        raise ValueError("unsupported attention mask: only the t2i dataset's causal mask with per-image condition padding "
                         "(dataset/t2i.py:123-128) is implemented")
    return emb


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
        self._weight_dtype = ("auto", True)
        self._w8 = {}
        self._score_ws = None
        self._sjd_ws = None
        self._prefix_ws = None
        self._given_ws = None
        self._slot_ws = None
        self._slot_prefix_ws = None
        self._slot_extend_ws = None
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

    def set_weight_dtype(self, dtype: str = "auto", head: bool = True):
        """Storage of the transformer's GEMM weights inside the engine of a bf16 / fp16 model: "auto" (the parameters themselves)
        or "fp8": every layer's wqkv, wo, w1, w3, w2 and, with head=True, the output head are quantised by the engine
        (lg_quantize_rows_e4m3: e4m3 codes with one power-of-two scale per output row) and the engine streams those codes, half
        the weight bytes. Activations, KV cache, norms and embeddings are untouched. The module's parameters and state_dict() stay
        the 16-bit tensors; the codes are re-made at the next engine() after a parameter moved (`.to()`) or was written in place
        through the parameter itself (load_state_dict, `weight.copy_()`: its version counter changes). A write through `weight.data`
        changes neither and would leave the old codes bound: call requantize() after one. Takes effect at the next engine() /
        setup_caches() / generate()."""
        if dtype not in ("auto", "fp8"):
            raise ValueError(f"weight dtype must be 'auto' or 'fp8', got {dtype!r}")
        if not isinstance(head, bool):
            raise ValueError(f"head must be a bool, got {head!r}")
        self._weight_dtype = (dtype, head if dtype == "fp8" else True)

    def requantize(self):
        """Drop the engine so that the next use re-makes it, and with it the fp8 codes, from the parameters as they are now. Only
        needed after a write through `weight.data`, which no tensor attribute records."""
        self._drop_engine()

    def fp8_weight_names(self):
        """state_dict names of the weights the current set_weight_dtype() setting stores in fp8 (empty for "auto")."""
        dtype, head = self._weight_dtype
        if dtype != "fp8":
            return []
        names = [f"layers.{i}.{w}" for i in range(self.n_layer) for w in FP8_LAYER_WEIGHTS]
        return names + ["output.weight"] if head else names

    def weight_codes(self, name: str, stored: bool = False) -> torch.Tensor:
        """uint8 e4m3 codes [N, K] the engine bound for fp8 weight `name`, column k at index k (stored=True: in the engine's stored
        K order, include/llamagen_b200.h)."""
        codes = self._w8[name][0]
        return codes if stored else codes[:, _lib.weight_fp8_stored_index(codes.shape[1]).to(codes.device)]

    def weight_scales(self, name: str) -> torch.Tensor:
        """fp32 row scales [N] the engine bound for fp8 weight `name`."""
        return self._w8[name][1]

    def _signature(self):
        p = self.tok_embeddings.weight
        sd = self.state_dict()
        # the engine holds its own codes of an fp8 weight: an in-place write to the parameter (load_state_dict, copy_) must re-make them
        versions = tuple(sd[n]._version for n in self.fp8_weight_names())
        return (p.device, p.dtype, tuple(t.data_ptr() for t in sd.values()), self._kv_cache, self._weight_dtype, versions)

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
        fp8 = set(self.fp8_weight_names())
        self._w8 = {}
        try:
            if fp8 and dt == _lib.LG_DTYPE_F32:
                raise _lib.LgError("fp8 weights need a bf16 or fp16 model (fp32 models keep fp32 weights)")
            stream = _lib.current_stream(p.device)
            for name, t in self.state_dict().items():
                if not t.is_contiguous():
                    raise _lib.LgError(f"parameter {name} must be contiguous")
                t_dt = _lib.dtype_code(t.dtype)
                if name in fp8:
                    # the engine's quantiser defines the stored bytes; codes and scales live as long as the engine
                    codes = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
                    scales = torch.empty(t.shape[0], dtype=torch.float32, device=t.device)
                    _lib.check(lib.lg_quantize_rows_e4m3(_lib.ptr(t), t.shape[0], t.shape[1], t_dt, _lib.ptr(codes), _lib.ptr(scales),
                                                         stream), f"quantize {name}")
                    self._w8[name] = (codes, scales)
                    _lib.check(lib.lg_engine_bind_weight(handle, (name + "_scale").encode(), _lib.ptr(scales),
                                                         _lib.shape_array(scales.shape), 1, _lib.LG_DTYPE_F32), f"bind {name}_scale")
                    t, t_dt = codes, _lib.LG_DTYPE_E4M3
                _lib.check(lib.lg_engine_bind_weight(handle, name.encode(), _lib.ptr(t), _lib.shape_array(t.shape),
                                                     t.dim(), t_dt), f"bind {name}")
            self.freqs_cis = self.freqs_cis.to(device=p.device, dtype=torch.float32).contiguous()
            _lib.check(lib.lg_engine_bind_weight(handle, b"freqs_cis", _lib.ptr(self.freqs_cis),
                                                 _lib.shape_array(self.freqs_cis.shape), 3, _lib.LG_DTYPE_F32),
                       "bind freqs_cis")
            if fp8:
                torch.cuda.current_stream(p.device).synchronize()   # lg_engine_finalize reads the scales back
            _lib.check(lib.lg_engine_finalize(handle), "lg_engine_finalize")
        except Exception:
            lib.lg_engine_destroy(handle)
            self._w8 = {}
            raise
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
            base, _ = self._device_buffer("_workspace", nbytes.value, grow=True)
            _lib.check(lib.lg_engine_set_workspace(handle, base, nbytes.value, max_batch_size,
                                                   max_seq_length), "lg_engine_set_workspace")
            self._ws_shape = (max_batch_size, max_seq_length)
        self.max_batch_size = max_batch_size
        self.max_seq_length = max_seq_length

    def _device_buffer(self, attr: str, nbytes: int, grow: bool = False):
        """The torch byte buffer self.<attr> with room for nbytes from a 256-byte aligned address (the engine's alignment), kept
        while it is on the model's device and large enough unless `grow`; the old buffer is dropped before the new one is allocated.
        Returns (aligned device pointer, usable bytes)."""
        dev = self.tok_embeddings.weight.device
        buf = getattr(self, attr)
        if grow or buf is None or buf.numel() < nbytes + 256 or buf.device != dev:
            setattr(self, attr, None)
            buf = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
            setattr(self, attr, buf)
        base = (buf.data_ptr() + 255) // 256 * 256
        return ctypes.c_void_p(base), buf.numel() - (base - buf.data_ptr())

    # ------------------------------------------------------------------ teacher-forced scoring (lg_score)
    def _score_scratch(self, rows: int, seq: int, nh: int):
        """The lg_score scratch for `rows` sequences of `seq` positions, capped at SCORE_SCRATCH_CAP bytes (the engine then scores
        the batch in image chunks); kept on the model like the setup_caches() workspace. Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        need, one = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(lib.lg_score_workspace_bytes(handle, rows, seq, ctypes.byref(need)), "lg_score_workspace_bytes")
        _lib.check(lib.lg_score_workspace_bytes(handle, nh, seq, ctypes.byref(one)), "lg_score_workspace_bytes")
        return self._device_buffer("_score_ws", need.value if need.value <= SCORE_SCRATCH_CAP else max(SCORE_SCRATCH_CAP, one.value))

    def _prefix_scratch(self, rows: int, seq: int, nh: int):
        """The scratch of generate(prefix=...)'s prefill of `rows` rows of `seq` = T + P positions, capped at PREFIX_SCRATCH_CAP bytes
        (the engine then prefills in chunks of rows); kept on the model like the setup_caches() workspace. Returns (device pointer,
        bytes), the bytes at most what was asked for."""
        lib, handle = _lib.load(), self.engine()
        need, one = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(lib.lg_prefix_workspace_bytes(handle, rows, seq, ctypes.byref(need)), "lg_prefix_workspace_bytes")
        _lib.check(lib.lg_prefix_workspace_bytes(handle, nh, seq, ctypes.byref(one)), "lg_prefix_workspace_bytes")
        want = need.value if need.value <= PREFIX_SCRATCH_CAP else max(PREFIX_SCRATCH_CAP, one.value)
        base, nbytes = self._device_buffer("_prefix_ws", want)
        return base, min(nbytes, want)

    def _given_scratch(self, given, T: int, use_cfg: bool):
        """The scratch of generate(given=..., given_mask=...) for given (int32 host [B, S], -1: drawn): the given tokens, the window
        passes' rows and the prefill of the leading run given to every image, the prefill part capped as _prefix_scratch caps it (so a
        mask of the first P columns prefills as generate(prefix=...) does); kept on the model like the setup_caches() workspace.
        Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        B, S = given.shape
        need = ctypes.c_size_t()
        _lib.check(lib.lg_given_workspace_bytes(handle, _lib.ptr(given), B, S, int(use_cfg), ctypes.byref(need)), "lg_given_workspace_bytes")
        want = need.value
        lead = (given >= 0).all(0).tolist() + [False]
        P = lead.index(False)
        if P > 0:
            nh = 2 if use_cfg else 1
            pneed, pone = ctypes.c_size_t(), ctypes.c_size_t()
            _lib.check(lib.lg_prefix_workspace_bytes(handle, nh * B, T + P, ctypes.byref(pneed)), "lg_prefix_workspace_bytes")
            _lib.check(lib.lg_prefix_workspace_bytes(handle, nh, T + P, ctypes.byref(pone)), "lg_prefix_workspace_bytes")
            want += (pneed.value if pneed.value <= PREFIX_SCRATCH_CAP else max(PREFIX_SCRATCH_CAP, pone.value)) - pneed.value
        base, nbytes = self._device_buffer("_given_ws", want)
        return base, min(nbytes, want)

    def _slot_scratch(self, use_cfg: bool):
        """The lg_prefill_slot scratch (serve.LLM's join of one t2i request), kept on the model like the setup_caches() workspace.
        Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_slot_workspace_bytes(handle, int(use_cfg), ctypes.byref(need)), "lg_slot_workspace_bytes")
        return self._device_buffer("_slot_ws", need.value)

    def _slot_prefix_scratch(self, use_cfg: bool, P: int):
        """The lg_prefill_slot_prefix scratch (serve.LLM's join of one image-completion request with P given tokens), kept on the model
        like _slot_scratch and grown to the longest prefix seen. Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_slot_prefix_workspace_bytes(handle, int(use_cfg), int(P), ctypes.byref(need)), "lg_slot_prefix_workspace_bytes")
        return self._device_buffer("_slot_prefix_ws", need.value)

    def _slot_extend_scratch(self, use_cfg: bool, K: int):
        """The lg_extend_slot scratch (serve.LLM's window pass over a run of K given tokens of one inpainting request), kept on the model
        like _slot_scratch and grown to the largest seen. Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_slot_extend_workspace_bytes(handle, int(use_cfg), int(K), ctypes.byref(need)), "lg_slot_extend_workspace_bytes")
        return self._device_buffer("_slot_extend_ws", need.value)

    def _sjd_scratch(self, B: int, use_cfg: bool, L: int):
        """The lg_generate_sjd scratch for B images and window L, kept on the model like the setup_caches() workspace.
        Returns (device pointer, bytes)."""
        lib, handle = _lib.load(), self.engine()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_sjd_workspace_bytes(handle, B, int(use_cfg), L, ctypes.byref(need)), "lg_sjd_workspace_bytes")
        return self._device_buffer("_sjd_ws", need.value)

    def _score(self, cond, idx, targets, emb_masks, cfg_scale: float, want_logits: bool, want_nll: bool):
        """lg_score over complete sequences: cond (c2i labels [B] / t2i features [B, T, C]), idx [B, S-1] or None (S = 1),
        targets [B, S] or None. Returns (logits fp32 [B, S, V] or None, nll fp32 [B, S] or None)."""
        lib, handle = _lib.load(), self.engine()
        dev = self.tok_embeddings.weight.device
        if self.model_type == "c2i":
            cond_dev = cond.to(device=dev, dtype=torch.int32).contiguous()
            if cond_dev.dim() != 1:
                raise ValueError("c2i cond must be a 1-D tensor of class labels")
            T = 1
        else:
            cond_dev = cond[:, : self.cls_token_num].to(device=dev, dtype=self.tok_embeddings.weight.dtype).contiguous()
            T = cond_dev.shape[1]
        B = cond_dev.shape[0]
        S = 1 if idx is None else idx.shape[1] + 1
        if idx is not None and tuple(idx.shape) != (B, S - 1):
            raise ValueError(f"idx must be [B, S-1] = [{B}, {S - 1}], got {tuple(idx.shape)}")
        if not 1 <= S <= self.block_size:
            raise ValueError(f"a scored sequence holds 1 .. block_size={self.block_size} tokens, got {S}")
        V = self.vocab_size
        idx_dev = idx.to(device=dev, dtype=torch.int32).contiguous() if idx is not None else None
        tgt = None
        if targets is not None:
            tgt = targets.to(device=dev, dtype=torch.int64)
            if tuple(tgt.shape) != (B, S):
                raise ValueError(f"targets must be [B, S] = [{B}, {S}], got {tuple(tgt.shape)}")
            if bool(((tgt < 0) | (tgt >= V)).any()):
                raise ValueError(f"targets must lie in [0, vocab_size={V})")
            tgt = tgt.to(torch.int32).contiguous()
        em = None
        if emb_masks is not None:
            if tuple(emb_masks.shape) != (B, T):
                raise ValueError(f"emb_masks must be [B, T] = [{B}, {T}], got {tuple(emb_masks.shape)}")
            em = emb_masks.to(device=dev, dtype=torch.float32).contiguous()
        use_cfg = cfg_scale > 1.0                               # generate.py:128
        nh = 2 if use_cfg else 1
        logits = torch.empty(B, S, V, dtype=torch.float32, device=dev) if want_logits else None
        nll = torch.empty(B, S, dtype=torch.float32, device=dev) if want_nll else None
        ws, ws_bytes = self._score_scratch(nh * B, T + S - 1, nh)
        _lib.check(lib.lg_score(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(idx_dev), _lib.ptr(tgt), B, T, S, int(use_cfg),
                                float(cfg_scale), ws, ws_bytes, _lib.ptr(logits), _lib.ptr(nll), _lib.current_stream(dev)),
                   "lg_score")
        return logits, nll

    # ------------------------------------------------------------------ reference-style forward
    def forward(self, idx, cond_idx, input_pos=None, targets=None, mask=None, valid=None, emb_masks=None):
        """Transformer.forward (gpt.py:341-382) through the engine, eval mode (no dropout).

        teacher-forced: idx [B, L] and cond_idx given -> (fp32 logits [B, L + 1, V] of positions cls_token_num - 1 .. (the
                 training branch's logits[:, cls_token_num - 1:]), loss): the mean cross entropy over targets [B, L + 1], or its
                 `valid`-weighted mean. t2i: emb_masks [B, T], or the dataset's attention `mask` ([B, 1, seq, seq] or [B, seq, seq],
                 dataset/t2i.py:123-128 sliced [:-1, :-1]) from which they are derived. Needs no setup_caches().
        prefill: idx=None, cond_idx given  -> fp32 logits [rows, 1, V] of the LAST condition position
                 (the only one generate() reads, generate.py:58; the reference materialises all T).
        decode : idx [rows, 1], cond_idx=None, input_pos=[p] -> fp32 logits [rows, 1, V].
        rows are taken as given (the caller has already doubled them for CFG, as in the reference)."""
        if idx is not None and cond_idx is not None:
            if mask is not None:
                if emb_masks is not None:
                    raise ValueError("pass either mask or emb_masks, not both")
                if self.model_type != "t2i":
                    raise ValueError("an attention mask applies to t2i models only (c2i sequences are plain causal)")
                emb_masks = emb_mask_from_attn_mask(mask, self.cls_token_num)
            logits, nll = self._score(cond_idx, idx, targets, emb_masks, 1.0, True, targets is not None)
            loss = None
            if valid is not None:                               # gpt.py:373-376
                w = valid.to(device=nll.device, dtype=torch.float32)[:, None].repeat(1, nll.shape[1]).reshape(-1)
                loss = (nll.reshape(-1) * w).sum() / torch.clamp(w.sum(), min=1.0)
            elif targets is not None:                           # gpt.py:377-378
                loss = nll.mean()
            return logits, loss
        if targets is not None:
            raise ValueError("targets need both idx and cond_idx (the teacher-forced forward)")
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
