"""T5 text encoder on the engine: transformers' `T5EncoderModel` forward (Flan-T5, T5 v1.1) in the library's own CUDA.

`T5Encoder` replaces the `T5Embedder` of the reference's language/t5.py (and `cond.HFT5Encoder`) on the device: a caption goes
in, `last_hidden_state` [B, T, d_model] and the attention mask come out, with no second framework model on the card. Parameters
keep the HuggingFace names, so a checkpoint directory loads as it is (`from_pretrained`). Tokenisation stays the HuggingFace
tokenizer of that directory (a CPU string operation); caption cleaning (ftfy / bs4) is skipped, as `HFT5Encoder` skips it.
"""
from __future__ import annotations

import ctypes
import glob
import json
import math
import os

import torch
from torch import nn

from . import _lib

MAX_T = 512   # the attention kernels keep a caption's K / V in shared memory


class T5Config:
    """The fields of a T5 `config.json` the encoder reads."""

    def __init__(self, num_layers, d_model, d_kv, num_heads, d_ff, vocab_size, relative_attention_num_buckets=32,
                 relative_attention_max_distance=128, layer_norm_epsilon=1e-6, feed_forward_proj="gated-gelu"):
        self.num_layers, self.d_model, self.d_kv, self.num_heads = int(num_layers), int(d_model), int(d_kv), int(num_heads)
        self.d_ff, self.vocab_size = int(d_ff), int(vocab_size)
        self.num_buckets = int(relative_attention_num_buckets)
        self.max_distance = int(relative_attention_max_distance)
        self.eps = float(layer_norm_epsilon)
        self.feed_forward_proj = feed_forward_proj

    @classmethod
    def from_json(cls, path):
        c = json.load(open(path))
        return cls(c["num_layers"], c["d_model"], c["d_kv"], c["num_heads"], c["d_ff"], c["vocab_size"],
                   c.get("relative_attention_num_buckets", 32), c.get("relative_attention_max_distance", 128),
                   c.get("layer_norm_epsilon", 1e-6), c.get("feed_forward_proj", "relu"))

    def check(self, dtype):
        """ValueError for what the engine does not run: fp16 (T5 overflows it), d_kv != 64, non-gated feed-forwards."""
        if dtype == torch.float16:
            raise ValueError("fp16 T5 is not supported: its activations overflow fp16 (transformers needs inf clamps and an fp32 wo); "
                             "use bfloat16 or float32")
        if dtype not in (torch.bfloat16, torch.float32):
            raise ValueError(f"unsupported T5 dtype {dtype} (bfloat16 or float32)")
        if self.d_kv != 64:
            raise ValueError(f"d_kv={self.d_kv} is not supported (the attention kernels take 64)")
        if self.feed_forward_proj != "gated-gelu":
            raise ValueError(f"feed_forward_proj={self.feed_forward_proj!r} is not supported (gated-gelu only)")


def relative_position_bucket(relative_position, num_buckets=32, max_distance=128):
    """Bidirectional relative-position bucket of transformers' T5Attention._relative_position_bucket, the same torch expression."""
    num_buckets //= 2
    ret = (relative_position > 0).to(torch.long) * num_buckets
    n = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = n < max_exact
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return ret + torch.where(is_small, n, large)


def bucket_table(T, num_buckets=32, max_distance=128, device="cpu"):
    """int32 [2T - 1]: entry (j - i) + T - 1 is the bucket of key j seen from query i, computed on `device` as the model would."""
    rel = torch.arange(-(T - 1), T, dtype=torch.long, device=device)
    return relative_position_bucket(rel, num_buckets, max_distance).to(torch.int32)


class _Norm(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))


def _linear(i, o):
    return nn.Linear(i, o, bias=False)


class _Block(nn.Module):
    def __init__(self, c: T5Config, has_bias: bool):
        super().__init__()
        inner = c.num_heads * c.d_kv
        attn = nn.Module()
        attn.SelfAttention = nn.Module()
        for n in ("q", "k", "v"):
            setattr(attn.SelfAttention, n, _linear(c.d_model, inner))
        attn.SelfAttention.o = _linear(inner, c.d_model)
        if has_bias:
            attn.SelfAttention.relative_attention_bias = nn.Embedding(c.num_buckets, c.num_heads)
        attn.layer_norm = _Norm(c.d_model)
        ff = nn.Module()
        ff.DenseReluDense = nn.Module()
        ff.DenseReluDense.wi_0 = _linear(c.d_model, c.d_ff)
        ff.DenseReluDense.wi_1 = _linear(c.d_model, c.d_ff)
        ff.DenseReluDense.wo = _linear(c.d_ff, c.d_model)
        ff.layer_norm = _Norm(c.d_model)
        self.layer = nn.ModuleList([attn, ff])


def _read_checkpoint(path):
    """Tensors of the files T5Embedder downloads: model.safetensors, pytorch_model.bin, or shards listed by their *.index.json."""
    def load(f):
        if f.endswith(".safetensors"):
            from safetensors.torch import load_file
            return load_file(f)
        return torch.load(f, map_location="cpu", weights_only=True)
    for single in ("model.safetensors", "pytorch_model.bin"):
        if os.path.exists(os.path.join(path, single)):
            return load(os.path.join(path, single))
    for index in ("model.safetensors.index.json", "pytorch_model.bin.index.json"):
        f = os.path.join(path, index)
        if os.path.exists(f):
            sd = {}
            for shard in sorted(set(json.load(open(f))["weight_map"].values())):
                sd.update(load(os.path.join(path, shard)))
            return sd
    found = sorted(glob.glob(os.path.join(path, "*.safetensors")) + glob.glob(os.path.join(path, "*.bin")))
    raise FileNotFoundError(f"no T5 checkpoint in {path} (model.safetensors, pytorch_model.bin or an *.index.json); found {found}")


def encoder_state_dict(sd):
    """The encoder's tensors of a T5 checkpoint: shared.weight (or the tied encoder.embed_tokens.weight) and encoder.*; the decoder
    and lm_head are dropped."""
    out = {k: v for k, v in sd.items() if k.startswith("encoder.") and k != "encoder.embed_tokens.weight"}
    emb = sd.get("shared.weight", sd.get("encoder.embed_tokens.weight"))
    if emb is not None:
        out["shared.weight"] = emb
    return out


class T5Encoder(nn.Module):
    """T5EncoderModel's forward on the engine. `encode(ids, mask)` -> last_hidden_state; `__call__(prompts)` -> (embs, mask) as
    T5Embedder.get_text_embeddings returns them (padded to max_length, truncated, special tokens added)."""

    def __init__(self, config: T5Config, max_length: int = 120, tokenizer=None):
        super().__init__()
        if not 1 <= max_length <= MAX_T:
            raise ValueError(f"max_length={max_length} outside [1, {MAX_T}]")
        self.config = config
        self.d_model = config.d_model
        self.max_length = max_length
        self.tokenizer = tokenizer
        self.tokenizer_path = None
        self.shared = nn.Embedding(config.vocab_size, config.d_model)
        self.encoder = nn.Module()
        self.encoder.block = nn.ModuleList([_Block(config, i == 0) for i in range(config.num_layers)])
        self.encoder.final_layer_norm = _Norm(config.d_model)
        self._engine = None
        self._engine_sig = None
        self._ws = None
        self._buckets = {}

    @classmethod
    def from_pretrained(cls, path, dtype=torch.bfloat16, device="cuda", max_length=120, tokenizer=None):
        cfg = T5Config.from_json(os.path.join(path, "config.json"))
        cfg.check(dtype)
        model = cls(cfg, max_length=max_length, tokenizer=tokenizer)
        model.tokenizer_path = path
        sd = encoder_state_dict(_read_checkpoint(path))
        want = model.state_dict()
        missing = sorted(set(want) - set(sd))
        if missing:
            raise KeyError(f"{path}: missing T5 encoder weights {missing[:8]}{' ...' if len(missing) > 8 else ''}")
        for k, v in want.items():
            if tuple(sd[k].shape) != tuple(v.shape):
                raise ValueError(f"{path}: {k} has shape {tuple(sd[k].shape)}, expected {tuple(v.shape)}")
        model.load_state_dict({k: sd[k] for k in want})
        return model.to(device=device, dtype=dtype).eval()

    # ------------------------------------------------------------------------------------------------ engine
    def _signature(self):
        # the engine borrows every parameter and copies none: storage pointers decide when it must be re-made, and an in-place
        # write (load_state_dict, copy_) is read by the next encode as it is
        p = self.shared.weight
        return (p.device, p.dtype, tuple(t.data_ptr() for t in self.state_dict().values()))

    def engine(self):
        """Create / refresh the C encoder for the parameters' current device + dtype."""
        p = self.shared.weight
        _lib.require_cuda(p, "T5Encoder.engine")
        self.config.check(p.dtype)
        sig = self._signature()
        if self._engine is not None and sig == self._engine_sig:
            return self._engine
        self._drop_engine()
        lib = _lib.load()
        c = self.config
        cfg = _lib.T5Cfg(c.num_layers, c.d_model, c.d_kv, c.num_heads, c.d_ff, c.vocab_size, c.num_buckets, 1, _lib.dtype_code(p.dtype),
                         c.eps)
        handle = ctypes.c_void_p()
        dev_index = p.device.index if p.device.index is not None else torch.cuda.current_device()
        _lib.check(lib.lg_t5_create(ctypes.byref(cfg), dev_index, ctypes.byref(handle)), "lg_t5_create")
        try:
            for name, t in self.state_dict().items():
                if not t.is_contiguous():
                    raise _lib.LgError(f"parameter {name} must be contiguous")
                _lib.check(lib.lg_t5_bind_weight(handle, name.encode(), _lib.ptr(t), _lib.shape_array(t.shape), t.dim(),
                                                 _lib.dtype_code(t.dtype)), f"bind {name}")
            _lib.check(lib.lg_t5_finalize(handle), "lg_t5_finalize")
        except Exception:
            lib.lg_t5_destroy(handle)
            raise
        self._engine, self._engine_sig = handle, sig
        self._ws, self._buckets = None, {}
        return handle

    def _drop_engine(self):
        if self._engine is not None:
            _lib.load().lg_t5_destroy(self._engine)
        self._engine = None
        self._engine_sig = None

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    def buckets(self, T):
        """The int32 bucket table of T tokens on the encoder's device (computed once per T)."""
        dev = self.shared.weight.device
        if (T, dev) not in self._buckets:
            self._buckets[(T, dev)] = bucket_table(T, self.config.num_buckets, self.config.max_distance, dev).contiguous()
        return self._buckets[(T, dev)]

    @torch.no_grad()
    def encode(self, input_ids, attention_mask):
        """last_hidden_state [B, T, d_model] in the parameters' dtype for input_ids / attention_mask [B, T]."""
        handle = self.engine()
        p = self.shared.weight
        if input_ids.dim() != 2 or tuple(attention_mask.shape) != tuple(input_ids.shape):
            raise ValueError(f"input_ids {tuple(input_ids.shape)} and attention_mask {tuple(attention_mask.shape)} must both be [B, T]")
        B, T = input_ids.shape
        if B < 1 or not 1 <= T <= MAX_T:
            raise ValueError(f"B={B} must be >= 1 and T={T} in [1, {MAX_T}]")
        ids = input_ids.to(device=p.device, dtype=torch.int32).contiguous()
        mask = (attention_mask.to(p.device) != 0).to(torch.int32).contiguous()
        if bool(((ids < 0) | (ids >= self.config.vocab_size)).any()):
            raise ValueError(f"input_ids outside [0, {self.config.vocab_size})")
        if bool((mask.sum(dim=1) == 0).any()):
            raise ValueError("every caption needs at least one valid token (an all-zero attention_mask row)")
        lib = _lib.load()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_t5_workspace_bytes(handle, B, T, ctypes.byref(need)), "lg_t5_workspace_bytes")
        if self._ws is None or self._ws.numel() < need.value:
            self._ws = torch.empty(need.value, dtype=torch.uint8, device=p.device)
        out = torch.empty(B, T, self.d_model, dtype=p.dtype, device=p.device)
        _lib.check(lib.lg_t5_encode(handle, _lib.ptr(ids), _lib.ptr(mask), _lib.ptr(self.buckets(T)), B, T, _lib.ptr(self._ws),
                                    self._ws.numel(), _lib.ptr(out), _lib.current_stream(p.device)), "lg_t5_encode")
        return out

    def tokenize(self, prompts):
        if self.tokenizer is None:
            if self.tokenizer_path is None:
                raise ValueError("T5Encoder has no tokenizer: pass tokenizer= or load with from_pretrained")
            from transformers import AutoTokenizer
            self.tokenizer = AutoTokenizer.from_pretrained(self.tokenizer_path)
        t = self.tokenizer(list(prompts), max_length=self.max_length, padding="max_length", truncation=True, return_attention_mask=True,
                           add_special_tokens=True, return_tensors="pt")
        return t["input_ids"], t["attention_mask"]

    def __call__(self, prompts):
        """(embs [B, max_length, d_model], mask [B, max_length]) for a list of caption strings."""
        ids, mask = self.tokenize(prompts)
        dev = self.shared.weight.device
        mask = mask.to(dev)
        return self.encode(ids.to(dev), mask), mask
