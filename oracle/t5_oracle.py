"""T5 encoder oracle — TEST INFRASTRUCTURE ONLY.

A functional torch restatement of transformers' T5EncoderModel forward (T5LayerNorm, T5Attention without 1/sqrt(d), relative
position bias of block 0 shared by every layer, gated-GELU feed-forward) with HuggingFace's rounding points: every op output is a
tensor of the run dtype, T5LayerNorm takes its variance in fp32 and rounds before the weight, softmax runs in fp32 and its result
is rounded back, NewGELUActivation is evaluated op by op in the run dtype. dtype torch.float64 runs everything in fp64 (the
variance and softmax too). Pinned to transformers' outputs by tests/test_t5.py over tests/golden/t5_tiny.pt."""
from __future__ import annotations

import math

import torch


def relative_position_bucket(rel, num_buckets=32, max_distance=128):
    """transformers' bidirectional T5Attention._relative_position_bucket."""
    num_buckets //= 2
    ret = (rel > 0).to(torch.long) * num_buckets
    n = torch.abs(rel)
    max_exact = num_buckets // 2
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return ret + torch.where(n < max_exact, n, large)


def _norm(x, w, eps, acc):
    var = x.to(acc).pow(2).mean(-1, keepdim=True)
    y = x * torch.rsqrt(var + eps)
    return w * y.to(w.dtype)


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def t5_encoder_oracle(sd, cfg, input_ids, attention_mask, dtype=torch.float32, buckets=None):
    """last_hidden_state [B, T, d_model] in `dtype`. sd: HF encoder state dict (shared.weight, encoder.*); cfg: dict with
    num_layers, num_heads, d_kv, num_buckets, max_distance, eps. buckets: optional [T, T] bucket matrix to use instead of the CPU
    one (a device-computed table)."""
    acc = torch.float64 if dtype == torch.float64 else torch.float32
    w = {k: v.to(dtype) for k, v in sd.items()}
    B, T = input_ids.shape
    H, dk, eps = cfg["num_heads"], cfg["d_kv"], cfg["eps"]
    h = w["shared.weight"][input_ids.long()]
    if buckets is None:
        pos = torch.arange(T)   # on the CPU, as transformers computes it for a CPU model
        buckets = relative_position_bucket(pos[None, :] - pos[:, None], cfg["num_buckets"], cfg["max_distance"])
    buckets = buckets.to(input_ids.device)
    bias = w["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"][buckets.long()].permute(2, 0, 1)[None]
    ext = (1.0 - attention_mask[:, None, None, :].to(dtype)) * torch.finfo(dtype).min
    pb = bias + ext
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer."
        x = _norm(h, w[p + "0.layer_norm.weight"], eps, acc)

        def heads(n):
            return (x @ w[p + f"0.SelfAttention.{n}.weight"].t()).view(B, T, H, dk).transpose(1, 2)
        q, k, v = heads("q"), heads("k"), heads("v")
        scores = q @ k.transpose(3, 2)
        scores = scores + pb
        attn = torch.softmax(scores.to(acc), dim=-1).to(dtype)
        o = (attn @ v).transpose(1, 2).reshape(B, T, H * dk)
        h = h + o @ w[p + "0.SelfAttention.o.weight"].t()
        x = _norm(h, w[p + "1.layer_norm.weight"], eps, acc)
        g = _gelu_new(x @ w[p + "1.DenseReluDense.wi_0.weight"].t())
        y = (g * (x @ w[p + "1.DenseReluDense.wi_1.weight"].t())) @ w[p + "1.DenseReluDense.wo.weight"].t()
        h = h + y
    return _norm(h, w["encoder.final_layer_norm.weight"], eps, acc)
