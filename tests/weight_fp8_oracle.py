"""fp8 (e4m3) GEMM weights in torch: the semantics of `Transformer.set_weight_dtype("fp8")`.

A weight W [N, K] of a bf16 / fp16 model is stored as e4m3 codes with one power-of-two scale per output row,
    s_n = 2^e with max_k |W[n, k]| / s_n in (224, 448], e clamped to [-15, 7] (fp16) / [-64, 64] (bf16), 1 for a zero row,
    code[n, k] = e4m3_satfinite_rne(float(W[n, k]) / s_n),
and the layer computes s_n * sum_k x[r, k] * code[n, k]. code * s_n is exact in bf16 and in fp16, so the unmodified GPTOracle on
`dequantized_state_dict` restates the engine exactly (up to the order of the fp32 sums)."""
import torch

from kv_fp8_oracle import E4M3_MAX

EXPONENTS = {torch.float16: (-15, 7), torch.bfloat16: (-64, 64)}
LAYER_WEIGHTS = ("attention.wqkv.weight", "attention.wo.weight", "feed_forward.w1.weight", "feed_forward.w3.weight",
                 "feed_forward.w2.weight")


def row_scales(W: torch.Tensor, dtype) -> torch.Tensor:
    """fp32 [N]: the power-of-two scale of every row of W (values as the model dtype holds them)."""
    amax = W.to(dtype).float().abs().amax(dim=1)
    m, ex = torch.frexp(amax)                               # amax = m * 2^ex, m in [0.5, 1); 448 = 0.875 * 2^9
    e = torch.where(m <= 0.875, ex - 9, ex - 8).clamp(*EXPONENTS[dtype])
    e = torch.where(amax > 0, e, torch.zeros_like(e))
    return torch.ldexp(torch.ones_like(amax), e)


def quantize_rows(W: torch.Tensor, dtype):
    """(codes uint8 [N, K] with column k at index k, scales fp32 [N]) of W in the model dtype."""
    s = row_scales(W, dtype)
    x = W.to(dtype).float() / s[:, None]
    return x.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8), s


def code_values(codes: torch.Tensor) -> torch.Tensor:
    """fp32 values of e4m3 codes."""
    return codes.view(torch.float8_e4m3fn).float()


def dequantize(codes: torch.Tensor, scales: torch.Tensor, dtype) -> torch.Tensor:
    """code * s in the model dtype (exact)."""
    return (code_values(codes) * scales[:, None]).to(dtype)


def fp8_names(state_dict, head: bool = True):
    names = [k for k in state_dict if k.startswith("layers.") and k.split(".", 2)[2] in LAYER_WEIGHTS]
    return names + ["output.weight"] if head else names


def dequantized_state_dict(sd, dtype, head: bool = True, out_dtype=None):
    """sd with every fp8-stored weight replaced by code * s as a model of `dtype` stores it; every floating-point tensor is then
    cast to out_dtype (default: left as it is; fp32 for the ref32 oracle - the values are the same)."""
    out = {k: v.clone() for k, v in sd.items()}
    for k in fp8_names(sd, head):
        codes, s = quantize_rows(sd[k], dtype)
        out[k] = dequantize(codes, s, dtype)
    if out_dtype is not None:
        out = {k: v.to(out_dtype) if v.is_floating_point() else v for k, v in out.items()}
    return out
