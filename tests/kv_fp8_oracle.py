"""The GPT oracle with an fp8 (e4m3) KV cache: the semantics of `Transformer.set_kv_cache("fp8", scales)`.

At the cache write (gpt.py:183-184) K (after RoPE) and V are stored as e4m3(x / s) * s in the model dtype, with one power-of-two
(k, v) scale per layer; every later read, including the current step's, sees those values. With powers of two in [2^-8, 2^7]
every stored value is exact in bf16 and fp16, so this restates the engine's fp8 cache exactly."""
import torch

from oracle import GPTOracle

E4M3_MAX = 448.0


def e4m3_bytes(x: torch.Tensor, s: float = 1.0) -> torch.Tensor:
    """The stored byte: e4m3_satfinite_rne(float(x) / s) as uint8 (saturating at +-448 instead of torch's NaN past 464)."""
    return (x.float() / s).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def e4m3_values(x: torch.Tensor, s: float = 1.0) -> torch.Tensor:
    """e4m3(x / s) * s in x's dtype (exact for power-of-two s in [2^-8, 2^7])."""
    return ((x.float() / s).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).float() * s).to(x.dtype)


class Fp8Cache:
    """One layer's K (or V) cache of GPTOracle with the fp8 write: `cache[idx] = x` stores e4m3_values(x, s), reads are plain
    tensor indexing. GPTOracle._layer only ever writes `cache[:, :, pos] = x` and reads `cache[:R]`, so it runs unchanged."""

    def __init__(self, tensor: torch.Tensor, scale: float):
        self.tensor, self.scale = tensor, scale

    def __setitem__(self, idx, x):
        self.tensor[idx] = e4m3_values(x, self.scale)

    def __getitem__(self, idx):
        return self.tensor[idx]


class KvFp8Oracle(GPTOracle):
    def __init__(self, state_dict, cfg, kv_fp8_scales=None):
        """kv_fp8_scales: [n_layer, 2] (k, v) per layer, or None for all 1.0."""
        super().__init__(state_dict, cfg)
        n = self.cfg.n_layer
        self.kv_scales = [(1.0, 1.0)] * n if kv_fp8_scales is None else [(float(k), float(v)) for k, v in kv_fp8_scales]

    def setup(self, rows: int, max_seq: int):
        super().setup(rows, max_seq)
        self.k = [Fp8Cache(t, ks) for t, (ks, _) in zip(self.k, self.kv_scales)]
        self.v = [Fp8Cache(t, vs) for t, (_, vs) in zip(self.v, self.kv_scales)]
