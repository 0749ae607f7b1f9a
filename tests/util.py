import ctypes
import os

import torch

from conftest import GOLDEN


def load_golden(name):
    """A golden case; a state_dict stored as name.sd<i>.pt parts (files stay under 1 MB) is joined back in key order."""
    case = torch.load(os.path.join(GOLDEN, name), map_location="cpu", weights_only=False)
    n = case.pop("state_dict_parts", 0) if isinstance(case, dict) else 0
    if n:
        sd = {}
        for i in range(n):
            sd.update(torch.load(os.path.join(GOLDEN, f"{name[:-3]}.sd{i}.pt"), map_location="cpu", weights_only=False))
        case["state_dict"] = sd
    return case


def build_gpt(cfg: dict, state_dict, dtype, device="cuda"):
    """Instantiate the product Transformer for an arbitrary (tiny) config and load a reference state_dict."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    keys = {k: v for k, v in cfg.items() if k in ModelArgs.__dataclass_fields__}
    m = Transformer(ModelArgs(**keys))
    missing, unexpected = m.load_state_dict(state_dict, strict=False)
    assert not missing and not unexpected, (missing, unexpected)
    return m.to(device=device, dtype=dtype).eval()


def oracle_cfg(model):
    c = model.config
    return dict(n_layer=c.n_layer, n_head=c.n_head, dim=c.dim, norm_eps=c.norm_eps, rope_base=c.rope_base,
                num_classes=c.num_classes, cls_token_num=c.cls_token_num, block_size=c.block_size, model_type=c.model_type)


def cpu_state(model, dtype=None):
    return {k: (v.detach().cpu().to(dtype) if dtype is not None else v.detach().cpu()) for k, v in model.state_dict().items()}


def top2_gap(logits):
    t = torch.topk(logits, 2, dim=-1).values
    return t[..., 0] - t[..., 1]


def test_gemm(x, w):
    """y = x @ w.T through lg_test_gemm (the engine's own GEMM dispatch)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    M, K = x.shape
    N = w.shape[0]
    dt = _lib.LG_DTYPE_BF16 if x.dtype == torch.bfloat16 else _lib.LG_DTYPE_F32
    y = torch.empty(M, N, dtype=torch.float32, device=x.device)
    scratch = torch.empty(16 * M * N + 1024, dtype=torch.float32, device=x.device)
    _lib.check(lib.lg_test_gemm(_lib.ptr(x), _lib.ptr(w), M, N, K, dt, _lib.ptr(y), _lib.ptr(scratch),
                                ctypes.c_size_t(scratch.numel() * 4), _lib.current_stream(x.device)), "lg_test_gemm")
    return y


def seeded_state_dict(shapes: dict, seed: int, fan_in: bool = False) -> dict:
    """Deterministic weights for a parameter layout {name: shape}: N(0, 0.02) for matrices (N(0, 1 / fan_in) with
    `fan_in`, which keeps conv activations at unit scale), 1 + N(0, 0.02) for vectors (norm weights, biases). The golden
    cases built by tests/golden/make_reference_api.py load these into the reference model, so a test can rebuild the
    same model without it."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        t = torch.randn(tuple(shapes[k]), generator=g)
        if t.dim() == 1:
            out[k] = 1.0 + 0.02 * t
        else:
            out[k] = t / (t[0].numel() ** 0.5) if fan_in else 0.02 * t
    return out
