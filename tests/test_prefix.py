"""CPU: image completion (generate(..., prefix=tokens)) without a GPU.

* The prefix oracle (one forward over the condition and the prefix, then decoding) gives, at every step k >= P, the logits of the
  oracle's teacher-forced generate() on the same tokens, in fp64, on the tiny golden c2i and t2i models: it is pinned to the path
  that is pinned to the reference.
* attn_plan sends fp8 caches with Tq > 128 from position 0 to the tensor-core causal kernel (kernel 2) for every head shape and
  16-bit dtype; fp8 windows and fp8 prefills of Tq <= 128 plan what they planned before.
* Argument rejections of generate(prefix=...), lg_generate_prefix and the samplers' --prefix-image / --prefix-rows."""
import argparse
import ctypes

import pytest
import torch

from oracle import GPTOracle
from prefix_oracle import prefix_oracle
from util import load_golden

LG_DT = {"f32": 0, "bf16": 1, "f16": 2}
LG_E4M3 = 3


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale, cfg_interval", [(1.0, -1), (4.0, -1), (4.0, 3)])
def test_prefix_oracle_equals_teacher_forced_oracle(name, cfg_scale, cfg_interval):
    g = load_golden(name)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in g["state_dict"].items()}
    cond = g["cond"].double() if g["cond"].is_floating_point() else g["cond"]
    toks = g[f"tokens_cfg{cfg_scale}"]
    S = toks.shape[1]
    kw = dict(emb_masks=g["emb_masks"], cfg_scale=cfg_scale, cfg_interval=cfg_interval, sample_logits=False)
    _, ref = GPTOracle(sd, g["cfg"]).generate(cond, S, teacher=toks, **kw)
    for P in (1, 2, S // 2, S - 1):
        out, logits = prefix_oracle(GPTOracle(sd, g["cfg"]), cond, toks[:, :P], S, teacher=toks, **kw)
        assert torch.equal(out[:, :P], toks[:, :P].to(torch.int32))
        assert (logits[:P] == 0).all()
        assert (logits[P:] - ref[P:]).abs().max().item() <= 1e-5, (name, P)


def _plan(monkeypatch, dt, kv, R, Tq, H, hd, hdp, S, pos_kind=0, value=0):
    from llamagen_b200 import _lib
    lib = _lib.load()
    for k in ("LG_ATTN_TMA", "LG_ATTN_PREFILL_TC", "LG_ATTN_DEEP", "LG_ATTN_NST"):
        monkeypatch.delenv(k, raising=False)
    out = (ctypes.c_int * 3)(-9, -9, -9)
    rc = lib.lg_test_attention_plan(LG_DT[dt], LG_E4M3 if kv == "fp8" else LG_DT[dt], R, Tq, H, hd, hdp, S, 2, pos_kind, value, 0, out)
    assert rc == 0, lib.lg_last_error().decode()
    return tuple(out)


HEADS = [(64, 64), (128, 128), (100, 112)]


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("hd, hdp", HEADS, ids=[f"hd{h}_{p}" for h, p in HEADS])
@pytest.mark.parametrize("Tq", [129, 257, 1143])
def test_fp8_long_prefill_plans_the_causal_tensor_core_kernel(dt, hd, hdp, Tq, monkeypatch):
    R = 58 if Tq == 1143 else 3                      # 58 x 1143 > 65535 query rows: beyond attention_kernel's grid
    assert _plan(monkeypatch, dt, "fp8", R, Tq, 2, hd, hdp, Tq + 7) == (2, 2, 0)
    assert _plan(monkeypatch, dt, "auto", R, Tq, 2, hd, hdp, Tq + 7) == (2, 2, 0)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_fp8_routes_that_stay(dt, monkeypatch):
    # windows (kernel 4's shape) stay on attention_kernel for fp8 caches
    assert _plan(monkeypatch, dt, "fp8", 4, 8, 2, 64, 64, 300, pos_kind=2) == (0, 0, 0)
    assert _plan(monkeypatch, dt, "auto", 4, 8, 2, 64, 64, 300, pos_kind=2) == (4, 2, 0)
    # Tq <= 128 prefill: kernel 3 at hd 64, attention_kernel otherwise
    for Tq in (2, 120, 128):
        assert _plan(monkeypatch, dt, "fp8", 6, Tq, 2, 64, 64, 377) == (3, 1, 0)
        assert _plan(monkeypatch, dt, "fp8", 6, Tq, 2, 128, 128, 377) == (0, 0, 0)
        assert _plan(monkeypatch, dt, "fp8", 6, Tq, 2, 100, 112, 377) == (0, 0, 0)
    # a long block that does not start at position 0 is not a prefill
    assert _plan(monkeypatch, dt, "fp8", 2, 129, 2, 64, 64, 300, pos_kind=0, value=5) == (0, 0, 0)


# ---------------------------------------------------------------------------------------------------------- rejections
class _Model:
    """What generate() reads before it needs a device."""

    def __init__(self):
        from llamagen_b200.gpt import ModelArgs, Transformer
        self.m = Transformer(ModelArgs(n_layer=1, n_head=2, dim=128, vocab_size=512, block_size=16, num_classes=10))


@pytest.mark.parametrize("prefix, kw, msg", [
    (torch.zeros(3, 4, dtype=torch.int64), {}, "[B, P]"),                     # wrong batch
    (torch.zeros(2, dtype=torch.int64), {}, "[B, P]"),                        # 1-D
    (torch.zeros(2, 0, dtype=torch.int64), {}, "prefix length"),              # P = 0
    (torch.zeros(2, 16, dtype=torch.int64), {}, "prefix length"),             # P = S
    (torch.zeros(2, 4), {}, "integer"),                                       # float ids
    (torch.full((2, 4), 512), {}, "vocab_size"),
    (torch.full((2, 4), -1), {}, "vocab_size"),
    (torch.zeros(2, 4, dtype=torch.int64), dict(teacher=torch.zeros(2, 16, dtype=torch.int64)), "teacher"),
    (torch.zeros(2, 4, dtype=torch.int64), dict(sjd_window=4), "sjd_window"),
], ids=["batch", "1d", "p0", "pS", "float", "too_large", "negative", "teacher", "sjd"])
def test_generate_prefix_rejections(prefix, kw, msg):
    from llamagen_b200 import generate
    m = _Model().m
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        generate(m, torch.tensor([1, 2]), 16, prefix=prefix, **kw)


def test_lg_generate_prefix_argument_errors_without_gpu():
    """The checks that need no workspace, on an engine bound to aligned placeholder addresses (never dereferenced)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    D, V, F = 128, 512, 384
    cfg = _lib.ModelCfg(1, 2, D, F, V, 1, 16, 10, 0, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    P_ = ctypes.c_void_p
    try:
        sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 1, 0)

        def call(**kw):
            a = dict(cond=P_(1 << 20), em=None, B=2, T=1, S=16, prefix=P_(2 << 20), P=4, ws=P_(4 << 20), ws_bytes=1 << 40,
                     out=P_(5 << 20))
            a.update(kw)
            rc = lib.lg_generate_prefix(h, a["cond"], a["em"], a["B"], a["T"], a["S"], ctypes.byref(sc), a["prefix"], a["P"], a["ws"],
                                        a["ws_bytes"], a["out"], None, None)
            return rc, lib.lg_last_error().decode()

        rc, err = call()
        assert rc < 0 and "not finalized" in err
        addr, keep = 1 << 24, []
        shapes = {"tok_embeddings.weight": (V, D), "norm.weight": (D,), "output.weight": (V, D),
                  "cls_embedding.embedding_table.weight": (11, D), "freqs_cis": (17, 32, 2),
                  "layers.0.attention.wqkv.weight": (3 * D, D), "layers.0.attention.wo.weight": (D, D),
                  "layers.0.feed_forward.w1.weight": (F, D), "layers.0.feed_forward.w3.weight": (F, D),
                  "layers.0.feed_forward.w2.weight": (D, F), "layers.0.attention_norm.weight": (D,), "layers.0.ffn_norm.weight": (D,)}
        for name, shp in shapes.items():
            arr = _lib.shape_array(shp)
            keep.append(arr)
            dt = _lib.LG_DTYPE_F32 if name == "freqs_cis" else _lib.LG_DTYPE_BF16
            assert lib.lg_engine_bind_weight(h, name.encode(), P_(addr), arr, len(shp), dt) == 0
            addr += 1 << 24
        assert lib.lg_engine_finalize(h) == 0, lib.lg_last_error()
        for kw, msg in [(dict(prefix=None), "null prefix"), (dict(P=0), "outside [1, S - 1]"), (dict(P=16), "outside [1, S - 1]"),
                        (dict(T=2), "cls_token_num"), (dict(em=P_(7 << 20)), "emb_mask"), (dict(cond=None), "null argument"),
                        ({}, "workspace not set")]:
            rc, err = call(**kw)
            assert rc < 0 and msg in err, (kw, rc, err)
        n1, n2 = ctypes.c_size_t(), ctypes.c_size_t()
        assert lib.lg_prefix_workspace_bytes(h, 2, 5, ctypes.byref(n1)) == 0 and lib.lg_prefix_workspace_bytes(h, 8, 5, ctypes.byref(n2)) == 0
        assert 0 < n1.value < n2.value
        assert lib.lg_prefix_workspace_bytes(h, 0, 5, ctypes.byref(n1)) < 0
        chains = ctypes.c_int(-5)
        assert lib.lg_test_prefix_chunks(h, ctypes.byref(chains)) == 0 and chains.value == 0
        assert lib.lg_test_prefix_chunks(h, None) == 0 and lib.lg_test_prefix_chunks(None, None) == -1
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("argv, msg", [
    (["--prefix-rows", "2"], "go together"),
    (["--prefix-image", "IMG"], "go together"),
    (["--prefix-image", "IMG", "--prefix-rows", "0"], "--prefix-rows must lie"),
    (["--prefix-image", "IMG", "--prefix-rows", "16"], "--prefix-rows must lie"),
    (["--prefix-image", "IMG", "--prefix-rows", "2", "--sjd-window", "4"], "sjd-window"),
    (["--prefix-image", "MISSING", "--prefix-rows", "2"], "not a file"),
])
@pytest.mark.parametrize("cli", ["sample_c2i", "sample_t2i"])
def test_cli_prefix_flag_rejections(cli, argv, msg, tmp_path):
    import importlib
    from llamagen_b200.sample.common import check_prefix_args
    mod = importlib.import_module(f"llamagen_b200.sample.{cli}")
    img = tmp_path / "img.png"
    img.write_bytes(b"")
    argv = [str(img) if a == "IMG" else str(tmp_path / "none.png") if a == "MISSING" else a for a in argv]
    args = mod.build_parser().parse_args(["--image-size", "256"] + argv)
    with pytest.raises(SystemExit, match=msg):
        check_prefix_args(args, 16)
    ok = mod.build_parser().parse_args(["--image-size", "256", "--prefix-image", str(img), "--prefix-rows", "15"])
    check_prefix_args(ok, 16)
    check_prefix_args(mod.build_parser().parse_args([]), 16)
