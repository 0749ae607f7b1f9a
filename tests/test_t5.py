"""CPU: the T5 encoder's oracle against transformers' outputs (tests/golden/t5_tiny.pt), the bucket table, the checkpoint loader,
the config refusals, lg_t5_workspace_bytes and the lg_t5_* argument checks through the C-ABI (nothing launched), and the
serve.LLM ValueErrors of a text encoder."""
import ctypes
import json
import os
import types

import pytest
import torch

from llamagen_b200 import _lib, serve
from llamagen_b200.t5 import T5Config, T5Encoder, bucket_table, encoder_state_dict
from oracle.t5_oracle import t5_encoder_oracle
from util import load_golden

TINY = dict(num_layers=2, d_model=128, d_kv=64, num_heads=2, d_ff=384, vocab_size=256)
OCFG = dict(num_layers=2, num_heads=2, d_kv=64, num_buckets=32, max_distance=128, eps=1e-6)


@pytest.fixture(scope="module")
def golden():
    return load_golden("t5_tiny.pt")


def test_oracle_reproduces_transformers(golden):
    g = golden
    o32 = t5_encoder_oracle(g["state_dict"], OCFG, g["ids"], g["mask"], torch.float32)
    assert (o32 - g["hidden_fp32"]).abs().max().item() <= 1e-5
    o16 = t5_encoder_oracle(g["state_dict"], OCFG, g["ids"], g["mask"], torch.bfloat16).float()
    # the oracle restates every rounding point of the bf16 forward: at most one bf16 ulp of the output's scale apart
    assert (o16 - g["hidden_bf16"].float()).abs().max().item() <= 2 ** -7 * g["hidden_fp32"].abs().max().item()
    o64 = t5_encoder_oracle(g["state_dict"], OCFG, g["ids"], g["mask"], torch.float64)
    assert (o64.float() - g["hidden_fp32"]).abs().max().item() <= 1e-4


def test_bucket_table_equals_transformers_for_every_T(golden):
    full = golden["buckets"]   # relative positions -511..511
    for T in range(1, 513):
        assert torch.equal(bucket_table(T), full[511 - (T - 1): 511 + T]), T


def _tiny_sd(seed=0):
    m = T5Encoder(T5Config(**TINY))
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(v.shape, generator=g) for k, v in m.state_dict().items()}


def _write_dir(tmp_path, cfg_extra=None):
    c = dict(TINY, relative_attention_num_buckets=32, layer_norm_epsilon=1e-6, feed_forward_proj="gated-gelu")
    c.update(cfg_extra or {})
    (tmp_path / "config.json").write_text(json.dumps(c))
    return tmp_path


def _loaded(path):
    return {k: v.clone() for k, v in T5Encoder.from_pretrained(str(path), dtype=torch.float32, device="cpu").state_dict().items()}


def test_loader_single_safetensors_and_defaults(tmp_path):
    from safetensors.torch import save_file
    sd = _tiny_sd()
    save_file(sd, str(_write_dir(tmp_path) / "model.safetensors"))
    got = _loaded(tmp_path)
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    assert T5Config.from_json(str(tmp_path / "config.json")).max_distance == 128


def test_loader_bin_shards_with_index(tmp_path):
    sd = _tiny_sd(1)
    keys = sorted(sd)
    shards = {"pytorch_model-00001-of-00002.bin": keys[::2], "pytorch_model-00002-of-00002.bin": keys[1::2]}
    _write_dir(tmp_path)
    wmap = {}
    for f, ks in shards.items():
        torch.save({k: sd[k] for k in ks}, str(tmp_path / f))
        wmap.update({k: f for k in ks})
    (tmp_path / "pytorch_model.bin.index.json").write_text(json.dumps({"weight_map": wmap}))
    got = _loaded(tmp_path)
    assert all(torch.equal(got[k], sd[k]) for k in sd)


def test_loader_full_conditional_generation_keys_and_tied_embedding(tmp_path):
    sd = _tiny_sd(2)
    full = dict(sd)
    full["encoder.embed_tokens.weight"] = full.pop("shared.weight")           # tied: only the encoder's name is stored
    full["decoder.block.0.layer.0.SelfAttention.q.weight"] = torch.zeros(3, 3)
    full["lm_head.weight"] = torch.zeros(5, 5)
    assert set(encoder_state_dict(full)) == set(sd)
    torch.save(full, str(_write_dir(tmp_path) / "pytorch_model.bin"))
    got = _loaded(tmp_path)
    assert all(torch.equal(got[k], sd[k]) for k in sd)


def test_loader_raises_on_missing_and_misshaped(tmp_path):
    sd = _tiny_sd(3)
    _write_dir(tmp_path)
    bad = dict(sd)
    del bad["encoder.block.1.layer.1.DenseReluDense.wo.weight"]
    torch.save(bad, str(tmp_path / "pytorch_model.bin"))
    with pytest.raises(KeyError, match="wo.weight"):
        _loaded(tmp_path)
    bad = dict(sd)
    bad["encoder.final_layer_norm.weight"] = torch.ones(64)
    torch.save(bad, str(tmp_path / "pytorch_model.bin"))
    with pytest.raises(ValueError, match="final_layer_norm"):
        _loaded(tmp_path)


@pytest.mark.parametrize("change, dtype, msg", [
    ({}, torch.float16, "fp16"),
    ({"d_kv": 128}, torch.bfloat16, "d_kv=128"),
    ({"feed_forward_proj": "relu"}, torch.bfloat16, "relu"),
])
def test_config_refusals(tmp_path, change, dtype, msg):
    torch.save(_tiny_sd(), str(_write_dir(tmp_path, change) / "pytorch_model.bin"))
    with pytest.raises(ValueError, match=msg):
        T5Encoder.from_pretrained(str(tmp_path), dtype=dtype, device="cpu")


def test_max_length_past_512_refused():
    with pytest.raises(ValueError, match="max_length=513"):
        T5Encoder(T5Config(**TINY), max_length=513)


def _cfg(name, dtype=_lib.LG_DTYPE_BF16, **kw):
    shapes = {"flan-t5-xl": (24, 2048, 64, 32, 5120, 32128), "t5-v1_1-xxl": (24, 4096, 64, 64, 10240, 32128), "tiny": (2, 128, 64, 2, 384, 256)}
    L, D, dk, H, F, V = shapes[name]
    c = dict(n_layer=L, d_model=D, d_kv=dk, n_head=H, d_ff=F, vocab_size=V, num_buckets=32, gated_gelu=1, dtype=dtype, eps=1e-6)
    c.update(kw)
    return _lib.T5Cfg(*c.values())


def _create(cfg):
    lib = _lib.load()
    h = ctypes.c_void_p()
    rc = lib.lg_t5_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    return rc, h, lib.lg_last_error().decode()


# bytes of lg_t5_workspace_bytes: h, xn, qkv, attention output and gated-GELU rows over whole 256-row chunks, plus the largest split-K
# slab of the four GEMM shapes at 256 rows
PINNED = {("flan-t5-xl", 1, 120): 19398656, ("flan-t5-xl", 64, 120): 277872640, ("flan-t5-xl", 8, 512): 153092096,
          ("t5-v1_1-xxl", 1, 120): 38797312, ("t5-v1_1-xxl", 64, 120): 555745280, ("t5-v1_1-xxl", 8, 512): 306184192}


@pytest.mark.parametrize("name, B, T", sorted(PINNED))
def test_workspace_bytes_are_pinned(name, B, T):
    rc, h, err = _create(_cfg(name))
    assert rc == 0, err
    n = ctypes.c_size_t()
    lib = _lib.load()
    assert lib.lg_t5_workspace_bytes(h, B, T, ctypes.byref(n)) == 0, lib.lg_last_error()
    lib.lg_t5_destroy(h)
    assert n.value == PINNED[(name, B, T)], n.value


@pytest.mark.parametrize("kw, msg", [
    (dict(dtype=_lib.LG_DTYPE_F16), "fp16 is not supported"),
    (dict(d_kv=128), "d_kv 128 is not supported"),
    (dict(gated_gelu=0), "gated-gelu"),
    (dict(d_model=100), "d_model 100"),
])
def test_create_refusals(kw, msg):
    rc, _, err = _create(_cfg("tiny", **kw))
    assert rc < 0 and msg in err, err


def test_argument_checks_without_launch():
    lib = _lib.load()
    rc, h, err = _create(_cfg("tiny"))
    assert rc == 0, err
    n = ctypes.c_size_t()
    assert lib.lg_t5_workspace_bytes(h, 1, 513, ctypes.byref(n)) < 0 and "T=513" in lib.lg_last_error().decode()
    assert lib.lg_t5_workspace_bytes(h, 0, 8, ctypes.byref(n)) < 0
    fake = ctypes.c_void_p(1 << 20)
    assert lib.lg_t5_encode(h, fake, fake, fake, 1, 8, fake, 1 << 30, fake, None) < 0
    assert "lg_t5_finalize first" in lib.lg_last_error().decode()
    assert lib.lg_t5_bind_weight(h, b"shared.weight", fake, _lib.shape_array((256, 128)), 2, _lib.LG_DTYPE_BF16) == 0
    assert lib.lg_t5_finalize(h) < 0 and "missing weight 'encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight'" in \
        lib.lg_last_error().decode()
    assert lib.lg_t5_bind_weight(h, b"shared.weight", fake, _lib.shape_array((256, 64)), 2, _lib.LG_DTYPE_BF16) == 0
    assert lib.lg_t5_finalize(h) < 0 and "'shared.weight' dim 1 is 64, expected 128" in lib.lg_last_error().decode()
    lib.lg_t5_destroy(h)
    # every weight bound (fake addresses): finalize checks names, shapes and alignment on the host and copies nothing, so the checks
    # of lg_t5_encode that need a ready encoder run here too
    rc, h, err = _create(_cfg("tiny"))
    D, I, F, V = 128, 128, 384, 256
    shapes = {"shared.weight": (V, D), "encoder.final_layer_norm.weight": (D,),
              "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (32, 2)}
    for i in range(2):
        p = f"encoder.block.{i}.layer."
        shapes.update({p + "0.SelfAttention.q.weight": (I, D), p + "0.SelfAttention.k.weight": (I, D), p + "0.SelfAttention.v.weight": (I, D),
                       p + "0.SelfAttention.o.weight": (D, I), p + "0.layer_norm.weight": (D,), p + "1.layer_norm.weight": (D,),
                       p + "1.DenseReluDense.wi_0.weight": (F, D), p + "1.DenseReluDense.wi_1.weight": (F, D),
                       p + "1.DenseReluDense.wo.weight": (D, F)})
    for name, shape in shapes.items():
        assert lib.lg_t5_bind_weight(h, name.encode(), fake, _lib.shape_array(shape), len(shape), _lib.LG_DTYPE_BF16) == 0
    assert lib.lg_t5_finalize(h) == 0, lib.lg_last_error()
    assert lib.lg_t5_workspace_bytes(h, 2, 8, ctypes.byref(n)) == 0
    ws = ctypes.c_void_p(1 << 24)
    for args, msg in [((2, 0, ws, n.value), "T=0"), ((2, 513, ws, 1 << 40), "T=513"), ((0, 8, ws, n.value), "B=0"),
                      ((2, 8, ctypes.c_void_p((1 << 24) + 16), n.value), "not 256-byte aligned"),
                      ((2, 8, ws, n.value - 1), f"workspace {n.value - 1} < {n.value}")]:
        B, T, w, nb = args
        assert lib.lg_t5_encode(h, fake, fake, fake, B, T, w, nb, fake, None) < 0
        assert msg in lib.lg_last_error().decode(), (args, lib.lg_last_error())
    assert lib.lg_t5_encode(h, None, fake, fake, 2, 8, ws, n.value, fake, None) < 0 and "null argument" in lib.lg_last_error().decode()
    lib.lg_t5_destroy(h)
    for args, msg in [((_lib.LG_DTYPE_F16, 1, 8, 2), "dtype 2"), ((_lib.LG_DTYPE_BF16, 1, 513, 2), "T=513"),
                      ((_lib.LG_DTYPE_BF16, 0, 8, 2), "B=0")]:
        assert lib.lg_test_t5_attention(*args, fake, fake, fake, fake, 32, fake, None, None) < 0
        assert msg in lib.lg_last_error().decode(), (args, lib.lg_last_error())


# ------------------------------------------------------------------------------------------------ serve.LLM with a text encoder
def _gpt(model_type="t2i", C=4):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=64,
                                 cls_token_num=6 if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None)


class _StubEncoder:
    d_model = 4

    def __init__(self):
        self.calls = []

    def __call__(self, prompts):
        self.calls.append(list(prompts))
        n = [len(p.split()) for p in prompts]
        mask = (torch.arange(6)[None, :] < torch.tensor(n)[:, None]).long()
        return torch.randn(len(prompts), 6, 4) * mask[:, :, None], mask


def test_serve_text_encoder_errors():
    with pytest.raises(ValueError, match="caption_dim"):
        serve.LLM(_gpt(C=8), text_encoder=_StubEncoder())
    with pytest.raises(ValueError, match="t2i"):
        serve.LLM(_gpt("c2i"), text_encoder=_StubEncoder())
    llm = serve.LLM(_gpt(), text_encoder=_StubEncoder())
    with pytest.raises(ValueError, match="not both"):
        llm.generate(prompts=["a cat"], prompt_embeds=[torch.zeros(2, 4)])
    with pytest.raises(ValueError, match="not both"):
        llm.add_request(prompt="a cat", prompt_embeds=torch.zeros(2, 4))
    with pytest.raises(ValueError, match="no tokenizer"):
        serve.LLM(_gpt()).generate(prompts=["a cat"])
    with pytest.raises(ValueError, match="no tokenizer"):
        serve.LLM(_gpt()).add_request(prompt="a cat")


def test_serve_prompts_enqueue_their_valid_feature_rows(monkeypatch):
    enc = _StubEncoder()
    llm = serve.LLM(_gpt(), text_encoder=enc, max_num_seqs=4)
    seen = []
    monkeypatch.setattr(serve.LLM, "_caption", lambda self, f: seen.append(f) or (torch.zeros(6, 4), torch.zeros(6)))
    llm.add_request(prompt="one two three")
    assert enc.calls == [["one two three"]] and seen[0].shape == (3, 4)
    llm._waiting.clear()
    feats = []
    monkeypatch.setattr(serve.LLM, "_enqueue_t2i", lambda self, c, p, pf: feats.append(c))
    llm.generate(prompts=["a", "b c d e", "f g"])
    assert enc.calls[1] == ["a", "b c d e", "f g"]   # one encoder call for the batch
    assert [s.shape[0] for s in seen[1:]] == [1, 4, 2]
