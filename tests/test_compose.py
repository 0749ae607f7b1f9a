"""CPU: composable guidance (generate(..., cond_weights=)) without a GPU.

* The compose oracle is pinned in fp64 on the golden models: K = 1 with weight s is GPTOracle.generate(cfg_scale=s) (with and
  without cfg_interval) and, on t2i, negative_oracle; a zero-weight condition drops out of tokens and logits exactly, in either place.
* Every ValueError of generate(cond_weights=...): shapes, K bounds, non-finite weights, class range, cfg_scale / cfg_interval /
  sjd_window / teacher / return_logits, and the existing given / prefix / logprobs exclusions.
* lg_generate_composed's argument checks on a placeholder engine, and the samplers' --compose-* flags."""
import ctypes

import pytest
import torch

from compose_oracle import compose_oracle
from negative_oracle import negative_oracle
from oracle import GPTOracle
from util import load_golden


def _sd64(g):
    sd = {k: v.double() if v.is_floating_point() else v for k, v in g["state_dict"].items()}
    cond = g["cond"].double() if g["cond"].is_floating_point() else g["cond"]
    return sd, cond


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("s, cfg_interval", [(4.0, -1), (7.5, 3), (1.5, -1)])
def test_k1_is_cfg(name, s, cfg_interval):
    g = load_golden(name)
    sd, cond = _sd64(g)
    S = g["S"]
    em = g["emb_masks"]
    kw = dict(cfg_interval=cfg_interval, sample_logits=False)
    want, wl = GPTOracle(sd, g["cfg"]).generate(cond, S, emb_masks=em, cfg_scale=s, **kw)
    got, gl = compose_oracle(GPTOracle(sd, g["cfg"]), cond[:, None], [s], S, emb_masks=None if em is None else em[:, None], **kw)
    assert torch.equal(got, want.to(torch.int32)) and torch.equal(gl, wl)


def test_k1_is_negative_oracle():
    g = load_golden("gpt_t2i.pt")
    sd, cond = _sd64(g)
    S, em = g["S"], g["emb_masks"]
    B, T, C = cond.shape
    neg = 0.5 * torch.randn(1, T, C, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    nm = torch.ones(1, T)
    nm[:, :30] = 0
    for nmask in (nm, None):
        want, wl = negative_oracle(GPTOracle(sd, g["cfg"]), cond, neg, S, emb_masks=em, negative_emb_masks=nmask, cfg_scale=4.0,
                                   sample_logits=False)
        got, gl = compose_oracle(GPTOracle(sd, g["cfg"]), cond[:, None], [4.0], S, emb_masks=em[:, None], negative=neg,
                                 negative_emb_masks=nmask, sample_logits=False)
        assert torch.equal(got, want) and torch.equal(gl, wl)


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_zero_weight_drops_its_condition(name):
    g = load_golden(name)
    sd, cond = _sd64(g)
    S, em = g["S"], g["emb_masks"]
    B = cond.shape[0]
    if g["cfg"]["model_type"] == "c2i":
        other = (cond + 5) % g["cfg"]["num_classes"]
        em1 = em2 = None
    else:
        other = 0.5 * torch.randn(cond.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
        em1 = em[:, None]
        em2 = torch.stack([em, em], 1)            # u attends with condition 1's mask: keep it the caption's in both orders
    w = torch.tensor([[4.0], [2.5]]).repeat(B // 2 + 1, 1)[:B].double()
    want, wl = compose_oracle(GPTOracle(sd, g["cfg"]), cond[:, None], w, S, emb_masks=em1, sample_logits=False)
    for pair, wz, e in ((torch.stack([cond, other], 1), torch.cat([w, 0 * w], 1), em2),
                        (torch.stack([other, cond], 1), torch.cat([0 * w, w], 1), em2)):
        got, gl = compose_oracle(GPTOracle(sd, g["cfg"]), pair, wz, S, emb_masks=e, sample_logits=False)
        assert torch.equal(got, want) and torch.equal(gl, wl)


# ------------------------------------------------------------------------------------------------------------------- errors
def _gpt(model_type):
    from llamagen_b200.gpt import ModelArgs, Transformer
    return Transformer(ModelArgs(n_layer=1, n_head=2, dim=64, vocab_size=32, block_size=16, cls_token_num=4 if model_type == "t2i" else 1,
                                 model_type=model_type, caption_dim=16, num_classes=10))


_C = torch.tensor([[1, 2], [3, 4]])
_T = torch.zeros(2, 2, 4, 16)
_W = [4.0, -1.0]


@pytest.mark.parametrize("kind, cond, kw, msg", [
    ("c2i", _C, dict(cfg_scale=4.0), "cfg_scale"),
    ("c2i", _C, dict(cfg_interval=3), "cfg_interval"),
    ("c2i", _C, dict(sjd_window=4), "sjd_window"),
    ("c2i", _C, dict(teacher=torch.zeros(2, 8, dtype=torch.long)), "teacher"),
    ("c2i", _C, dict(return_logits=True), "return_logits"),
    ("c2i", _C, dict(cond_weights=[1.0] * 9), "K=9"),
    ("c2i", torch.zeros(2, 0, dtype=torch.long), dict(cond_weights=[]), "K=0"),
    ("c2i", _C, dict(cond_weights=[float("nan"), 1.0]), "finite"),
    ("c2i", _C, dict(cond_weights=[float("inf"), 1.0]), "finite"),
    ("c2i", _C, dict(cond_weights=[1e39, 1.0]), "finite"),
    ("c2i", _C, dict(cond_weights=[True, False]), "real numbers"),
    ("c2i", _C, dict(cond_weights=torch.ones(2, 2, 2)), r"\[K\] or \[B, K\]"),
    ("c2i", _C, dict(cond_weights=torch.ones(3, 2)), r"\[K\] or \[B, K\]"),
    ("c2i", _C, dict(cond_weights=[1.0, 2.0, 3.0]), r"\[B, K\]"),
    ("c2i", torch.tensor([1, 2]), {}, r"\[B, K\]"),
    ("c2i", _C.float(), {}, "integer"),
    ("c2i", torch.tensor([[1, 10], [3, 4]]), {}, "num_classes"),
    ("c2i", torch.tensor([[1, -1], [3, 4]]), {}, "num_classes"),
    ("c2i", _C, dict(emb_masks=torch.ones(2, 2, 1)), "t2i"),
    ("t2i", torch.zeros(2, 4, 16), {}, r"\[B, K, T, C\]"),
    ("t2i", torch.zeros(2, 2, 5, 16), {}, r"\[B, K, T, C\]"),
    ("t2i", torch.zeros(2, 2, 4, 8), {}, r"\[B, K, T, C\]"),
    ("t2i", _T, dict(emb_masks=torch.ones(2, 4)), "emb_masks"),
    ("t2i", _T, dict(emb_masks=torch.ones(2, 3, 4)), "emb_masks"),
    ("t2i", _T, dict(negative_cond=torch.zeros(3, 4, 16)), "negative_cond"),
    ("t2i", _T, dict(negative_cond=torch.zeros(1, 4, 8)), "negative_cond"),
    ("t2i", _T, dict(negative_emb_masks=torch.ones(1, 4)), "needs negative_cond"),
    ("t2i", _T, dict(negative_cond=torch.zeros(1, 4, 16), negative_emb_masks=torch.ones(1, 5)), "negative_emb_masks"),
    ("c2i", _C, dict(prefix=torch.zeros(2, 3, dtype=torch.long), given=torch.zeros(2, 8, dtype=torch.long),
                     given_mask=torch.zeros(8, dtype=torch.bool)), "prefix"),
    ("c2i", _C, dict(return_logprobs=True, given=torch.zeros(2, 8, dtype=torch.long), given_mask=torch.zeros(8, dtype=torch.bool)),
     "return_logprobs"),
    ("c2i", _C, dict(prefix=torch.zeros(2, 8, dtype=torch.long)), "prefix length"),
    ("c2i", _C, dict(prefix=torch.full((2, 3), 99)), "vocab_size"),
    ("c2i", _C, dict(given=torch.zeros(2, 8, dtype=torch.long), given_mask=torch.ones(8, dtype=torch.bool)), "at least one"),
    ("c2i", _C, dict(top_logprobs=3), "return_logprobs"),
], ids=lambda v: None)
def test_generate_compose_rejections(kind, cond, kw, msg):
    from llamagen_b200 import generate
    kw = dict(kw)
    w = kw.pop("cond_weights", _W)
    with pytest.raises(ValueError, match=msg):
        generate(_gpt(kind), cond, 8, cond_weights=w, **kw)


def test_lg_generate_composed_argument_errors_without_gpu():
    """The checks that need no workspace, on an engine bound to aligned placeholder addresses (never dereferenced)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    D, V, F = 128, 512, 384
    cfg = _lib.ModelCfg(1, 2, D, F, V, 1, 16, 10, 0, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    P_ = ctypes.c_void_p
    try:
        def call(**kw):
            a = dict(cond=P_(1 << 20), em=None, neg=None, nm=None, B=2, K=2, T=1, S=16, interval=-1, w=P_(2 << 20), prefix=None, P=0,
                     given=None, ws=P_(4 << 20), ws_bytes=1 << 40, lp=None, out=P_(5 << 20))
            a.update(kw)
            sc = _lib.SampleCfg(1.0, a["interval"], 1.0, 0, 1.0, 1, 0)
            g = a["given"]
            rc = lib.lg_generate_composed(h, a["cond"], a["em"], a["neg"], a["nm"], a["B"], a["K"], a["T"], a["S"], ctypes.byref(sc), a["w"],
                                          a["prefix"], a["P"], None if g is None else _lib.ptr(g), a["ws"], a["ws_bytes"], a["lp"],
                                          a["out"], None)
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
        given = torch.full((4, 16), -1, dtype=torch.int32)
        given[:, :3] = 7
        split = given.clone()
        split[1, 2] = 8                                          # row 1 of image 0 disagrees with its row 0
        bad_lp = _lib.Logprobs(0, 0, 0, 0, 21)
        for kw, msg in [(dict(w=None), "null cond, sc, weights"), (dict(cond=None), "null cond"), (dict(out=None), "null cond"),
                        (dict(K=0), "K=0"), (dict(K=9), "K=9"), (dict(B=0), "B=0"), (dict(interval=3), "cfg_interval=3"),
                        (dict(P=3), "prefix length P=3"), (dict(prefix=P_(6 << 20)), "prefix length P=0"), (dict(P=16, prefix=P_(6 << 20)), "P=16"),
                        (dict(given=given, P=2, prefix=P_(6 << 20)), "no prefix"), (dict(lp=ctypes.byref(bad_lp)), "top_n=21"),
                        (dict(given=split), "differs from its row 0"), (dict(T=2), "cls_token_num"), (dict(em=P_(7 << 20)), "emb_mask"),
                        (dict(neg=P_(8 << 20)), "t2i models only"), ({}, "workspace not set")]:
            rc, err = call(**kw)
            assert rc < 0 and msg in err, (kw, rc, err)
        rc, err = call(K=1, interval=3)                          # K = 1 keeps cfg_interval
        assert rc < 0 and "workspace not set" in err
    finally:
        lib.lg_engine_destroy(h)


# ------------------------------------------------------------------------------------------------------------------- CLI
def test_cli_compose_flags_parse_and_map_to_generate(tmp_path):
    from llamagen_b200.sample import sample_c2i, sample_c2i_ddp, sample_t2i, sample_t2i_ddp
    from llamagen_b200.sample.common import (check_compose_args, compose_caption_cond, compose_class_cond, compose_entries,
                                             guidance_kwargs)
    for mod in (sample_c2i, sample_c2i_ddp):
        plain = mod.build_parser().parse_args([])
        check_compose_args(plain, 1000)
        assert guidance_kwargs(plain) == {"cfg_scale": 4.0, "cfg_interval": -1}
        labels = torch.tensor([1, 2, 3])
        assert compose_class_cond(plain, labels) is labels
        args = mod.build_parser().parse_args(["--compose-class", "5", "0.6", "--compose-class", "9", "-1.5", "--cfg-scale", "3"])
        check_compose_args(args, 1000)
        assert guidance_kwargs(args) == {"cond_weights": [3.0, 0.6, -1.5]}
        assert torch.equal(compose_class_cond(args, labels), torch.tensor([[1, 5, 9], [2, 5, 9], [3, 5, 9]]))
    npy = tmp_path / "f.npy"
    npy.write_bytes(b"")
    for mod in (sample_t2i, sample_t2i_ddp):
        plain = mod.build_parser().parse_args([])
        assert compose_entries(plain) == [] and guidance_kwargs(plain, cfg_interval=False) == {"cfg_scale": 7.5}
        args = mod.build_parser().parse_args(["--compose-prompt", "watercolor", "0.6", "--compose-cond-npy", str(npy), "-2"])
        check_compose_args(args)
        assert guidance_kwargs(args, cfg_interval=False) == {"cond_weights": [7.5, 0.6, -2.0]}
    c, m = torch.zeros(3, 4, 8), torch.ones(3, 4)
    assert compose_caption_cond(c, m, []) == (c, m)
    cc, mm = compose_caption_cond(c, m, [(torch.ones(1, 4, 8), torch.zeros(1, 4))])
    assert cc.shape == (3, 2, 4, 8) and mm.shape == (3, 2, 4) and cc[:, 1].eq(1).all() and mm[:, 1].eq(0).all()


@pytest.mark.parametrize("argv, msg", [
    (["--compose-class", "5", "x"], "not a number"),
    (["--compose-class", "5", "inf"], "not finite"),
    (["--compose-class", "5", "1e39"], "not finite"),
    (["--compose-class", "five", "1"], "not an integer"),
    (["--compose-class", "1000", "1"], r"\[0, 1000\)"),
    (["--compose-class", "-1", "1"], r"\[0, 1000\)"),
    (["--compose-class", "5", "1", "--sjd-window", "4"], "sjd-window"),
    (["--compose-class", "5", "1", "--cfg-interval", "3"], "cfg-interval"),
    (sum((["--compose-class", str(i), "1"] for i in range(8)), []), "at most 7"),
])
def test_cli_compose_class_rejections(argv, msg):
    from llamagen_b200.sample import sample_c2i
    from llamagen_b200.sample.common import check_compose_args
    with pytest.raises(SystemExit, match=msg):
        check_compose_args(sample_c2i.build_parser().parse_args(argv), 1000)


def test_cli_compose_prompt_rejections(tmp_path):
    from llamagen_b200.sample import sample_t2i
    from llamagen_b200.sample.common import check_compose_args, compose_caption_features
    p = sample_t2i.build_parser()
    with pytest.raises(SystemExit, match="not a file"):
        check_compose_args(p.parse_args(["--compose-cond-npy", str(tmp_path / "none.npy"), "1"]))
    with pytest.raises(SystemExit, match="not a number"):
        check_compose_args(p.parse_args(["--compose-prompt", "a cat", "heavy"]))
    with pytest.raises(SystemExit, match="text encoder"):
        compose_caption_features(p.parse_args(["--compose-prompt", "a cat", "1"]), None, "cpu", torch.float32)
    # without --compose-* a negative still needs --cfg-scale > 1; with them the composed call always mixes
    with pytest.raises(SystemExit, match="cfg-scale > 1"):
        sample_t2i.check_negative_args(p.parse_args(["--negative-prompt", "blurry", "--cfg-scale", "1"]))
    sample_t2i.check_negative_args(p.parse_args(["--negative-prompt", "blurry", "--cfg-scale", "1", "--compose-prompt", "a", "2"]))
