"""CPU: the scoring C-ABI (lg_score_workspace_bytes / lg_score) without a GPU, the teacher-forced scoring oracle against the
reference's golden logits, the t2i attention-mask -> emb_masks derivation and the code-directory parsing of the score_c2i CLI."""
import ctypes
import json

import numpy as np
import pytest
import torch

from oracle import GPTOracle
from score_oracle import score_oracle
from util import load_golden

_GPT_L = dict(n_layer=24, n_head=16, dim=1024, ffn_dim=2816, vocab_size=16384, cls_token_num=1, num_classes=1000, caption_dim=0)
_TINY_T2I = dict(n_layer=2, n_head=4, dim=256, ffn_dim=704, vocab_size=1024, cls_token_num=8, num_classes=0, caption_dim=64)
_TINY_HD100 = dict(n_layer=2, n_head=2, dim=200, ffn_dim=544, vocab_size=1024, cls_token_num=1, num_classes=10, caption_dim=0)


def _engine(m, t2i, dtype):
    from llamagen_b200 import _lib
    lib = _lib.load()
    cfg = _lib.ModelCfg(m["n_layer"], m["n_head"], m["dim"], m["ffn_dim"], m["vocab_size"], m["cls_token_num"], 256, m["num_classes"],
                        m["caption_dim"], _lib.LG_MODEL_T2I if t2i else _lib.LG_MODEL_C2I, dtype, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
    return lib, h


@pytest.mark.parametrize("m, t2i, sizes", [
    (_GPT_L, False, {(64, 256): 662700032, (128, 256): 1325400064, (2, 17): 2894848}),
    # ffn_dim 704: the w1 | w3 boundary is not on a 128-row tile, so that GEMM plans mma.sync (one slab) instead of wgmma (two)
    (_TINY_T2I, True, {(2, 9): 207616, (16, 263): 42584064}),
    (_TINY_HD100, False, {(2, 17): 413952, (128, 256): 260046848}),                    # 112-wide K / V rows
], ids=["c2i_gpt_l", "t2i_tiny_ffn704", "c2i_hd100"])
def test_score_workspace_bytes_are_pinned(m, t2i, sizes, monkeypatch):
    """lg_score's scratch (one layer of K / V, activations and GEMM partials of rows * seq positions, the caption MLP, one head
    chunk) is host arithmetic: its size, computed without a GPU, must not move. The GEMM partials follow the default GEMM plan."""
    from llamagen_b200 import _lib
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    lib, h = _engine(m, t2i, _lib.LG_DTYPE_BF16)
    try:
        got = {}
        for rows, seq in sizes:
            n = ctypes.c_size_t()
            assert lib.lg_score_workspace_bytes(h, rows, seq, ctypes.byref(n)) == 0, lib.lg_last_error()
            got[(rows, seq)] = n.value
        assert got == sizes
        n = ctypes.c_size_t()
        assert lib.lg_score_workspace_bytes(h, 2, m["cls_token_num"] + 256, ctypes.byref(n)) < 0       # seq past T + block_size - 1
        assert b"seq" in lib.lg_last_error()
    finally:
        lib.lg_engine_destroy(h)


def test_score_argument_errors_without_gpu():
    """Every argument is checked before any launch; the engine is bound to aligned placeholder addresses (never dereferenced)."""
    from llamagen_b200 import _lib
    m = dict(_GPT_L, n_layer=1)
    lib, h = _engine(m, False, _lib.LG_DTYPE_BF16)
    P = ctypes.c_void_p
    try:
        def call(**kw):
            a = dict(cond=P(1 << 20), em=None, idx=P(2 << 20), tg=P(3 << 20), B=2, T=1, S=16, cfg=0, scale=1.0, ws=P(4 << 20),
                     ws_bytes=1 << 40, logits=P(5 << 20), nll=P(6 << 20))
            a.update(kw)
            rc = lib.lg_score(h, a["cond"], a["em"], a["idx"], a["tg"], a["B"], a["T"], a["S"], a["cfg"], a["scale"], a["ws"],
                              a["ws_bytes"], a["logits"], a["nll"], None)
            return rc, lib.lg_last_error().decode()

        rc, err = call()
        assert rc < 0 and "not finalized" in err
        addr = 1 << 24
        keep = []
        shapes = {"tok_embeddings.weight": (16384, 1024), "norm.weight": (1024,), "output.weight": (16384, 1024),
                  "cls_embedding.embedding_table.weight": (1001, 1024), "freqs_cis": (257, 32, 2),
                  "layers.0.attention.wqkv.weight": (3072, 1024), "layers.0.attention.wo.weight": (1024, 1024),
                  "layers.0.feed_forward.w1.weight": (2816, 1024), "layers.0.feed_forward.w3.weight": (2816, 1024),
                  "layers.0.feed_forward.w2.weight": (1024, 2816), "layers.0.attention_norm.weight": (1024,),
                  "layers.0.ffn_norm.weight": (1024,)}
        for name, shp in shapes.items():
            arr = _lib.shape_array(shp)
            keep.append(arr)
            dt = _lib.LG_DTYPE_F32 if name == "freqs_cis" else _lib.LG_DTYPE_BF16
            assert lib.lg_engine_bind_weight(h, name.encode(), P(addr), arr, len(shp), dt) == 0
            addr += 1 << 24
        assert lib.lg_engine_finalize(h) == 0, lib.lg_last_error()
        for kw, msg in [(dict(cond=None), "cond"), (dict(B=0), "cond"), (dict(T=2), "cls_token_num"), (dict(S=0), "block_size"),
                        (dict(S=257), "block_size"), (dict(idx=None), "idx"), (dict(S=1), "idx"),
                        (dict(logits=None, nll=None), "nothing to write"), (dict(tg=None), "needs targets"),
                        (dict(em=P(7 << 20)), "emb_mask"), (dict(cfg=1, scale=float("inf")), "finite"), (dict(ws=None), "aligned"),
                        (dict(ws=P((4 << 20) + 16)), "aligned"), (dict(ws_bytes=1 << 20), "too small")]:
            rc, err = call(**kw)
            assert rc < 0 and msg in err, (kw, rc, err)
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
def test_score_oracle_reproduces_golden_logits(name, cfg_scale):
    """One teacher-forced pass of the oracle gives the logits the reference's generate() produced step by step."""
    g = load_golden(name)
    toks = g[f"tokens_cfg{cfg_scale}"]
    logits, nll = score_oracle(GPTOracle(g["state_dict"], g["cfg"]), g["cond"], toks, g["emb_masks"], cfg_scale)
    ref = g[f"logits_cfg{cfg_scale}"].transpose(0, 1)
    assert logits.shape == ref.shape
    assert (logits - ref).abs().max().item() <= 1e-4
    want = torch.nn.functional.cross_entropy(ref.reshape(-1, ref.shape[-1]), toks.reshape(-1).long(), reduction="none")
    assert torch.allclose(nll.reshape(-1), want, atol=1e-4)


def _dataset_mask(emb_mask, max_seq):
    """dataset/t2i.py:123-128 for one image, as train_t2i.py:158,164 feeds it: [1, 1, max_seq - 1, max_seq - 1] bool."""
    T = emb_mask.shape[0]
    attn = torch.tril(torch.ones(max_seq, max_seq))
    attn[:, :T] = attn[:, :T] * emb_mask.unsqueeze(0)
    eye = torch.eye(max_seq, max_seq)
    attn = (attn * (1 - eye) + eye).unsqueeze(0).to(torch.bool)
    return attn.unsqueeze(1)[:, :, :-1, :-1]


def test_attn_mask_to_emb_masks():
    from llamagen_b200.gpt import emb_mask_from_attn_mask
    T, L = 8, 8 + 16
    ems = torch.stack([(torch.arange(T) >= p).float() for p in (3, 0, T)])      # ragged, all one, all zero
    mask = torch.cat([_dataset_mask(e, L) for e in ems])
    assert torch.equal(emb_mask_from_attn_mask(mask, T), ems)
    assert torch.equal(emb_mask_from_attn_mask(mask[:, 0].float(), T), ems)       # [B, seq, seq], float
    one = torch.cat([_dataset_mask(e, T + 1) for e in ems])                        # seq == T (a single scored token)
    assert torch.equal(emb_mask_from_attn_mask(one, T)[:, : T - 1], ems[:, : T - 1])
    bad = mask.clone()
    bad[0, 0, T + 3, T + 5] = True                                                 # a future key
    bad2 = mask.clone()
    bad2[1, 0, T + 2, 2] = False                                                   # a condition key hidden from one row only
    bad3 = mask.clone()
    bad3[2, 0, 5, 5] = False                                                       # the diagonal
    for b in (bad, bad2, bad3, mask.repeat(1, 2, 1, 1), mask[:, :, :, :-1], mask[:, :, : T - 1, : T - 1]):
        with pytest.raises(ValueError):
            emb_mask_from_attn_mask(b, T)


def test_score_cli_reads_code_directory(tmp_path):
    from llamagen_b200.sample.score_c2i import code_files, load_item
    codes, labels = tmp_path / "imagenet256_codes", tmp_path / "imagenet256_labels"
    codes.mkdir()
    labels.mkdir()
    rng = np.random.default_rng(0)
    want = {}
    for i in (0, 1, 2, 10):
        x = rng.integers(0, 1024, size=(1, 2, 16), dtype=np.int64)
        np.save(codes / f"{i}.npy", x)
        np.save(labels / f"{i}.npy", np.array([i % 7]))
        want[i] = x
    (codes / "notes.txt").write_text("ignored")
    files = code_files(str(tmp_path))
    assert [int(c.rsplit("/", 1)[1][:-4]) for c, _ in files] == [0, 1, 2, 10]
    for (c, l), i in zip(files, (0, 1, 2, 10)):
        t, y = load_item(c, l, 1)
        assert torch.equal(t, torch.from_numpy(want[i][0, 1])) and y == i % 7
    with pytest.raises(SystemExit):
        load_item(*files[0], 2)
    np.save(codes / "11.npy", want[0])
    with pytest.raises(SystemExit):
        code_files(str(tmp_path))
    with pytest.raises(SystemExit):
        code_files(str(codes))
