"""CPU: inpainting (generate(..., given=tokens, given_mask=mask)) without a GPU.

* The given oracle is pinned in fp64 on the tiny golden models: an all-False mask is GPTOracle.generate, a mask of the first P
  columns is the prefix oracle, and any mask takes the given tokens and, elsewhere, the teacher-forced oracle's logits.
* lg_test_given_plan: the segments of the plan for all-False, leading-only, trailing-only, box-hole, runs of 1, runs > 64 and
  per-image masks.
* Every ValueError of generate(given=...), the C entry's argument checks, and the samplers' --inpaint-image / --inpaint-box."""
import ctypes

import pytest
import torch

from given_oracle import given_oracle
from oracle import GPTOracle
from prefix_oracle import prefix_oracle
from util import load_golden

LEAD, DECODE, EXTEND, TAIL = 0, 1, 2, 3


def _sd64(g):
    sd = {k: v.double() if v.is_floating_point() else v for k, v in g["state_dict"].items()}
    cond = g["cond"].double() if g["cond"].is_floating_point() else g["cond"]
    return sd, cond


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale, cfg_interval", [(1.0, -1), (4.0, -1), (4.0, 3)])
def test_given_oracle_is_pinned(name, cfg_scale, cfg_interval):
    g = load_golden(name)
    sd, cond = _sd64(g)
    toks = g[f"tokens_cfg{cfg_scale}"]
    B, S = toks.shape
    kw = dict(emb_masks=g["emb_masks"], cfg_scale=cfg_scale, cfg_interval=cfg_interval, sample_logits=False)
    plain, _ = GPTOracle(sd, g["cfg"]).generate(cond, S, **kw)
    none = torch.zeros(B, S, dtype=torch.bool)
    out, _ = given_oracle(GPTOracle(sd, g["cfg"]), cond, toks, none, S, **kw)
    assert torch.equal(out, plain.to(torch.int32))
    for P in (1, S // 2, S - 1):
        lead = none.clone()
        lead[:, :P] = True
        out, logits = given_oracle(GPTOracle(sd, g["cfg"]), cond, toks, lead, S, **kw)
        want, wl = prefix_oracle(GPTOracle(sd, g["cfg"]), cond, toks[:, :P], S, **kw)
        assert torch.equal(out, want) and (logits - wl).abs().max().item() <= 1e-9, P
    # a hole and per-image masks: given tokens kept, the rest drawn from the teacher-forced oracle's logits of the final sequence
    mask = torch.rand(B, S, generator=torch.Generator().manual_seed(3)) < 0.5
    mask[:, 5:9] = True
    mask[0, 0] = False
    gv = (toks + 7) % g["cfg"]["vocab_size"]
    out, logits = given_oracle(GPTOracle(sd, g["cfg"]), cond, gv, mask, S, **kw)
    assert torch.equal(out[mask], gv[mask].to(torch.int32))
    _, ref = GPTOracle(sd, g["cfg"]).generate(cond, S, teacher=out.long(), **kw)
    assert (logits - ref).abs().max().item() <= 1e-9
    assert torch.equal(out[~mask], ref.argmax(-1).T[~mask].to(torch.int32))


# ------------------------------------------------------------------------------------------------------------------- plan
def _plan(given):
    from llamagen_b200 import _lib
    lib = _lib.load()
    g = torch.as_tensor(given, dtype=torch.int32).contiguous()
    B, S = g.shape
    buf = (ctypes.c_int32 * (3 * S + 3))()
    n = lib.lg_test_given_plan(_lib.ptr(g), B, S, buf, S + 1)
    assert n > 0, lib.lg_last_error().decode()
    return [tuple(buf[3 * i:3 * i + 3]) for i in range(n)]


def _given(mask, B=None):
    m = torch.as_tensor(mask, dtype=torch.bool)
    m = m.view(1, -1).expand(B or 1, -1) if m.dim() == 1 else m
    return torch.where(m, torch.full(m.shape, 5), torch.full(m.shape, -1))


def _box(grid, top, left, bottom, right):
    m = torch.ones(grid, grid, dtype=torch.bool)
    m[top:bottom, left:right] = False
    return m.reshape(-1)


def _covers(plan, S):
    """Every token is in exactly one segment's range; LEAD and EXTEND also draw the token after their range."""
    seen = []
    for kind, start, n in plan:
        seen += range(start, start + n)
        if kind in (LEAD, EXTEND):
            seen.append(start + n)
    assert seen == list(range(S)), plan


def test_plan_all_false_leading_trailing():
    S = 256
    assert _plan(_given(torch.zeros(S))) == [(LEAD, 0, 0), (DECODE, 1, S - 1)]
    lead = torch.zeros(S)
    lead[:100] = 1
    assert _plan(_given(lead)) == [(LEAD, 0, 100), (DECODE, 101, S - 101)]
    lead[:S - 1] = 1
    assert _plan(_given(lead)) == [(LEAD, 0, S - 1)]
    tail = torch.zeros(S)
    tail[200:] = 1
    assert _plan(_given(tail)) == [(LEAD, 0, 0), (DECODE, 1, 199), (TAIL, 200, 56)]
    for m in (lead, tail):
        _covers(_plan(_given(m)), S)


def test_plan_box_hole():
    """The issue's 8 x 8 hole in a 16 x 16 grid: one prefill, 7 window passes of 8 given tokens, 56 decode steps, one copied tail."""
    plan = _plan(_given(_box(16, 4, 4, 12, 12)))
    assert plan[0] == (LEAD, 0, 4 * 16 + 4)
    ext = [p for p in plan if p[0] == EXTEND]
    dec = [p for p in plan if p[0] == DECODE]
    assert len(ext) == 7 and all(n == 8 for _, _, n in ext)
    assert len(dec) == 8 and sum(n for _, _, n in dec) == 56
    assert plan[-1] == (TAIL, 12 * 16 - 4, 4 * 16 + 4)
    _covers(plan, 256)


def test_plan_runs_of_one_and_long_runs():
    S = 200
    alt = torch.arange(S) % 2 == 1                        # every odd token given: runs of 1
    plan = _plan(_given(alt))
    assert plan[0] == (LEAD, 0, 0) and plan[-1] == (TAIL, S - 1, 1)
    assert [p for p in plan[1:-1]] == [(EXTEND, k, 1) for k in range(1, S - 1, 2)]
    _covers(plan, S)
    long = torch.zeros(S, dtype=torch.bool)
    long[10:150] = True                                   # one run of 140 > 64: one EXTEND (run in chunks of 64 rows)
    assert _plan(_given(long)) == [(LEAD, 0, 0), (DECODE, 1, 9), (EXTEND, 10, 140), (DECODE, 151, 49)]


def test_plan_per_image_masks():
    """A position drawn by any image is a DECODE step; only runs given to every image become LEAD, EXTEND or TAIL."""
    S = 32
    m = torch.zeros(3, S, dtype=torch.bool)
    m[:, :4] = True
    m[0, 4:6] = True                                      # image 0 also gives 4, 5: still decoded for the others
    m[:, 10:20] = True
    m[1, 20] = True
    m[:, 28:] = True
    assert _plan(_given(m)) == [(LEAD, 0, 4), (DECODE, 5, 5), (EXTEND, 10, 10), (DECODE, 21, 7), (TAIL, 28, 4)]


def test_plan_rejections():
    from llamagen_b200 import _lib
    lib = _lib.load()
    buf = (ctypes.c_int32 * 30)()
    g = torch.full((2, 8), 3, dtype=torch.int32)
    assert lib.lg_test_given_plan(_lib.ptr(g), 2, 8, buf, 10) < 0 and "every token is given" in lib.lg_last_error().decode()
    g[1, 3] = -2
    assert lib.lg_test_given_plan(_lib.ptr(g), 2, 8, buf, 10) < 0 and "-1 for a drawn token" in lib.lg_last_error().decode()
    assert lib.lg_test_given_plan(None, 2, 8, buf, 10) < 0


# ------------------------------------------------------------------------------------------------------------- rejections
class _Model:
    """What generate() reads before it needs a device."""

    def __init__(self):
        from llamagen_b200.gpt import ModelArgs, Transformer
        self.m = Transformer(ModelArgs(n_layer=1, n_head=2, dim=128, vocab_size=512, block_size=16, num_classes=10))


_G = torch.zeros(2, 16, dtype=torch.int64)
_M = torch.arange(16) < 4


@pytest.mark.parametrize("kw, msg", [
    (dict(given=_G), "go together"),
    (dict(given_mask=_M), "go together"),
    (dict(given=torch.zeros(3, 16, dtype=torch.int64), given_mask=_M), "[B, S] or [1, S]"),
    (dict(given=torch.zeros(2, 15, dtype=torch.int64), given_mask=_M), "[B, S] or [1, S]"),
    (dict(given=torch.zeros(16, dtype=torch.int64), given_mask=_M), "[B, S] or [1, S]"),
    (dict(given=_G, given_mask=torch.ones(3, 16, dtype=torch.bool)), "given_mask must be"),
    (dict(given=_G, given_mask=torch.ones(15, dtype=torch.bool)), "given_mask must be"),
    (dict(given=_G, given_mask=_M.long()), "bool"),
    (dict(given=_G.float(), given_mask=_M), "integer"),
    (dict(given=_G, given_mask=torch.ones(16, dtype=torch.bool)), "at least one token"),
    (dict(given=torch.full((2, 16), 512), given_mask=_M), "vocab_size"),
    (dict(given=torch.full((2, 16), -1), given_mask=_M), "vocab_size"),
    (dict(given=_G, given_mask=_M, prefix=torch.zeros(2, 4, dtype=torch.int64)), "prefix"),
    (dict(given=_G, given_mask=_M, teacher=torch.zeros(2, 16, dtype=torch.int64)), "teacher"),
    (dict(given=_G, given_mask=_M, sjd_window=4), "sjd_window"),
    (dict(given=_G, given_mask=_M, return_logits=True), "return_logits"),
    (dict(given=_G, given_mask=_M, return_logprobs=True), "return_logprobs"),
], ids=["mask_missing", "given_missing", "batch", "length", "1d", "mask_batch", "mask_length", "mask_dtype", "float", "all_true",
        "too_large", "negative", "prefix", "teacher", "sjd", "logits", "logprobs"])
def test_generate_given_rejections(kw, msg):
    from llamagen_b200 import generate
    m = _Model().m
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        generate(m, torch.tensor([1, 2]), 16, **kw)


def test_out_of_range_ids_outside_the_mask_are_not_read():
    from llamagen_b200.generate import _check_given
    g = torch.full((2, 16), 9999)
    g[:, :4] = 7
    out = _check_given(g, (torch.arange(16) < 4).view(1, -1), 2, 16, 512)
    assert out.dtype == torch.int32 and out.shape == (2, 16)
    assert (out[:, :4] == 7).all() and (out[:, 4:] == -1).all()


def test_lg_generate_given_argument_errors_without_gpu():
    """The checks that need no workspace, on an engine bound to aligned placeholder addresses (never dereferenced)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    D, V, F = 128, 512, 384
    cfg = _lib.ModelCfg(1, 2, D, F, V, 1, 16, 10, 0, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    P_ = ctypes.c_void_p
    given = torch.full((2, 16), -1, dtype=torch.int32)
    given[:, :4] = 3
    try:
        sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 1, 0)

        def call(**kw):
            a = dict(cond=P_(1 << 20), em=None, neg=None, nm=None, B=2, T=1, S=16, given=given, ws=P_(4 << 20), ws_bytes=1 << 40,
                     out=P_(5 << 20))
            a.update(kw)
            g = a["given"]
            rc = lib.lg_generate_given(h, a["cond"], a["em"], a["neg"], a["nm"], a["B"], a["T"], a["S"], ctypes.byref(sc),
                                       None if g is None else _lib.ptr(g), a["ws"], a["ws_bytes"], a["out"], None)
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
        full = torch.full((2, 16), 3, dtype=torch.int32)
        big = given.clone()
        big[1, 2] = V
        low = given.clone()
        low[0, 9] = -2
        for kw, msg in [(dict(given=None), "null given"), (dict(T=2), "cls_token_num"), (dict(em=P_(7 << 20)), "emb_mask"),
                        (dict(cond=None), "null cond"), (dict(out=None), "null cond"), (dict(S=17), "block_size"),
                        (dict(B=0), "B=0"), (dict(given=full), "every token is given"), (dict(given=big), "vocab_size"),
                        (dict(given=low), "-1 for a drawn token"), (dict(neg=P_(8 << 20)), "t2i models only"),
                        ({}, "workspace not set")]:
            rc, err = call(**kw)
            assert rc < 0 and msg in err, (kw, rc, err)
        n1, n2, n3 = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        hole = torch.full((2, 16), 3, dtype=torch.int32)
        hole[:, 5] = -1
        hole[:, 12] = -1                                  # LEAD 5, EXTEND [6, 12), a TAIL
        assert lib.lg_given_workspace_bytes(h, _lib.ptr(given), 2, 16, 1, ctypes.byref(n1)) == 0
        assert lib.lg_given_workspace_bytes(h, _lib.ptr(hole), 2, 16, 1, ctypes.byref(n2)) == 0
        assert lib.lg_given_workspace_bytes(h, _lib.ptr(hole), 2, 16, 0, ctypes.byref(n3)) == 0
        assert 0 < n1.value < n2.value and n3.value < n2.value          # the window rows, and twice the rows under CFG
        assert lib.lg_given_workspace_bytes(h, _lib.ptr(full), 2, 16, 1, ctypes.byref(n1)) < 0
        assert lib.lg_given_workspace_bytes(h, None, 2, 16, 1, ctypes.byref(n1)) < 0
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("argv, msg", [
    (["--inpaint-box", "0", "0", "4", "4"], "go together"),
    (["--inpaint-image", "IMG"], "go together"),
    (["--inpaint-image", "IMG", "--inpaint-box", "2", "0", "2", "4"], "TOP < BOTTOM"),
    (["--inpaint-image", "IMG", "--inpaint-box", "0", "5", "4", "3"], "TOP < BOTTOM"),
    (["--inpaint-image", "IMG", "--inpaint-box", "-1", "0", "4", "4"], "TOP < BOTTOM"),
    (["--inpaint-image", "IMG", "--inpaint-box", "0", "0", "17", "4"], "TOP < BOTTOM"),
    (["--inpaint-image", "IMG", "--inpaint-box", "0", "0", "4", "4", "--prefix-image", "IMG", "--prefix-rows", "2"], "prefix-image"),
    (["--inpaint-image", "IMG", "--inpaint-box", "0", "0", "4", "4", "--sjd-window", "4"], "sjd-window"),
    (["--inpaint-image", "MISSING", "--inpaint-box", "0", "0", "4", "4"], "not a file"),
])
@pytest.mark.parametrize("cli", ["sample_c2i", "sample_t2i"])
def test_cli_inpaint_flag_rejections(cli, argv, msg, tmp_path):
    import importlib
    from llamagen_b200.sample.common import check_inpaint_args
    mod = importlib.import_module(f"llamagen_b200.sample.{cli}")
    img = tmp_path / "img.png"
    img.write_bytes(b"")
    argv = [str(img) if a == "IMG" else str(tmp_path / "none.png") if a == "MISSING" else a for a in argv]
    args = mod.build_parser().parse_args(["--image-size", "256"] + argv)
    with pytest.raises(SystemExit, match=msg):
        check_inpaint_args(args, 16)
    ok = mod.build_parser().parse_args(["--image-size", "256", "--inpaint-image", str(img), "--inpaint-box", "0", "0", "16", "16"])
    check_inpaint_args(ok, 16)
    check_inpaint_args(mod.build_parser().parse_args([]), 16)


def test_cli_inpaint_mask():
    from llamagen_b200.sample.common import inpaint_mask
    m = inpaint_mask((1, 1, 3, 4), 4).view(4, 4)
    assert (~m).sum() == 6 and not m[1:3, 1:4].any() and m[0].all() and m[3].all() and m[:, 0].all()


@pytest.mark.parametrize("cli", ["sample_c2i_ddp", "sample_t2i_ddp"])
def test_ddp_cli_inpaint_flags(cli, tmp_path):
    import importlib
    from llamagen_b200.sample.common import check_inpaint_args
    mod = importlib.import_module(f"llamagen_b200.sample.{cli}")
    img = tmp_path / "img.png"
    img.write_bytes(b"")
    ok = mod.build_parser().parse_args(["--image-size", "256", "--inpaint-image", str(img), "--inpaint-box", "4", "4", "12", "12"])
    check_inpaint_args(ok, 16)
    for argv, msg in ((["--inpaint-box", "4", "4", "12", "12"], "go together"),
                      (["--inpaint-image", str(img), "--inpaint-box", "4", "4", "12", "17"], "TOP < BOTTOM")):
        with pytest.raises(SystemExit, match=msg):
            check_inpaint_args(mod.build_parser().parse_args(["--image-size", "256"] + argv), 16)
    check_inpaint_args(mod.build_parser().parse_args([]), 16)
