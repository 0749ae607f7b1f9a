"""GPU: the order between the kernels of eager decode steps, on every 16-bit path.

Every kernel of a decode step is launched with programmatic dependent launch (PDL), and the fused decode attention reads the
position counter before its dependency wait (DESIGN §4, "Reads before the dependency wait"). An eager step therefore launches its
first kernel without PDL; in graph replay the graph launch orders the step. Each case runs each configuration once and compares
bit for bit against two references with the same arithmetic:

* graph replay: the default run;
* PDL off: the same call after lib.lg_set_pdl(0), where every kernel starts after its predecessor has completed.

Compared are the tokens and log-probabilities of a top-k sampled run and the logits of a teacher-forced greedy run (without a
teacher on the negative-prompt path, which does not take one). Models are registry GPT-B models with V = 16384, whose sample kernel
runs long enough for a step's first kernels to start beside it.

* Eager (LG_NO_GRAPH=1, fused tail on) against graph replay against PDL off, over bf16 / fp16, c2i / t2i (ragged emb-masks, one
  negative prompt), the batched (R > 8) and small-row (R <= 8) decode paths, 16-bit and fp8 KV caches, 16-bit and fp8 weights and
  one and two decode chains, paired rather than as the full product.
* Short runs in the default mode, where every decode step is eager (fewer than 3 steps after the first): generate(S) and
  generate(S, prefix=) with S - P - 1 in {1, 2, 3} equal the first S tokens of a long graph-mode run of the same call (the draw is
  keyed by seed, image and token index); inpainting holes of 1 and 2 tokens and an extend followed by one or two draws equal the
  PDL-off run.
* serve.LLM, a mixed bf16 stream with a prefix and an inpainting request: its steps are eager with positions written by torch, and
  PDL on equals PDL off."""
import contextlib
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

V = 16384
TOPK = 100
T2I = dict(model_type="t2i", cls_token_num=120, caption_dim=2048)


def _model(dtype, kv="auto", weights="auto", **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(7)
    m = GPT_models["GPT-B"](block_size=256, vocab_size=V, **kw)
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dtype).eval()
    m.set_kv_cache(kv)
    m.set_weight_dtype(weights)
    return m


@contextlib.contextmanager
def _pdl_off():
    """PDL off for the calls inside; afterwards the state LG_PDL selects (on unless LG_PDL=0), which every other caller runs with."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    prev = 0 if os.environ.get("LG_PDL", "1").strip() == "0" else 1
    _lib.check(lib.lg_set_pdl(0), "lg_set_pdl")
    try:
        yield
    finally:
        _lib.check(lib.lg_set_pdl(prev), "lg_set_pdl")


def _gen(m, cond, S, **kw):
    from llamagen_b200 import generate
    out = generate(m, cond.cuda(), S, **kw)
    torch.cuda.synchronize()
    return tuple(o.cpu() for o in out) if isinstance(out, tuple) else out.cpu()


def _chains(m, cond, S, em, B):
    """Decode chains of this model, batch and workspace: a prefix call decides its chain count as lg_generate does (engine.cu,
    generate_impl's `split`) and reports it through lg_test_prefix_chunks."""
    from llamagen_b200 import _lib
    pf = torch.zeros(B, 1, dtype=torch.long)
    _gen(m, cond, S, emb_masks=em, cfg_scale=4.0, prefix=pf, seed=0)
    n = ctypes.c_int(0)
    _lib.load().lg_test_prefix_chunks(m.engine(), ctypes.byref(n))
    return n.value


def _ragged(B, T, seed):
    """emb-masks as the t2i pipeline makes them: the caption's n tokens at the end of the T slots, n different per image"""
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(1, T + 1, (B,), generator=g)
    n[0] = T
    return (torch.arange(T)[None] >= (T - n)[:, None]).float()


def _runs(m, cond, S, em, neg, teacher):
    """(greedy tokens, logits, sampled tokens, logprobs) of one configuration"""
    kw = dict(emb_masks=em, cfg_scale=4.0)
    if neg is not None:
        kw["negative_cond"] = neg
    forced = _gen(m, cond, S, sample_logits=False, return_logits=True, teacher=teacher, **kw) if neg is None else \
        _gen(m, cond, S, sample_logits=False, return_logits=True, **kw)
    toks, lp = _gen(m, cond, S, top_k=TOPK, seed=5, return_logprobs=True, **kw)
    return forced[0], forced[1], toks, lp


def _first_diff(a, b):
    if a.shape != b.shape:
        return f"shapes {tuple(a.shape)} / {tuple(b.shape)}"
    bad = (a != b).nonzero()
    if bad.numel() == 0:
        return "equal"
    d = (a.double() - b.double()).abs().max().item() if a.is_floating_point() else None
    return f"first difference at {tuple(bad[0].tolist())}, max |diff| {d}"


def _assert_same(got, want, what):
    for name, a, b in zip(("greedy tokens", "logits", "sampled tokens", "logprobs"), got, want):
        assert torch.equal(a, b), f"{what}: {name}: {_first_diff(a, b)}"


# (id, dtype, model kwargs, B, kv, weights, LG_SPLIT, chains, negative prompt)
# Chains: the workspace of R = 2B rows splits in two when R / 2 is even and >= 16 and a GPT-B layer (14.2 MB in 16 bits) is at most
# a third of the L2, and a call takes the split when LG_SPLIT is unset or >= 2, R is the workspace's rows and B is a multiple of the
# chain count (engine.cu, lg_engine_set_workspace and generate_impl's `split`); B = 16 splits, B = 24 under LG_SPLIT=1 and B = 9
# (R / 2 odd) do not. R <= 8 takes the small-row path, whose workspace never splits.
CASES = [
    ("c2i-bf16-batched-1chain", torch.bfloat16, {}, 24, "auto", "auto", "1", 1, False),
    ("c2i-fp16-batched-2chains-kvfp8", torch.float16, {}, 16, "fp8", "auto", None, 2, False),
    ("c2i-bf16-small-w8", torch.bfloat16, {}, 2, "auto", "fp8", None, 1, False),
    ("c2i-fp16-small-kvfp8-w8", torch.float16, {}, 3, "fp8", "fp8", None, 1, False),
    ("t2i-bf16-batched-2chains-w8-negative", torch.bfloat16, T2I, 16, "auto", "fp8", None, 2, True),
    ("t2i-fp16-batched-1chain-kvfp8", torch.float16, T2I, 9, "fp8", "auto", None, 1, False),
    ("t2i-bf16-small", torch.bfloat16, T2I, 4, "auto", "auto", None, 1, False),
]


@pytest.mark.parametrize("dtype,kw,B,kv,weights,split,chains,negative", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_eager_equals_graph_equals_pdl_off(dtype, kw, B, kv, weights, split, chains, negative, monkeypatch):
    S = 10
    monkeypatch.delenv("LG_NO_GRAPH", raising=False)
    monkeypatch.delenv("LG_FUSE_TAIL", raising=False)
    if split is None:
        monkeypatch.delenv("LG_SPLIT", raising=False)
    else:
        monkeypatch.setenv("LG_SPLIT", split)
    m = _model(dtype, kv, weights, **kw)
    g = torch.Generator().manual_seed(B)
    if m.model_type == "c2i":
        cond, em, neg = torch.randint(0, 1000, (B,), generator=g), None, None
    else:
        T, C = m.config.cls_token_num, m.config.caption_dim
        cond = torch.randn(B, T, C, generator=g).to(dtype)
        em = _ragged(B, T, B)
        neg = torch.randn(1, T, C, generator=g).to(dtype) if negative else None
    if chains == 1 and split is None:
        assert 2 * B <= 8 or B % 2 == 1, "the configuration must keep one chain"
    if 2 * B <= 8:
        assert chains == 1                                    # small-row path
    teacher = torch.randint(0, V, (B, S), generator=g, dtype=torch.int32)
    graph = _runs(m, cond, S, em, neg, teacher)
    assert _chains(m, cond, S, em, B) == chains
    with _pdl_off():
        off = _runs(m, cond, S, em, neg, teacher)
    _assert_same(graph, off, "graph replay vs PDL off")
    monkeypatch.setenv("LG_NO_GRAPH", "1")
    m._drop_engine()                                          # LG_NO_GRAPH is read when the engine is created
    eager = _runs(m, cond, S, em, neg, teacher)
    assert _chains(m, cond, S, em, B) == chains
    _assert_same(eager, graph, "eager vs graph replay")


SHORT = [("bf16-batched", torch.bfloat16, 24), ("fp16-small", torch.float16, 2)]


@pytest.mark.parametrize("dtype,B", [c[1:] for c in SHORT], ids=[c[0] for c in SHORT])
def test_short_runs_equal_long_graph_run(dtype, B, monkeypatch):
    """S - P - 1 in {1, 2, 3}: every decode step is eager; the first S tokens of a long graph-mode run of the same call."""
    for k in ("LG_NO_GRAPH", "LG_FUSE_TAIL", "LG_SPLIT"):
        monkeypatch.delenv(k, raising=False)
    m = _model(dtype)
    g = torch.Generator().manual_seed(11)
    cond = torch.randint(0, 1000, (B,), generator=g)
    L = 16                                                    # 14 decode steps after the first: graph replay
    teacher = torch.randint(0, V, (B, L), generator=g, dtype=torch.int32)
    kw = dict(cfg_scale=4.0, top_k=TOPK, seed=5)
    long_toks, long_lp = _gen(m, cond, L, return_logprobs=True, **kw)
    _, long_logits = _gen(m, cond, L, cfg_scale=4.0, sample_logits=False, return_logits=True, teacher=teacher)
    for S in (2, 3, 4):
        toks, lp = _gen(m, cond, S, return_logprobs=True, **kw)
        assert torch.equal(toks, long_toks[:, :S]), (S, _first_diff(toks, long_toks[:, :S]))
        assert torch.equal(lp, long_lp[:, :S]), (S, _first_diff(lp, long_lp[:, :S]))
        _, logits = _gen(m, cond, S, cfg_scale=4.0, sample_logits=False, return_logits=True, teacher=teacher[:, :S].contiguous())
        assert torch.equal(logits, long_logits[:S]), (S, _first_diff(logits, long_logits[:S]))
    P = 8
    pf = torch.randint(0, V, (B, P), generator=g)
    long_toks, long_lp = _gen(m, cond, L, prefix=pf, return_logprobs=True, **kw)
    for S in (P + 2, P + 3, P + 4):                           # P = S - 2, S - 3, S - 4
        toks, lp = _gen(m, cond, S, prefix=pf, return_logprobs=True, **kw)
        assert torch.equal(toks, long_toks[:, :S]), (S, _first_diff(toks, long_toks[:, :S]))
        assert torch.equal(lp, long_lp[:, :S]), (S, _first_diff(lp, long_lp[:, :S]))


def _mask(S, runs):
    mk = torch.zeros(S, dtype=torch.bool)
    for a, b in runs:
        mk[a:b] = True
    return mk


@pytest.mark.parametrize("dtype,B", [c[1:] for c in SHORT], ids=[c[0] for c in SHORT])
def test_inpainting_short_holes_equal_pdl_off(dtype, B, monkeypatch):
    """Holes whose decode steps are all eager, and decode steps right after an extend pass (whose set_counters kernel writes the
    position counter), against the same calls with PDL off."""
    for k in ("LG_NO_GRAPH", "LG_FUSE_TAIL", "LG_SPLIT"):
        monkeypatch.delenv(k, raising=False)
    S = 12
    m = _model(dtype)
    g = torch.Generator().manual_seed(13)
    cond = torch.randint(0, 1000, (B,), generator=g)
    given = torch.randint(0, V, (B, S), generator=g)
    masks = {
        "interior hole of 1": _mask(S, [(0, 6), (7, S)]),
        "hole of 2 at the end": _mask(S, [(0, S - 2)]),
        "extend, then 3 draws": _mask(S, [(0, 3), (5, 9)]),
        "extend, then 2 draws": _mask(S, [(0, 3), (5, 10)]),
    }
    for what, mk in masks.items():
        kw = dict(cfg_scale=4.0, top_k=TOPK, seed=5, given=given, given_mask=mk)
        on = _gen(m, cond, S, **kw)
        with _pdl_off():
            off = _gen(m, cond, S, **kw)
        assert torch.equal(on[:, mk], given[:, mk].to(on.dtype)), what
        assert torch.equal(on, off), (what, _first_diff(on, off))


def test_serve_mixed_stream_pdl_on_equals_off():
    """A running bf16 batch with a plain, a prefix and an inpainting request: serving's decode steps are eager and their per-row
    positions come from torch, so PDL on and off give the same tokens (inpainting requests take no logprobs)."""
    from llamagen_b200.serve import LLM, SamplingParams
    S = 16
    m = _model(torch.bfloat16)
    g = torch.Generator().manual_seed(17)
    pf = torch.randint(0, V, (5,), generator=g)
    given = torch.randint(0, V, (S,), generator=g)
    mk = _mask(S, [(0, 4), (6, 12)])
    reqs = [([207], {}), ([360], {"prefix": pf}), ([387], {"given": given, "given_mask": mk}), ([974], {})]
    sp = SamplingParams(temperature=1.0, top_p=1.0, top_k=TOPK, max_tokens=S)

    def run():
        llm = LLM(m, cfg_scale=4.0, num_classes=1000, max_num_seqs=4, seed=11)
        outs = []
        for i, (c, kw) in enumerate(reqs):
            llm.add_request(c, sp, **kw)
            if i == 1:
                outs += llm.step()                            # the later requests join a running batch
        while llm.has_unfinished_requests():
            outs += llm.step()
        torch.cuda.synchronize()
        return {int(o.request_id): list(o.outputs[0].token_ids) for o in outs}

    on = run()
    with _pdl_off():
        off = run()
    assert sorted(on) == list(range(len(reqs)))
    assert torch.equal(torch.tensor(on[1][:5]), pf)
    assert torch.equal(torch.tensor(on[2])[mk], given[mk])
    assert on == off
