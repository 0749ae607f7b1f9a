"""Speculative Jacobi decoding without a GPU: the rule (tests/sjd_oracle.py) is lossless and greedy-exact on a toy Markov model,
the scratch sizes of lg_sjd_workspace_bytes are pinned, and generate() rejects bad arguments before it touches a device."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import sjd_oracle as so


def _toy(V, seed, sharp):
    rng = np.random.default_rng(seed)
    logits = rng.standard_normal((V + 1, V)) * sharp
    p = np.exp(logits - logits.max(1, keepdims=True))
    p = (p / p.sum(1, keepdims=True)).astype(np.float32)
    return p[0], p[1:]


def _exact(p0, table, S):
    """The autoregressive distribution of every full sequence."""
    V = table.shape[0]
    out = {}
    for seq in itertools.product(range(V), repeat=S):
        pr = float(p0[seq[0]])
        for a, b in zip(seq, seq[1:]):
            pr *= float(table[a, b])
        out[seq] = pr
    return out


@pytest.mark.parametrize("L", [2, 3, 4, 5, 6, 7])
def test_greedy_sjd_equals_greedy_ar(L):
    S = 8
    for seed in range(20):
        p0, table = _toy(16, seed, 1.0)
        want = [int(np.argmax(p0))]
        for _ in range(S - 1):
            want.append(int(np.argmax(table[want[-1]])))
        got, passes = so.toy_run(p0, table, S, L, seed, greedy=True)
        assert got == want and 1 <= passes <= S - 1


@pytest.mark.parametrize("L", [2, 3])
def test_sjd_is_lossless_in_distribution(L):
    """10^5 seeded runs of V = 16, S = 4. Under the exact law the expected total variation of the empirical histogram is about
    sum_x sqrt(p_x (1 - p_x) / (2 pi N)) (E_tv below); the bound 1.3 E_tv + 0.004 sits far inside the distance a lossy rule
    reaches (accepting every draft: asserted too)."""
    V, S, N = 16, 4, 100_000
    p0, table = _toy(V, 7, 2.0)
    exact = _exact(p0, table, S)
    counts, multi = {}, 0
    for seed in range(N):
        seq, passes = so.toy_run(p0, table, S, L, seed, greedy=False)
        counts[tuple(seq)] = counts.get(tuple(seq), 0) + 1
        multi += passes < S - 1
    tv = 0.5 * sum(abs(counts.get(x, 0) / N - p) for x, p in exact.items())
    e_tv = sum(np.sqrt(p * (1 - p) / (2 * np.pi * N)) for p in exact.values())
    assert tv < 1.3 * e_tv + 0.004, (tv, e_tv)
    assert multi > N // 100     # drafts were accepted in a real share of the runs

    # the same check sees a lossy rule: drafts accepted unconditionally
    uniform = so.uniform
    try:
        so.uniform = lambda seed, b, k, purpose: np.float32(0.0) if purpose == so.ACCEPT else uniform(seed, b, k, purpose)
        lossy = {}
        for seed in range(N // 10):
            seq, _ = so.toy_run(p0, table, S, L, seed, greedy=False)
            lossy[tuple(seq)] = lossy.get(tuple(seq), 0) + 1
    finally:
        so.uniform = uniform
    tv_lossy = 0.5 * sum(abs(lossy.get(x, 0) / (N // 10) - p) for x, p in exact.items())
    assert tv_lossy > 3 * (1.3 * e_tv + 0.004), tv_lossy


def test_uniform_keys_are_distinct():
    us = {float(so.uniform(5, b, k, pr)) for b in range(4) for k in range(16) for pr in (so.ACCEPT, so.RESIDUAL, so.INIT)}
    assert len(us) == 4 * 16 * 3
    assert so.pass_seed(5, 0, 0) != so.pass_seed(5, 0, 1) != so.pass_seed(5, 1, 1)


_GPT_L = dict(n_layer=24, n_head=16, dim=1024, ffn_dim=2816, vocab_size=16384, cls_token_num=1, num_classes=1000, caption_dim=0,
              block_size=256)
_GPT_XL_T2I = dict(n_layer=36, n_head=20, dim=1280, ffn_dim=3584, vocab_size=16384, cls_token_num=120, num_classes=0, caption_dim=2048,
                   block_size=1024)


@pytest.mark.parametrize("m, t2i, sizes", [
    (_GPT_L, False, {(1, 1, 4): 1686016, (8, 1, 16): 53874944, (64, 1, 32): 861980160, (64, 0, 8): 141309184}),
    (_GPT_XL_T2I, True, {(1, 1, 16): 6851072, (4, 0, 2): 2238976}),
], ids=["c2i_gpt_l", "t2i_gpt_xl"])
def test_sjd_workspace_bytes_are_pinned(m, t2i, sizes, monkeypatch):
    """(B, use_cfg, L) -> bytes of lg_generate_sjd's scratch for bf16 models; host arithmetic, no GPU."""
    from llamagen_b200 import _lib
    monkeypatch.delenv("LG_GEMM_TC", raising=False)
    lib = _lib.load()
    cfg = _lib.ModelCfg(m["n_layer"], m["n_head"], m["dim"], m["ffn_dim"], m["vocab_size"], m["cls_token_num"], m["block_size"],
                        m["num_classes"], m["caption_dim"], _lib.LG_MODEL_T2I if t2i else _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    try:
        got = {}
        for B, c, L in sizes:
            n = ctypes.c_size_t()
            assert lib.lg_sjd_workspace_bytes(h, B, c, L, ctypes.byref(n)) == 0, lib.lg_last_error()
            got[(B, c, L)] = n.value
        assert got == sizes
        n = ctypes.c_size_t()
        for B, L in ((1, 1), (1, 65), (0, 4)):
            assert lib.lg_sjd_workspace_bytes(h, B, 1, L, ctypes.byref(n)) < 0
            assert b"lg_sjd_workspace_bytes" in lib.lg_last_error()
    finally:
        lib.lg_engine_destroy(h)


@pytest.mark.parametrize("kwargs, match", [
    (dict(sjd_window=1), "sjd_window must be an integer in"),
    (dict(sjd_window=65), "sjd_window must be an integer in"),
    (dict(sjd_window=2.5), "sjd_window must be an integer in"),
    (dict(sjd_window=True), "sjd_window must be an integer in"),
    (dict(sjd_window=4, teacher=torch.zeros(1, 4, dtype=torch.int32)), "cannot be combined"),
    (dict(sjd_window=4, return_logits=True), "cannot be combined"),
    (dict(return_stats=True), "return_stats needs sjd_window"),
])
def test_generate_sjd_argument_errors(kwargs, match):
    from llamagen_b200 import GPT_models, generate
    model = GPT_models["GPT-B"](block_size=16, vocab_size=64)
    with pytest.raises(ValueError, match=match):
        generate(model, torch.tensor([1]), 4, **kwargs)


def test_sampler_cli_flag():
    from llamagen_b200.sample import sample_c2i, sample_t2i
    from llamagen_b200.sample.common import sjd_kwargs
    a = sample_c2i.build_parser().parse_args(["--sjd-window", "8"])
    assert a.sjd_window == 8 and sjd_kwargs(a) == {"sjd_window": 8}
    b = sample_t2i.build_parser().parse_args([])
    assert b.sjd_window is None and sjd_kwargs(b) == {}
