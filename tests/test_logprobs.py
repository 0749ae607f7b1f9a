"""CPU: token log-probabilities in serve.LLM and generate() without a GPU: the SamplingParams(logprobs=, best_of=) range checks and their
refusals under sjd_window, generate()'s refusals, the top_n bounds of the C-ABI, the float64 oracle, and the host logic of serve.LLM with
the device stubbed (test_serve_n's _Device) and the library replaced by a recorder: best_of's selection and order, None for prefix
tokens, null-class twins mirroring logprobs, and draws that switch to lg_sample_rows_logprobs only while a slot asks."""
import ctypes
import math

import numpy as np
import pytest
import torch

import logprob_oracle as lo
from llamagen_b200 import serve
from test_serve_n import SP, _Device, _drive
from test_serve_guidance import _model


# ------------------------------------------------------------------------------------------------------------ argument checks
def test_sampling_params_ranges():
    for kind in ("c2i", "t2i"):
        llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=4)
        for bad in (dict(logprobs=-1), dict(logprobs=21), dict(logprobs=2.0), dict(logprobs=True), dict(best_of=0),
                    dict(n=3, best_of=2), dict(best_of=5), dict(best_of=1.5), dict(best_of=False)):
            with pytest.raises(ValueError, match="logprobs|best_of"):
                llm._guidance(SP(max_tokens=4, **bad))
        for ok in (dict(logprobs=0), dict(logprobs=20), dict(best_of=4), dict(n=2, best_of=2), dict(logprobs=np.int64(3), best_of=np.int32(3))):
            llm._guidance(SP(max_tokens=4, **ok))
    sjd = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=4, sjd_window=3)
    for kw in (dict(logprobs=0), dict(best_of=2)):
        with pytest.raises(ValueError, match="sjd_window"):
            sjd.add_request([1], SP(max_tokens=8, **kw))


def test_positional_fields_keep_their_meaning():
    sp = SP(0.0, 0.9, 50, 16, 2.0, 3, 7, 2, 5, 4)
    assert (sp.n, sp.logprobs, sp.best_of) == (2, 5, 4)
    c = serve.CompletionOutput(1, [3], "length", -1.5, [None])
    assert (c.cumulative_logprob, c.logprobs) == (-1.5, [None])


def test_generate_refusals():
    from llamagen_b200 import generate
    from llamagen_b200.gpt import ModelArgs, Transformer
    m = Transformer(ModelArgs(n_layer=1, n_head=2, dim=64, vocab_size=64, block_size=16, num_classes=10))
    cond = torch.tensor([1, 2])
    for kw, msg in [(dict(teacher=torch.zeros(2, 4, dtype=torch.int32)), "score"), (dict(sjd_window=2), "sjd_window"),
                    (dict(return_logits=True), "return_logits")]:
        with pytest.raises(ValueError, match=msg):
            generate(m, cond, 4, return_logprobs=True, **kw)
    for kw, msg in [(dict(top_logprobs=3), "needs return_logprobs"), (dict(return_logprobs=True, top_logprobs=0), r"\[1, 20\]"),
                    (dict(return_logprobs=True, top_logprobs=21), r"\[1, 20\]"), (dict(return_logprobs=True, top_logprobs=True), r"\[1, 20\]")]:
        with pytest.raises(ValueError, match=msg):
            generate(m, cond, 4, **kw)


def test_c_abi_top_n_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)
    sc = _lib.SampleCfg(1.0, -1, 1.0, 0, 1.0, 0, 0)
    for spec, msg in [(_lib.Logprobs(1 << 20, 0, 1 << 20, 1 << 20, 21), b"lg_sample_rows_logprobs: top_n=21 outside [0, 20]"),
                      (_lib.Logprobs(1 << 20, 0, 1 << 20, 0, 3), b"lg_sample_rows_logprobs: top_n=3 needs both"),
                      (_lib.Logprobs(1 << 20, 0, 0, 0, -1), b"top_n=-1 outside")]:
        assert lib.lg_sample_rows_logprobs(p, 1, 64, 0, 0, ctypes.byref(sc), p, p, None, None, None, ctypes.byref(spec), p, p, 1, None) < 0
        assert msg in lib.lg_last_error(), lib.lg_last_error()
    on = _lib.Logprobs(1 << 20, 0, 0, 0, 0)
    assert lib.lg_sample_rows_logprobs(p, 1, 64, 0, 0, ctypes.byref(sc), p, p, None, None, None, ctypes.byref(on), p, None, 1, None) < 0
    assert b"logprobs are indexed as out_seq" in lib.lg_last_error()
    bad = _lib.Logprobs(1 << 20, 0, 1 << 20, 1 << 20, 21)
    assert lib.lg_generate_logprobs(None, p, None, None, None, 1, 1, 8, ctypes.byref(sc), None, 0, None, 0, ctypes.byref(bad), p, None) < 0
    assert b"lg_generate_logprobs: top_n=21" in lib.lg_last_error()
    assert lib.lg_generate_logprobs(None, p, None, None, None, 1, 1, 8, ctypes.byref(sc), None, 0, None, 0, None, p, None) < 0
    assert b"lg_generate_logprobs: null engine" in lib.lg_last_error()


def test_oracle():
    x = np.array([1.0, 3.0, 3.0, -np.inf, 0.5, 2.0], np.float32)
    kept = np.array([True, True, True, False, False, True])
    lp = lo.logprobs(x, kept)
    assert math.isclose(np.exp(lp[kept]).sum(), 1.0) and np.isneginf(lp[~kept]).all()
    assert lo.rank(x, kept, 1) == 1 and lo.rank(x, kept, 5) == 3 and lo.rank(x, kept, 0) == 4
    ids, tl = lo.top(x, kept, 6)
    assert ids.tolist() == [1, 2, 5, 0, -1, -1] and np.isneginf(tl[4:]).all() and tl[0] == tl[1]


# ------------------------------------------------------------------------------------------------------------ serve host logic
class _Lib:
    """Stands in for the library: records every call by name; lg_sample_rows_logprobs also records its top_n."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*a):
            top = [x._obj.top_n for x in a if hasattr(x, "_obj") and isinstance(x._obj, serve._lib.Logprobs)]
            self.calls.append((name, top[0] if top else None))
            return 0
        return call


def _lp(rid, img, k):
    """The logprob the stub writes for token k of image img of request rid."""
    return -0.1 * ((7 * img + 3) % 5 + 1) - 0.001 * k - 0.01 * rid


def _stub(monkeypatch, llm):
    """test_serve_n's device stub, with every decode and join also running the real _draw against the recording library; after each
    device call the logprob rows of every running slot hold _lp and made-up ranks and alternatives."""
    lib = _Lib()
    monkeypatch.setattr(serve._lib, "load", lambda: lib)
    monkeypatch.setattr(serve._lib, "current_stream", lambda dev: None)
    dev = _Device(monkeypatch, llm)

    def fill(st):
        if "lp" not in st:
            return
        for b, req in enumerate(llm._slots):
            if req is not None:
                for k in range(st["S"]):
                    st["lp"][b, k] = _lp(int(req.request_id), llm._img[b], k)
                    st["rank"][b, k] = 2
                    st["top_ids"][b, k] = torch.arange(20) + 10000
                    st["top_lp"][b, k] = -torch.arange(20).float()

    def wrap(name, rows):
        inner = getattr(serve.LLM, name)

        def fn(self, st, params, *a):
            sl = rows(self, st, *a)
            self._draw(st, params, None, sl, st["pos"], st["out"])
            inner(self, st, params, *a)
            fill(st)
        monkeypatch.setattr(serve.LLM, name, fn)
    wrap("_device_step", lambda llm_, st: slice(0, llm_.max_num_seqs))
    wrap("_device_decode_t2i", lambda llm_, st: slice(0, llm_.max_num_seqs))
    wrap("_device_join_prefix", lambda llm_, st, slot, P: slice(slot, slot + 1))
    wrap("_device_join_t2i", lambda llm_, st, slot: slice(slot, slot + 1))
    return lib, dev


def test_no_switch_while_no_request_asks(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=4, seed=0)
    lib, _ = _stub(monkeypatch, llm)
    llm.add_request([3], SP(max_tokens=4))
    llm.add_request([4], SP(max_tokens=4, n=2))
    _drive(llm)
    names = {n for n, _ in lib.calls}
    assert names == {"lg_sample_rows_keyed"} and "lp" not in llm._state
    # a request with logprobs switches the draws while it runs, with 20 alternatives when it asks for any, and only then
    lib.calls.clear()
    llm.add_request([5], SP(max_tokens=3))
    llm.step()
    llm.add_request([6], SP(max_tokens=3, logprobs=2))
    _drive(llm)
    assert [c for c in lib.calls] == [("lg_sample_rows_guided", None), ("lg_sample_rows_logprobs", 20), ("lg_sample_rows_logprobs", 20),
                                      ("lg_sample_rows_logprobs", 20)]
    lib.calls.clear()
    llm.add_request([6], SP(max_tokens=2, best_of=1))
    _drive(llm)
    assert lib.calls == [("lg_sample_rows_logprobs", 0)] * 2


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_best_of_selection_order_and_prefix_entries(monkeypatch, kind):
    from test_serve_guidance import _add
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=6, seed=0)
    _stub(monkeypatch, llm)
    S = 5
    _add(llm, 0, SP(max_tokens=S, n=2, best_of=5, logprobs=1))
    _add(llm, 1, SP(max_tokens=S, n=3), prefix=[1, 2])
    outs = _drive(llm)
    o = outs["0"][1]
    cums = {j: float(np.sum([np.float32(_lp(0, j, k)) for k in range(S)], dtype=np.float64)) for j in range(5)}
    assert [c.index for c in o.outputs] == [1, 4]            # the two largest sums, descending
    for c in o.outputs:
        assert c.cumulative_logprob == pytest.approx(cums[c.index], abs=1e-12)
        assert len(c.logprobs) == S and all(isinstance(d, dict) for d in c.logprobs)
        tok = c.token_ids[0]
        assert c.logprobs[0][tok] == serve.Logprob(pytest.approx(_lp(0, c.index, 0)), 2) and c.logprobs[0][10000] == serve.Logprob(0.0, 1)
    # without logprobs or best_of: index order, no logprob fields
    assert [(c.index, c.cumulative_logprob, c.logprobs) for c in outs["1"][1].outputs] == [(0, None, None), (1, None, None), (2, None, None)]
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=6, seed=0)
    _stub(monkeypatch, llm)
    _add(llm, 7, SP(max_tokens=S, logprobs=0, n=2), prefix=[4, 5])
    c = _drive(llm)["0"][1].outputs
    assert [len(x.logprobs) for x in c] == [S, S] and c[0].logprobs[:2] == [None, None]
    assert all(len(d) == 1 for d in c[0].logprobs[2:])       # logprobs=0: the drawn token alone
    assert c[1].cumulative_logprob == pytest.approx(sum(float(np.float32(_lp(0, 1, k))) for k in range(2, S)), abs=1e-9)


def test_twins_mirror_logprobs(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=6, seed=0)
    _stub(monkeypatch, llm)
    sp = [SP(max_tokens=3, n=1, best_of=3, logprobs=2), SP(max_tokens=3)]
    outs = llm.generate(prompt_token_ids=[[3], [4], [10], [10]], sampling_params=sp + sp)
    for r, t in ((0, 2), (1, 3)):
        assert [(c.index, c.token_ids, c.cumulative_logprob, c.logprobs) for c in outs[t].outputs] == \
            [(c.index, c.token_ids, c.cumulative_logprob, c.logprobs) for c in outs[r].outputs]
    assert outs[0].outputs[0].logprobs is not None and outs[1].outputs[0].logprobs is None
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=4, seed=0)
    rid = llm.add_request([3], SP(max_tokens=3, logprobs=2))
    for bad in (SP(max_tokens=3), SP(max_tokens=3, logprobs=2, best_of=2)):
        with pytest.raises(ValueError, match="twin"):
            llm.add_request([10], bad, twin_of=rid)
