"""CPU: per-image temperature / top_k / top_p (lg_sample_cfg's row arrays) without a GPU: SampleCfg's layout and positional
compatibility, the argument handling and ValueErrors of generate() and sample() with the library calls stubbed, and
serve.LLM(per_request_sampling=True) with the device calls stubbed: a mixed-filter stream takes the steps of a uniform one, every join
and decode sees its slots' filters in the device state, t2i temperature 0 is greedy and c2i is not, a max_tokens change still drains
(and without the flag a top_k change), twins carry their request's filters, and the SJD schedule runs under the flag."""
import ctypes
import importlib
import types

import numpy as np
import pytest
import torch

from llamagen_b200 import _lib, serve
from test_serve_guidance import _add, _model
from test_serve_sjd import _Device as _SjdDevice, _drive

gen_mod = importlib.import_module("llamagen_b200.generate")
SP = serve.SamplingParams
V = 64


def _read(ptr, ctype, n):
    return list((ctype * n).from_address(ptr)) if ptr else None


def test_sample_cfg_layout_and_positional_compatibility():
    sc = _lib.SampleCfg(4.0, -1, 1.0, 100, 0.95, 0, 0)
    assert (sc.cfg_scale, sc.cfg_interval, sc.top_k, sc.greedy, sc.seed) == (4.0, -1, 100, 0, 0)
    assert sc.temperature_rows is None and sc.top_k_rows is None and sc.top_p_rows is None and sc.greedy_rows is None
    assert ctypes.sizeof(_lib.SampleCfg) == 64 and _lib.SampleCfg.temperature_rows.offset == 32
    assert [_lib.SampleCfg.__dict__[f].offset for f in ("top_k_rows", "top_p_rows", "greedy_rows")] == [40, 48, 56]


# ------------------------------------------------------------------------------------------------------------ generate() / sample()
class _Lib:
    """Records lg_sample / lg_generate*: the scalars and the row arrays' values at the call."""

    def __init__(self, B):
        self.B, self.calls = B, []

    def __getattr__(self, name):
        def call(*a):
            sc = next(x._obj for x in a if hasattr(x, "_obj") and isinstance(x._obj, _lib.SampleCfg))
            self.calls.append((name, (sc.temperature, sc.top_k, sc.top_p, sc.greedy),
                               (_read(sc.temperature_rows, ctypes.c_float, self.B), _read(sc.top_k_rows, ctypes.c_int32, self.B),
                                _read(sc.top_p_rows, ctypes.c_float, self.B), _read(sc.greedy_rows, ctypes.c_int32, self.B))))
            return 0
        return call


@pytest.fixture
def stubbed(monkeypatch):
    lib = _Lib(4)
    monkeypatch.setattr(_lib, "load", lambda *a, **k: lib)
    monkeypatch.setattr(_lib, "require_cuda", lambda t, what: t)
    monkeypatch.setattr(_lib, "current_stream", lambda dev: None)
    monkeypatch.setattr(gen_mod, "Transformer", object)
    model = types.SimpleNamespace(model_type="c2i", tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=V,
                                  setup_caches=lambda **kw: None, engine=lambda: None)
    return lib, model


def test_generate_per_image_filters_reach_the_call(stubbed):
    lib, model = stubbed
    cond = torch.tensor([1, 2, 3, 4])
    gen_mod.generate(model, cond, 8, cfg_scale=4.0, temperature=0.9, top_k=200, top_p=0.95, seed=1)
    name, scal, rows = lib.calls[-1]
    assert name == "lg_generate" and scal == (pytest.approx(0.9), 200, pytest.approx(0.95), 0) and rows == (None,) * 4
    gen_mod.generate(model, cond, 8, cfg_scale=4.0, temperature=[1.0, 0.7, 1.3, 0.0], top_k=np.array([0, -1, 7, 2 ** 40]),
                     top_p=torch.tensor([1.0, 0.9, 0.0, 1.5]), seed=1)
    name, _, (t, k, p, g) = lib.calls[-1]
    assert t == pytest.approx([1.0, 0.7, 1.3, 0.0]) and k == [0, 0, 7, 2 ** 31 - 1] and p == pytest.approx([1.0, 0.9, 0.0, 1.5])
    assert g is None                                         # greedy stays the call's sample_logits
    gen_mod.generate(model, cond, 8, temperature=0.5, top_k=[1, 2, 3, 4], seed=1)   # a number beside rows is repeated
    _, _, (t, k, p, _) = lib.calls[-1]
    assert t == [0.5] * 4 and k == [1, 2, 3, 4] and p == [1.0] * 4
    gen_mod.generate(model, cond, 8, top_k=torch.tensor(5), seed=1)                 # a 0-d tensor is a number
    assert lib.calls[-1][1][1] == 5 and lib.calls[-1][2] == (None,) * 4


@pytest.mark.parametrize("kw, match", [
    (dict(temperature=[1.0, 1.0, 1.0]), "4 values"), (dict(top_k=[1, 2, 3, 4, 5]), "4 values"), (dict(top_p=[[1.0] * 4]), "4 values"),
    (dict(temperature=[1.0, float("nan"), 1.0, 1.0]), "temperature"), (dict(temperature=[1.0, float("inf"), 1.0, 1.0]), "temperature"),
    (dict(temperature=[1.0, -0.5, 1.0, 1.0]), "temperature"), (dict(top_k=[1, 2.5, 3, 4]), "top_k"),
    (dict(top_k=[1, float("inf"), 3, 4]), "top_k"), (dict(top_p=[1.0, float("nan"), 1.0, 1.0]), "top_p"),
    (dict(top_k=[True, False, True, True]), "real numbers")])
def test_generate_and_sample_value_errors(stubbed, kw, match):
    lib, model = stubbed
    with pytest.raises(ValueError, match=match):
        gen_mod.generate(model, torch.tensor([1, 2, 3, 4]), 8, seed=1, **kw)
    with pytest.raises(ValueError, match=match):
        gen_mod.sample(torch.zeros(4, 1, V), seed=1, **kw)
    assert not lib.calls


def test_sample_rows(stubbed):
    lib, _ = stubbed
    gen_mod.sample(torch.zeros(4, 1, V), temperature=[1.0, 0.5, 2.0, 0.0], top_k=[0, 3, 9, 70], top_p=0.9, seed=3)
    name, _, (t, k, p, g) = lib.calls[-1]
    assert name == "lg_sample" and t == [1.0, 0.5, 2.0, 0.0] and k == [0, 3, 9, 70] and p == pytest.approx([0.9] * 4) and g is None
    gen_mod.sample(torch.zeros(4, 1, V), temperature=0.5, top_k=3, seed=3, sample_logits=False)
    assert lib.calls[-1][1] == (0.5, 3, 1.0, 1) and lib.calls[-1][2] == (None,) * 4


# ------------------------------------------------------------------------------------------------------------ serve.LLM
def _want(llm, p):
    return (np.float32(p.temperature), max(0, int(p.top_k)), np.float32(p.top_p), int(llm.t2i and p.temperature == 0))


def _check(llm, st, slot):
    p = llm._slots[slot].params
    got = (np.float32(st["temp"][slot]), int(st["topk"][slot]), np.float32(st["topp"][slot]), int(st["greedy"][slot]))
    assert got == _want(llm, p), (slot, llm._slots[slot].request_id, got)


class _Device:
    """Stand-ins for the device calls: every join and decode checks its slots' filters in the device state, and that the draw's
    SampleCfg points at them."""

    def __init__(self, monkeypatch, llm):
        self.llm, self.joins, self.decodes = llm, [], 0
        monkeypatch.setattr(serve.LLM, "_device_join_prefix", lambda llm, st, params, slot, P: self.join(llm, st, params, slot))
        monkeypatch.setattr(serve.LLM, "_device_step", lambda llm, st, params: self.decode(llm, st, params))
        monkeypatch.setattr(serve.LLM, "_device_join_t2i", lambda llm, st, params, slot: self.join(llm, st, params, slot))
        monkeypatch.setattr(serve.LLM, "_device_decode_t2i", lambda llm, st, params: self.decode(llm, st, params))

    def join(self, llm, st, params, slot):
        _check(llm, st, slot)
        sc = llm._sample_cfg(st, params, slice(slot, slot + 1))
        assert sc.temperature_rows == st["temp"][slot:].data_ptr() and sc.greedy_rows == st["greedy"][slot:].data_ptr()
        self.joins.append((slot, llm._slots[slot].request_id, llm.steps_run))
        st["tok"][slot] = 1

    def decode(self, llm, st, params):
        self.decodes += 1
        for b in range(llm.max_num_seqs):
            if llm._slots[b] is not None:
                _check(llm, st, b)
        sc = llm._sample_cfg(st, params, slice(0, llm.max_num_seqs))
        assert (sc.top_k_rows, sc.top_p_rows) == (st["topk"].data_ptr(), st["topp"].data_ptr())
        st["tok"].fill_(2)


FILTERS = [(1.0, 4000, 1.0), (1.0, 1000, 1.0), (0.9, 2000, 0.95), (1.0, 16384, 0.9), (0.0, -1, 1.0), (1.3, 0, 0.5), (0.7, 7, 1.0)]


def _stream(monkeypatch, kind, params, per_request=True, slots=3):
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=slots, seed=100, per_request_sampling=per_request)
    dev = _Device(monkeypatch, llm)
    for i, sp in enumerate(params[:4]):
        _add(llm, i, sp)
    llm.step()
    for i, sp in enumerate(params[4:], start=4):
        _add(llm, i, sp, prefix=[3, 4] if i == 5 else None)
    while llm.has_unfinished_requests():
        llm.step()
    return llm, dev


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_mixed_filters_share_one_batch(monkeypatch, kind):
    S = 4
    mixed = [SP(temperature=t, top_k=k, top_p=p, max_tokens=S, seed=i) for i, (t, k, p) in enumerate(FILTERS)]
    llm, dev = _stream(monkeypatch, kind, mixed)
    uniform, _ = _stream(monkeypatch, kind, [SP(max_tokens=S, seed=i) for i in range(len(FILTERS))])
    assert llm.steps_run == uniform.steps_run and dev.decodes > 0
    # the mixed stream without the flag drains at every change of filters
    drained, _ = _stream(monkeypatch, kind, mixed, per_request=False)
    assert drained.steps_run > llm.steps_run
    st = llm._state
    if kind == "t2i":       # the last joins: request 4 (temperature 0) was greedy in its slot, the others are not
        assert any(llm._slots[s] is None for s in range(3)) and {int(st["greedy"][s]) for s, r, _ in dev.joins if r == "4"} == {1}
    else:
        assert int(st["greedy"].sum()) == 0


def test_greedy_is_t2i_temperature_zero(monkeypatch):
    for kind, want in (("t2i", 1), ("c2i", 0)):
        llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=2, seed=0, per_request_sampling=True)
        seen = []
        dev = _Device(monkeypatch, llm)
        inner = dev.join
        dev.join = lambda llm_, st, params, slot: (seen.append(int(st["greedy"][slot])), inner(llm_, st, params, slot))
        _add(llm, 0, SP(temperature=0.0, max_tokens=2))
        _add(llm, 1, SP(temperature=1.0, max_tokens=2))
        while llm.has_unfinished_requests():
            llm.step()
        if kind == "t2i":
            assert seen == [want, 0]
        assert int(llm._state["greedy"][0]) == want and float(llm._state["temp"][0]) == 0.0


@pytest.mark.parametrize("per_request", [True, False])
def test_max_tokens_change_drains_and_without_the_flag_top_k_too(monkeypatch, per_request):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2, seed=0, per_request_sampling=per_request)
    _Device(monkeypatch, llm)
    for i, sp in enumerate([SP(top_k=10, max_tokens=3), SP(top_k=20, max_tokens=3), SP(top_k=10, max_tokens=4)]):
        _add(llm, i, sp)
    while llm.has_unfinished_requests():
        llm.step()
    # with the flag requests 0 and 1 share the batch and request 2 waits for them; without it every request waits
    assert llm.steps_run == (3 + 4 if per_request else 3 + 3 + 4)


def test_value_errors_and_twins():
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=2, per_request_sampling=True)
    t2i = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=2, per_request_sampling=True)
    f = torch.randn(3, 4)
    for sp in (SP(temperature=float("nan")), SP(temperature=-1.0), SP(temperature=float("inf")), SP(top_k=2.5), SP(top_p=float("nan")),
               SP(top_k=[3]), SP(temperature="1")):
        with pytest.raises(ValueError):
            llm.add_request([1], sp)
        with pytest.raises(ValueError):
            t2i.add_request(prompt_embeds=f, sampling_params=sp)
        with pytest.raises(ValueError):
            llm.generate(prompt_token_ids=[[1], [2], [10], [10]], sampling_params=[SP(), sp, SP(), sp])
    assert llm.get_num_unfinished_requests() == 0 and t2i.get_num_unfinished_requests() == 0
    # accepted: top_k -1 / 0 (off), numpy numbers, temperature 0, top_p outside (0, 1)
    for sp in (SP(top_k=-1), SP(top_k=0), SP(top_k=np.int64(5), temperature=np.float32(0.5)), SP(temperature=0.0, top_p=0.0),
               SP(top_p=2.0)):
        llm.add_request([1], sp)
    # a twin carries its request's filters
    sp = SP(temperature=0.8, top_k=50, top_p=0.9, max_tokens=2)
    rid = llm.add_request([3], sp)
    llm.add_request([10], sp, twin_of=rid)
    for other in (SP(temperature=1.0, top_k=50, top_p=0.9, max_tokens=2), SP(temperature=0.8, top_k=51, top_p=0.9, max_tokens=2),
                  SP(temperature=0.8, top_k=50, top_p=1.0, max_tokens=2)):
        with pytest.raises(ValueError, match="twin"):
            llm.add_request([10], other, twin_of=rid)
    # without the flag the filters are not checked when a request is added, as before
    serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2).add_request([1], SP(top_k=2.5))


def test_sjd_schedule_with_per_request_filters(monkeypatch):
    S = 8
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=3, seed=1, sjd_window=3, per_request_sampling=True)
    dev = _SjdDevice(monkeypatch, llm, seed=4)
    run = dev.run

    def checked(llm_, st):
        for b in range(llm_.max_num_seqs):
            if llm_._slots[b] is not None:
                _check(llm_, st, b)
        sc = llm_._sample_cfg(st, llm_._params, slice(0, llm_.max_num_seqs))
        assert sc.temperature_rows == st["temp"].data_ptr()
        run(llm_, st)
    monkeypatch.setattr(serve.LLM, "_device_sjd_pass", lambda llm_, st, params, dbg=None: checked(llm_, st))
    for i, (t, k, p) in enumerate(FILTERS):
        _add(llm, i, SP(temperature=t, top_k=k, top_p=p, max_tokens=S))
    outs = _drive(llm)
    assert sorted(outs) == [str(i) for i in range(len(FILTERS))]
    uni = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=3, seed=1, sjd_window=3, per_request_sampling=True)
    _SjdDevice(monkeypatch, uni, seed=4)
    for i in range(len(FILTERS)):
        _add(uni, i, SP(max_tokens=S))
    _drive(uni)
    assert llm.steps_run == uni.steps_run
