"""CPU: per-request guidance and seeds in serve.LLM with the device calls stubbed (SamplingParams(cfg_scale=, cfg_interval=, seed=)):
requests that differ only in these share one running batch, every join writes its slot's scale, interval and seed before its draw,
freed slots are rewritten by the next request, a change of top_k / max_tokens still drains, null-class twins mirror their request,
the ValueErrors; and the argument checks of lg_sample_rows_guided through the C-ABI without a GPU."""
import ctypes
import types

import numpy as np
import pytest
import torch

from llamagen_b200 import serve

T, C, V = 6, 4, 64
SP = serve.SamplingParams


def _model(model_type):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=V,
                                 cls_token_num=T if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None)


class _Device:
    """Stand-ins for the device calls. Every draw (a join's or a decode's) checks that each slot it draws for holds its request's
    guidance scale, cfg_interval and seed in the device state at that moment, and records (slot, request id) per draw."""

    def __init__(self, monkeypatch, llm):
        self.llm, self.joins, self.decodes = llm, [], 0
        monkeypatch.setattr(serve.LLM, "_device_join_prefix", lambda llm, *a: self.join(llm, *a[:3]))
        monkeypatch.setattr(serve.LLM, "_device_step", lambda llm, *a: self.decode(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_join_t2i", lambda llm, *a: self.join(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_decode_t2i", lambda llm, *a: self.decode(llm, *a))

    def expect(self, req):
        """(cfg, interval, seed) the slot of req must hold: its SamplingParams, or the LLM's defaults."""
        p, llm = req.params, self.llm
        return (llm.cfg_scale if p.cfg_scale is None else p.cfg_scale, -1 if p.cfg_interval is None else p.cfg_interval,
                llm._seed + int(req.request_id) if p.seed is None else p.seed)

    def check(self, st, slot):
        req = self.llm._slots[slot]
        want = self.expect(req)
        assert int(st["seeds"][slot]) == want[2], (slot, req.request_id)
        if "cfg" in st:
            assert float(st["cfg"][slot]) == pytest.approx(want[0], abs=0) and int(st["interval"][slot]) == want[1], (slot, req.request_id)
        else:
            assert self.llm.cfg_scale <= 1.0

    def join(self, llm, st, params, slot):
        self.check(st, slot)
        self.joins.append((slot, llm._slots[slot].request_id, llm.steps_run))
        k = 0 if llm._slots[slot].prefix is None else int(llm._slots[slot].prefix.numel())
        st["out"][slot, k] = 1
        st["tok"][slot] = 1

    def decode(self, llm, st, params):
        self.decodes += 1
        B = llm.max_num_seqs
        for b in range(B):
            if llm._slots[b] is not None:
                self.check(st, b)
        k = st["step"] if llm.t2i else st["pos"][:B]
        for b in range(B):
            st["out"][b, int(k[b]) % st["S"]] = 2
        st["tok"].fill_(2)


def _feats(n, seed):
    return torch.randn(n, C, generator=torch.Generator().manual_seed(seed))


def _add(llm, i, sp, **kw):
    if llm.t2i:
        return llm.add_request(prompt_embeds=_feats(2 + i % 3, i), sampling_params=sp, **kw)
    return llm.add_request([i % 10], sp, **kw)


def _schedule(monkeypatch, kind, params):
    """Four requests, one step, three more (one of them a completion request), then run to the end on three slots. Returns
    (steps_run, the stub, {request id: slot of its join})."""
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=3, seed=100)
    dev = _Device(monkeypatch, llm)
    for i, sp in enumerate(params[:4]):
        _add(llm, i, sp)
    outs = llm.step()                                       # r0 .. r2 join; r3 waits for a slot
    for i, sp in enumerate(params[4:], start=4):
        _add(llm, i, sp, prefix=[3, 4] if i == 5 else None)
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert sorted(int(o.request_id) for o in outs) == list(range(len(params)))
    assert all(len(o.outputs[0].token_ids) == params[0].max_tokens for o in outs)
    return llm.steps_run, dev


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_mixed_guidance_shares_one_batch_and_every_draw_sees_its_slot(monkeypatch, kind):
    S = 4
    mixed = [SP(top_k=10, max_tokens=S, cfg_scale=c, cfg_interval=k, seed=s)
             for c, k, s in [(1.0, None, None), (7.5, 3, 12345), (None, 0, None), (2.0, None, 2 ** 63 - 1), (0.5, 5, 7),
                             (4.0, -1, None), (7.5, None, 0)]]
    steps, dev = _schedule(monkeypatch, kind, mixed)       # every join and decode checks the slots' cfg / interval / seed
    uniform, _ = _schedule(monkeypatch, kind, [SP(top_k=10, max_tokens=S)] * len(mixed))
    # no drain: the mixed requests take exactly the steps of requests with one SamplingParams (a drain per change would add S - 1
    # steps for each of the six changes)
    assert steps == uniform and steps < 7 * S // 2, (steps, uniform)
    assert dev.decodes > 0
    if kind == "t2i":                                      # t2i: every request joins through a device join, slots are reused
        assert [rid for _, rid, _ in dev.joins] == [str(i) for i in range(7)]
        assert len({s for s, _, _ in dev.joins}) == 3


def test_slots_are_rewritten_by_the_next_request(monkeypatch):
    llm = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=1, seed=5)
    dev = _Device(monkeypatch, llm)
    for i, sp in enumerate([SP(max_tokens=2, cfg_scale=7.5, cfg_interval=1, seed=9), SP(max_tokens=2), SP(max_tokens=2, cfg_scale=1.0)]):
        _add(llm, i, sp)
    while llm.has_unfinished_requests():
        llm.step()
    st = llm._state
    assert [(s, r) for s, r, _ in dev.joins] == [(0, "0"), (0, "1"), (0, "2")]
    # the last request's values are what the slot holds now: the second request's defaults overwrote the first one's 7.5 / 1 / 9
    assert float(st["cfg"][0]) == 1.0 and int(st["interval"][0]) == -1 and int(st["seeds"][0]) == 5 + 2


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_top_k_or_max_tokens_change_still_drains(monkeypatch, kind):
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=2, seed=0)
    dev = _Device(monkeypatch, llm)
    a = SP(top_k=10, max_tokens=3, cfg_scale=2.0, seed=1)
    b = SP(top_k=20, max_tokens=3, cfg_scale=2.0, seed=1)          # same guidance and seed, other top_k
    c = SP(top_k=10, max_tokens=4, cfg_scale=7.5)                  # other max_tokens
    for i, sp in enumerate([a, b, a, c]):
        _add(llm, i, sp)
    while llm.has_unfinished_requests():
        llm.step()
    # every request differs from the one before it in top_k or max_tokens: each waits for the drain of the previous one
    assert llm.steps_run == 3 + 3 + 3 + 4
    if kind == "t2i":
        assert [(rid, step) for _, rid, step in dev.joins] == [("0", 0), ("1", 3), ("2", 6), ("3", 9)]


def test_c2i_twins_mirror_their_request(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=2, seed=0)
    dev = _Device(monkeypatch, llm)
    sp = [SP(max_tokens=2, cfg_scale=7.5, cfg_interval=0, seed=31), SP(max_tokens=2, cfg_scale=1.0)]
    outs = llm.generate(prompt_token_ids=[[3], [4], [10], [10]], sampling_params=sp + sp)
    assert [o.request_id for o in outs] == ["0", "1", "2", "3"]
    assert outs[2].outputs[0].token_ids == outs[0].outputs[0].token_ids and outs[3].outputs[0].token_ids == outs[1].outputs[0].token_ids
    assert dev.decodes == 2 and llm.steps_run == 2
    # a twin added by hand may repeat its request's params, not change their guidance or seed
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=2, seed=0)
    rid = llm.add_request([3], sp[0])
    llm.add_request([10], sp[0], twin_of=rid)
    for other in (SP(max_tokens=2, cfg_scale=7.0, cfg_interval=0, seed=31), SP(max_tokens=2, cfg_scale=7.5, seed=31),
                  SP(max_tokens=2, cfg_scale=7.5, cfg_interval=0)):
        with pytest.raises(ValueError, match="twin"):
            llm.add_request([10], other, twin_of=rid)
    with pytest.raises(ValueError):                                # LLM.generate: the twins' params must equal their requests'
        serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10).generate(prompt_token_ids=[[3], [10]],
                                                                          sampling_params=[sp[0], SP(max_tokens=2, cfg_scale=7.5)])


def test_value_errors():
    t2i = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=2)
    t2i_nocfg = serve.LLM(_model("t2i"), cfg_scale=1.0, max_num_seqs=2)
    c2i, c2i_nocfg = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2), serve.LLM(_model("c2i"), cfg_scale=1.0, max_num_seqs=2)
    f = _feats(3, 0)
    bad_params = [SP(cfg_scale=float("nan")), SP(cfg_scale=float("inf")), SP(cfg_scale=-float("inf")), SP(cfg_scale="4"),
                  SP(cfg_scale=True), SP(cfg_interval=-2), SP(cfg_interval=1.5), SP(cfg_interval="3"), SP(cfg_interval=True),
                  SP(seed=-1), SP(seed=2 ** 63), SP(seed=1.0), SP(seed="1"), SP(seed=False)]
    bad = []
    for sp in bad_params:
        bad += [lambda sp=sp: t2i.add_request(prompt_embeds=f, sampling_params=sp),
                lambda sp=sp: t2i.generate(prompt_embeds=[f, f], sampling_params=[SP(), sp]),
                lambda sp=sp: c2i_nocfg.add_request([1], sp),
                lambda sp=sp: c2i_nocfg.generate(prompt_token_ids=[[1], [2]], sampling_params=[SP(), sp])]
    bad += [
        lambda: t2i_nocfg.add_request(prompt_embeds=f, sampling_params=SP(cfg_scale=1.5)),       # no unconditional rows
        lambda: t2i_nocfg.generate(prompt_embeds=[f, f], sampling_params=[SP(), SP(cfg_scale=4.0)]),
        lambda: c2i_nocfg.add_request([1], SP(cfg_scale=1.0001)),
        lambda: c2i_nocfg.generate(prompt_token_ids=[[1], [2]], sampling_params=[SP(), SP(cfg_scale=2.0)]),
        # a negative prompt with an effective cfg_scale <= 1
        lambda: t2i.add_request(prompt_embeds=f, negative_prompt_embeds=f, sampling_params=SP(cfg_scale=1.0)),
        lambda: t2i.generate(prompt_embeds=[f, f], negative_prompt_embeds=[None, f], sampling_params=[SP(), SP(cfg_scale=0.5)]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    for llm in (t2i, t2i_nocfg, c2i, c2i_nocfg):
        assert llm.get_num_unfinished_requests() == 0                 # nothing was queued
    # accepted: cfg_interval on an LLM without CFG (no effect), scales <= 1 anywhere, numpy integers and floats, the seed bounds
    t2i_nocfg.add_request(prompt_embeds=f, sampling_params=SP(cfg_interval=3, cfg_scale=0.0))
    c2i.add_request([1], SP(cfg_scale=np.float32(7.5), cfg_interval=np.int64(2), seed=np.int64(2 ** 63 - 1)))
    c2i.add_request([1], SP(cfg_scale=1, seed=0))
    t2i.add_request(prompt_embeds=f, negative_prompt_embeds=f, sampling_params=SP(cfg_scale=1.01))
    assert [r.cfg for r in c2i._waiting] == [7.5, 1.0] and [r.seed for r in c2i._waiting] == [2 ** 63 - 1, 0]
    assert (t2i_nocfg._waiting[0].interval, t2i._waiting[0].cfg) == (3, pytest.approx(1.01))


def test_positional_sampling_params_keep_their_meaning():
    sp = SP(0.0, 0.9, 50, 16)
    assert (sp.temperature, sp.top_p, sp.top_k, sp.max_tokens) == (0.0, 0.9, 50, 16)
    assert (sp.cfg_scale, sp.cfg_interval, sp.seed) == (None, None, None)


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_sample_rows_guided_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no call below reaches a launch
    sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 0, 0)

    def guided(logits=p, B=1, V=V, mix=1, sc=ctypes.byref(sc), seeds=p, steps=p, cfg=p, interval=p, idx=p, seq=p):
        return lib.lg_sample_rows_guided(logits, B, V, mix, _lib.LG_DTYPE_F32, sc, seeds, steps, cfg, interval, idx, seq, 1, None)

    def plain(logits=p, seeds=p, steps=p, idx=p, seq=p, B=1):
        return lib.lg_sample_rows(logits, B, V, 1, _lib.LG_DTYPE_F32, ctypes.byref(sc), seeds, steps, idx, seq, 1, None)

    for rc_call, msg in [
        (lambda: guided(mix=0), b"lg_sample_rows_guided: per-row cfg_rows / interval_rows need mix_cfg"),
        (lambda: guided(mix=0, interval=None), b"need mix_cfg"),
        (lambda: guided(mix=0, cfg=None), b"need mix_cfg"),
        (lambda: guided(logits=None), b"lg_sample_rows_guided: null argument"),
        (lambda: guided(sc=None), b"lg_sample_rows_guided: null argument"),
        (lambda: guided(seeds=None), b"lg_sample_rows_guided: null argument"),
        (lambda: guided(steps=None), b"lg_sample_rows_guided: null argument"),
        (lambda: guided(idx=None, seq=None), b"lg_sample_rows_guided: null argument"),
        (lambda: guided(B=0), b"bad shape B=0"),
        (lambda: guided(B=0, mix=0, cfg=None, interval=None), b"bad shape B=0"),
        (lambda: plain(logits=None), b"lg_sample_rows: null argument"),
        (lambda: plain(idx=None, seq=None), b"lg_sample_rows: null argument"),
        (lambda: plain(B=0), b"bad shape B=0"),
    ]:
        assert rc_call() < 0, msg
        assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
