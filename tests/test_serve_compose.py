"""CPU: composable-guidance requests in serve.LLM (SamplingParams(cond_weights=)) with the engine replaced by a recording library that
draws on the host: a composed request takes n * K slots (the lowest free ones, at once, never overtaken), its lead and condition slots
and image indices, the gather table and lead map in the device state before every draw (freed slots rewritten, plain slots plain), no
drain on a change of cond_weights, a sample's K slots freed together with the lead slot's token row as its output, every ValueError,
null-class twins mirroring cond_weights, LLM.generate's nested conditions with one encoder call, and the argument checks of
lg_sample_rows_composed through the C-ABI without a GPU."""
import ctypes
import types

import pytest
import torch

from llamagen_b200 import _lib, serve

T2I_T, C, V, M = 6, 4, 64, 8
SP = serve.SamplingParams
DRAWS = ("lg_sample_rows", "lg_sample_rows_guided", "lg_sample_rows_keyed", "lg_sample_rows_logprobs", "lg_sample_rows_given",
         "lg_sample_rows_composed")


def _model(model_type):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=V,
                                 cls_token_num=T2I_T if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None, engine=lambda: None,
                                 _slot_scratch=lambda use_cfg: (None, 0), _slot_prefix_scratch=lambda use_cfg, P: (None, 0),
                                 _slot_extend_scratch=lambda use_cfg, K: (None, 0))


def _token(seed, img, k):
    """The token the host draw makes for image img of a request with this seed at index k."""
    return 16 + (seed * 7 + img * 13 + k) % 48


class _Lib:
    """The engine's entry points serve.LLM calls, recorded as (name, step, detail). Every draw is made on the host from the pointers it
    is given, and checks the gather table: every running slot's row of st["mix_rows"] / st["mix_w"] / st["lead"] is what its request
    and role make it, and a composed draw's rows are read where the pointers say."""

    def __init__(self, llm):
        self.llm, self.real, self.calls, self.draws = llm, _lib.load(), [], []

    def __getattr__(self, name):
        if name in DRAWS:
            return lambda *a: self.draw(name, *a)
        if name.startswith(("lg_decode", "lg_prefill", "lg_copy", "lg_extend")):
            return lambda *a: self.rec(name, a)
        return getattr(self.real, name)

    def rec(self, name, args):
        if name.startswith("lg_decode"):
            self.check_inputs()
        detail = None
        if name == "lg_copy_slot_kv":
            detail = (args[1], [args[2][i] for i in range(args[3])], args[6])
        elif name.startswith("lg_prefill"):
            detail = args[-7]   # the slot
        self.calls.append((name, self.llm.steps_run, detail))
        return 0

    def expected_row(self, s):
        llm, B = self.llm, self.llm.max_num_seqs
        r = llm._slots[s]
        if r.weights is None:
            return [-1] * (1 + M), [0.0] * M
        if llm._lead[s] != s:
            return [-2] + [-1] * M, [0.0] * M
        slots = [s] + [c for c in range(B) if c != s and llm._lead[c] == s]
        return [B + s] + slots + [-1] * (M - r.K), list(r.weights) + [0.0] * (M - r.K)

    def check_tables(self):
        st, llm = self.llm._state, self.llm
        if "mix_rows" not in st:
            assert all(r is None or r.weights is None for r in llm._slots)
            return
        for s, r in enumerate(llm._slots):
            if r is not None:
                row, w = self.expected_row(s)
                assert st["mix_rows"][s].tolist() == row, (s, st["mix_rows"][s].tolist(), row)
                assert st["mix_w"][s].tolist() == pytest.approx(w, abs=0), s
                assert int(st["lead"][s]) == llm._lead[s], s

    def check_inputs(self):
        """Before a decode: a condition slot's next input is its lead's token, or at position 0 (c2i) its own class."""
        st, llm = self.llm._state, self.llm
        for s, r in enumerate(llm._slots):
            if r is not None and r.weights is not None and llm._lead[s] != s:
                lead = llm._lead[s]
                if not llm.t2i and int(st["pos"][s]) == 0:
                    assert int(st["tok"][s]) == r.prompt_token_ids[(s in llm._sample_slots(lead)) and llm._sample_slots(lead).index(s)]
                else:
                    assert int(st["tok"][s]) == int(st["tok"][lead]), (s, lead)

    def draw(self, name, logits, *a):
        st, llm = self.llm._state, self.llm
        if name == "lg_sample_rows_composed":
            nrows, n, V_, dt, sc, seeds, steps, cfg, interval, img, given, mix_rows, mix_w = a[:13]
        else:
            n, V_, use_cfg, dt, sc, seeds, steps = a[:7]
            mix_rows = None
        out_seq = a[-3]
        self.check_tables()
        s0 = (seeds.value - st["seeds"].data_ptr()) // 8
        src = next(t for t in (st["pos"], st["join_step"], st.get("step"), st.get("step0")) if t is not None and
                   0 <= steps.value - t.data_ptr() < t.numel() * 4)
        step = src.view(-1)[(steps.value - src.data_ptr()) // 4:][:n if src.numel() > 1 else 1]
        row0 = (out_seq.value - st["out"].data_ptr()) // (4 * st["S"])
        roles = []
        for j in range(n):
            slot, k = s0 + j, int(step[j if step.numel() > 1 else 0])
            req = llm._slots[slot]
            if mix_rows is not None:
                if mix_rows.value == st["join_rows"].data_ptr():
                    row = st["join_rows"][0].tolist()
                    assert row[:1 + req.K] == [1] + [2 * i for i in range(req.K)] and n == 1 and nrows == 2 * req.K
                    assert st["join_w"][0].tolist()[:req.K] == pytest.approx(list(req.weights), abs=0)
                else:
                    row = st["mix_rows"].view(-1)[(mix_rows.value - st["mix_rows"].data_ptr()) // 4:][j * (1 + M):(j + 1) * (1 + M)].tolist()
                    assert nrows == 2 * llm.max_num_seqs
                roles.append(row[0])
                if row[0] == -2:
                    continue
            elif req is not None:
                assert req.weights is None, f"slot {slot}: a composed request drawn by {name}"
            t = 0 if req is None else _token(req.seed, llm._img[slot], k)
            st["out"][row0 + j, k] = t
            st["tok"][s0 + j] = t
        self.draws.append((name, llm.steps_run, s0, n, roles))
        self.calls.append((name, llm.steps_run, (s0, n)))
        return 0


class _Encoder:
    """A stub text encoder: caption i of a call is features filled with len(text); records every call's strings."""
    d_model = C

    def __init__(self):
        self.calls = []

    def __call__(self, texts):
        self.calls.append(list(texts))
        embs = torch.stack([torch.full((T2I_T, C), float(len(t))) for t in texts])
        return embs, torch.ones(len(texts), T2I_T, dtype=torch.int64)


def _llm(monkeypatch, kind, cfg_scale=4.0, **kw):
    llm = serve.LLM(_model(kind), cfg_scale=cfg_scale, num_classes=10, seed=5, **kw)
    lib = _Lib(llm)
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "current_stream", lambda dev: None)
    return llm, lib


def _feats(i):
    return torch.randn(2 + i % 3, C, generator=torch.Generator().manual_seed(i))


def _add(llm, i, sp, K=None, **kw):
    """Request i: plain, or with sp.cond_weights K conditions (classes i + c, or captions of seeds i, 100 + i, ...)."""
    K = None if sp.cond_weights is None else len(sp.cond_weights)
    if llm.t2i:
        emb = _feats(i) if K is None else [_feats(100 * c + i) for c in range(K)]
        return llm.add_request(prompt_embeds=emb, sampling_params=sp, **kw)
    return llm.add_request([i % 10] if K is None else [(i + c) % 10 for c in range(K)], sp, **kw)


def _drive(llm, watch=None):
    outs = {}
    while llm.has_unfinished_requests():
        step = llm.steps_run
        for o in llm.step():
            assert o.request_id not in outs
            outs[o.request_id] = (step, o)
        if watch is not None:
            watch(llm)
    return outs


def _samples_whole(llm):
    """Every running composed sample holds all K of its slots (they are freed together)."""
    for s, r in enumerate(llm._slots):
        if r is not None and llm._lead[s] == s:
            assert len(llm._sample_slots(s)) == r.K, (s, llm._sample_slots(s))


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_admission_roles_tables_and_outputs(monkeypatch, kind):
    S = 5
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=8)
    reqs = [SP(max_tokens=S, cond_weights=(3.0, 1.5)),                     # slots 0, 1
            SP(max_tokens=S),                                              # slot 2
            SP(max_tokens=S, cond_weights=(2.0, -0.5, 0.0), n=2),          # slots 3 .. 8: waits (only 5 free)
            SP(max_tokens=S)]                                              # not overtaking it
    for i, sp in enumerate(reqs):
        _add(llm, i, sp)
    llm.step()
    assert [None if r is None else r.request_id for r in llm._slots] == ["0", "0", "1"] + [None] * 5
    assert llm._lead[:3] == [0, 0, 2] and llm._img[:3] == [0, 0, 0]
    assert [r.request_id for r in llm._waiting] == ["2", "3"]            # the composed request waits, and the plain one behind it
    outs = _drive(llm, _samples_whole)
    assert sorted(outs, key=int) == ["0", "1", "2", "3"]
    assert outs["2"][0] > outs["0"][0] and outs["3"][0] >= outs["2"][0]       # request 3 did not overtake request 2
    for step, o in outs.values():
        r_out = o.outputs
        sp = reqs[int(o.request_id)]
        assert [c.index for c in r_out] == list(range(sp.n))
        seed = llm._seed + int(o.request_id)
        for c in r_out:      # the lead slot's token row: every token the host drew for that sample's image index
            assert c.token_ids == [_token(seed, c.index, k) for k in range(S)], o.request_id
    # the batch draws while a composed slot ran were composed draws (the stub refuses any other draw of a composed slot), with -2 rows
    # for the condition slots
    composed = [d for d in lib.draws if d[0] == "lg_sample_rows_composed"]
    assert composed and any(-2 in d[4] for d in composed)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_lowest_free_slots_image_major(monkeypatch, kind):
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=8)
    sp = SP(max_tokens=6)
    _add(llm, 0, sp)                                                      # slot 0
    _add(llm, 1, sp)                                                      # slot 1
    llm.step()
    _add(llm, 2, sp)                                                      # slot 2, one step later
    _add(llm, 3, SP(max_tokens=6, cond_weights=(1.5, 2.5, 0.5), n=2))     # 6 slots: waits for slots 0 and 1, then 0, 1, 3 .. 6
    llm.step()
    assert [r.request_id for r in llm._waiting] == ["3"]
    while llm._waiting:
        llm.step()
    slots = [s for s, r in enumerate(llm._slots) if r is not None and r.request_id == "3"]
    assert slots == [0, 1, 3, 4, 5, 6]
    # sample j's condition i in the (j K + i)-th slot: leads 0 and 4, image indices 0 and 1
    assert [llm._lead[s] for s in slots] == [0, 0, 0, 4, 4, 4] and [llm._img[s] for s in slots] == [0, 0, 0, 1, 1, 1]
    B = llm.max_num_seqs
    st = llm._state
    assert st["mix_rows"][0].tolist() == [B + 0, 0, 1, 3] + [-1] * 5 and st["mix_rows"][4].tolist() == [B + 4, 4, 5, 6] + [-1] * 5
    assert [st["mix_rows"][s][0].item() for s in (1, 3, 5, 6)] == [-2] * 4 and st["mix_rows"][2][0].item() == -1
    _drive(llm, _samples_whole)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_freed_slots_are_rewritten(monkeypatch, kind):
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=3)
    for i, sp in enumerate([SP(max_tokens=3, cond_weights=(2.0, 1.0, 0.5)), SP(max_tokens=3), SP(max_tokens=3, cond_weights=(4.0, 1.0)),
                            SP(max_tokens=3, cond_weights=(7.5,))]):
        _add(llm, i, sp)
    outs = _drive(llm)          # every draw checks every running slot's row (plain rows -1 in slots a composed request held)
    assert sorted(outs, key=int) == ["0", "1", "2", "3"]
    st = llm._state
    assert st["mix_rows"][0].tolist()[:2] == [3 + 0, 0] and st["lead"].tolist() == [0, 1, 2]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_cond_weights_do_not_drain(monkeypatch, kind):
    S = 4

    def run(params):
        llm, lib = _llm(monkeypatch, kind, max_num_seqs=4)
        for i, sp in enumerate(params):
            _add(llm, i, sp)
        outs = _drive(llm)
        assert len(outs) == len(params)
        return llm.steps_run

    mixed = [SP(max_tokens=S, cond_weights=w) for w in [(2.0, 2.0), (1.0, -1.0), (4.0, 0.0), (3.0, 3.0), (0.5, 8.0), (1.0, 1.0)]]
    uniform = [SP(max_tokens=S, cond_weights=(2.0, 2.0))] * len(mixed)
    assert run(mixed) == run(uniform) < 6 * S


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("prefix", [False, True])
def test_joins_prefill_each_condition_and_fan_out(monkeypatch, kind, prefix):
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=6)
    P = 2 if prefix else 0
    _add(llm, 0, SP(max_tokens=5, cond_weights=(3.0, 0.5, 1.0), n=2), prefix=[7, 8] if prefix else None)
    outs = _drive(llm)
    prefills = [d for n, step, d in lib.calls if n.startswith("lg_prefill")]
    copies = [d for n, step, d in lib.calls if n == "lg_copy_slot_kv"]
    if kind == "c2i" and not prefix:        # the K classes enter at position 0: no prefill, no copy
        assert prefills == [] and copies == []
    else:                                   # sample 0's K slots, each alone, then condition i's K / V to sample 1's slot 3 + i
        assert prefills == [0, 1, 2]
        assert copies == [(0, [3], llm.model.cls_token_num + P), (1, [4], llm.model.cls_token_num + P), (2, [5], llm.model.cls_token_num + P)]
        join_draws = [d for d in lib.draws if d[1] == 0 and d[3] == 1]
        assert [d[2] for d in join_draws] == [0, 3] and all(d[0] == "lg_sample_rows_composed" for d in join_draws)
    toks = outs["0"][1].outputs
    seed = llm._seed
    for c in toks:
        assert c.token_ids[:P] == [7, 8][:P]
        assert c.token_ids[P:] == [_token(seed, c.index, k) for k in range(P, 5)]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_plain_batches_call_what_they_called(monkeypatch, kind):
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=3)
    for i in range(4):
        _add(llm, i, SP(max_tokens=3))
    _drive(llm)
    assert "mix_rows" not in llm._state
    assert not any(n == "lg_sample_rows_composed" for n, _, _ in lib.calls)
    # once a composed request has run, later plain-only batches draw as before
    _add(llm, 9, SP(max_tokens=3, cond_weights=(2.0, 1.0)))
    _drive(llm)
    n_before = len(lib.calls)
    _add(llm, 10, SP(max_tokens=3))
    _drive(llm)
    assert not any(n == "lg_sample_rows_composed" for n, _, _ in lib.calls[n_before:])


def test_value_errors():
    f = _feats(0)
    c2i = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=4)
    t2i = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=4)
    c2i_nocfg = serve.LLM(_model("c2i"), cfg_scale=1.0, num_classes=10, max_num_seqs=4)
    t2i_sjd = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=4, sjd_window=4)
    w2 = (2.0, 1.0)
    bad = [
        lambda: c2i_nocfg.add_request([1, 2], SP(cond_weights=w2)),                       # no unconditional rows
        lambda: c2i.add_request([1, 2], SP(cond_weights=w2, cfg_scale=4.0)),              # cfg_scale with the weights
        lambda: t2i.add_request(prompt_embeds=[f, f], sampling_params=SP(cond_weights=w2, cfg_scale=2.0)),
        lambda: c2i.add_request([1, 2], SP(cond_weights=w2, cfg_interval=3)),             # cfg_interval with K > 1
        lambda: c2i.add_request([1, 2, 3], SP(cond_weights=w2)),                          # K != the conditions
        lambda: c2i.add_request([1], SP(cond_weights=w2)),
        lambda: c2i.add_request([1, 10], SP(cond_weights=w2)),                            # the null class is no condition
        lambda: t2i.add_request(prompt_embeds=[f], sampling_params=SP(cond_weights=w2)),
        lambda: t2i.add_request(prompt_embeds=f, sampling_params=SP(cond_weights=w2)),
        lambda: t2i.add_request(prompt_embeds=[f, f, f], sampling_params=SP(cond_weights=w2)),
        lambda: c2i.add_request([1, 2], SP(max_tokens=4, cond_weights=w2), given=[1, 2, 3, 4], given_mask=[True, False, False, False]),
        lambda: t2i.add_request(prompt_embeds=[f, f], sampling_params=SP(max_tokens=4, cond_weights=w2), given=[1, 2, 3, 4],
                                given_mask=[True, False, False, False]),
        lambda: t2i_sjd.add_request(prompt_embeds=[f, f], sampling_params=SP(cond_weights=w2)),   # SJD
        lambda: t2i_sjd.add_request(prompt_embeds=f, sampling_params=SP(cond_weights=(2.0,))),
        lambda: c2i.add_request([1, 2], SP(cond_weights=w2, n=3)),                        # n K = 6 > 4 slots
        lambda: c2i.add_request([1, 2], SP(cond_weights=w2, n=1, best_of=3)),             # best_of K = 6 > 4
        lambda: c2i.add_request([1] * 9, SP(cond_weights=(1.0,) * 9, n=1)),               # K > 8
        lambda: c2i.add_request([], SP(cond_weights=())),
        lambda: c2i.add_request([1], SP(cond_weights=(float("nan"),))),
        lambda: c2i.add_request([1], SP(cond_weights=(1e39,))),                           # not finite in fp32
        lambda: c2i.add_request([1], SP(cond_weights=(True,))),
        lambda: c2i.add_request([1], SP(cond_weights="2")),
        lambda: c2i.add_request([1], SP(cond_weights=2.0)),
        lambda: c2i.add_request([1, 2], SP(cond_weights=((1.0, 2.0),))),
        lambda: c2i.generate(prompt_token_ids=[[1, 2, 3], [3], [10], [10]], sampling_params=[SP(cond_weights=w2), SP()] * 2),
        lambda: c2i.generate(prompt_token_ids=[[3], [1, 2, 3], [10], [10]], sampling_params=[SP(), SP(cond_weights=w2)] * 2),
        lambda: t2i.generate(prompt_embeds=[f, [f]], sampling_params=[SP(), SP(cond_weights=w2)]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    for llm in (c2i, t2i, c2i_nocfg, t2i_sjd):
        assert llm.get_num_unfinished_requests() == 0, llm       # nothing was queued
    # accepted: K = 1 with a bare caption, zero and negative weights, cfg_interval with K = 1, numpy weights, a negative prompt
    import numpy as np
    t2i.add_request(prompt_embeds=f, sampling_params=SP(cond_weights=[7.5], cfg_interval=2))
    t2i.add_request(prompt_embeds=[f, f], negative_prompt_embeds=f, sampling_params=SP(cond_weights=np.array([0.0, -1.0])))
    c2i.add_request([1, 2], SP(cond_weights=w2, n=2))
    assert [r.weights for r in t2i._waiting] == [(7.5,), (0.0, -1.0)] and t2i._waiting[0].interval == 2
    assert SP(cond_weights=[1, 2]).cond_weights == (1, 2) and hash(SP(cond_weights=[1, 2])) == hash(SP(cond_weights=(1, 2)))


def test_c2i_twins_mirror_cond_weights(monkeypatch):
    llm, lib = _llm(monkeypatch, "c2i", max_num_seqs=4)
    sp = [SP(max_tokens=3, cond_weights=(3.0, -0.5), seed=11), SP(max_tokens=3)]
    outs = llm.generate(prompt_token_ids=[[3, 4], [5], [10], [10]], sampling_params=sp + sp)
    assert [o.request_id for o in outs] == ["0", "1", "2", "3"]
    assert outs[0].prompt_token_ids == [3, 4] and outs[2].prompt_token_ids == [10]
    assert outs[2].outputs[0].token_ids == outs[0].outputs[0].token_ids == [_token(11, 0, k) for k in range(3)]
    llm, lib = _llm(monkeypatch, "c2i", max_num_seqs=4)
    rid = llm.add_request([3, 4], sp[0])
    llm.add_request([10], sp[0], twin_of=rid)
    for other in (SP(max_tokens=3, cond_weights=(3.0, -0.25), seed=11), SP(max_tokens=3, seed=11)):
        with pytest.raises(ValueError, match="twin"):
            llm.add_request([10], other, twin_of=rid)
    with pytest.raises(ValueError):                              # a twin's prompt stays the single null class
        llm.add_request([10, 10], sp[0], twin_of=rid)


def test_generate_nested_conditions_one_encoder_call(monkeypatch):
    enc = _Encoder()
    llm = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=4, seed=3, text_encoder=enc)
    lib = _Lib(llm)
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "current_stream", lambda dev: None)
    sp = [SP(max_tokens=3, cond_weights=(2.0, 1.0)), SP(max_tokens=3), SP(max_tokens=3, cond_weights=(5.0,))]
    outs = llm.generate(prompts=[["a castle", "watercolor"], "a dog", "x"], sampling_params=sp, negative_prompts=[None, None, "blurry"])
    assert enc.calls == [["a castle", "watercolor", "a dog", "x", "blurry"]]
    assert [len(o.outputs) for o in outs] == [1, 1, 1]
    # the prompt_embeds surface: a list of K captions for a composed request, a bare caption for K = 1
    f = [_feats(i) for i in range(3)]
    outs = llm.generate(prompt_embeds=[[f[0], f[1]], f[2], f[0]], sampling_params=sp)
    assert len(outs) == 3
    # add_request(prompt=[...]) with a negative: one encoder call
    enc.calls.clear()
    llm.add_request(prompt=["a", "bb", "ccc"], negative_prompt="dddd", sampling_params=SP(max_tokens=3, cond_weights=(1.0, 2.0, 3.0)))
    assert enc.calls == [["a", "bb", "ccc", "dddd"]]
    r = llm._waiting[-1]
    assert [float(c[0][-1, 0]) for c in r.conds] == [1.0, 2.0, 3.0] and float(r.neg[-1, 0]) == 4.0
    _drive(llm)


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_sample_rows_composed_argument_checks():
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no call below reaches a launch
    sc = _lib.SampleCfg(1.0, -1, 1.0, 0, 1.0, 0, 0)

    def composed(logits=p, rows=2, B=1, V=V, rd=_lib.LG_DTYPE_F32, sc=ctypes.byref(sc), seeds=p, steps=p, given=None, mix=p, w=p,
                 lp=None, idx=p, seq=p, stride=1):
        return lib.lg_sample_rows_composed(logits, rows, B, V, rd, sc, seeds, steps, None, None, None, given, mix, w, lp, idx, seq, stride,
                                           None)

    fn = b"lg_sample_rows_composed"
    for call, msg in [
        (lambda: composed(rows=1), fn + b": bad shape rows=1 B=1"),
        (lambda: composed(rows=7, B=4), fn + b": bad shape rows=7 B=4"),
        (lambda: composed(B=0), fn + b": bad shape"),
        (lambda: composed(V=0), fn + b": bad shape"),
        (lambda: composed(mix=None), fn + b": mix_rows and mix_weights go together"),
        (lambda: composed(w=None), fn + b": mix_rows and mix_weights go together"),
        (lambda: composed(logits=None), fn + b": null argument"),
        (lambda: composed(sc=None), fn + b": null argument"),
        (lambda: composed(seeds=None), fn + b": null argument"),
        (lambda: composed(steps=None), fn + b": null argument"),
        (lambda: composed(idx=None, seq=None), fn + b": null argument"),
        (lambda: composed(given=p, seq=None), fn + b": given tokens are indexed as out_seq and need it"),
        (lambda: composed(given=p, stride=0), fn + b": given tokens are indexed as out_seq and need it"),
        (lambda: composed(lp=ctypes.byref(_lib.Logprobs(1 << 20, 0, 0, 0, 0)), seq=None), fn + b": logprobs are indexed as out_seq"),
        (lambda: composed(lp=ctypes.byref(_lib.Logprobs(1 << 20, 0, 1 << 20, 1 << 20, 21))), fn + b": top_n=21 outside [0, 20]"),
        (lambda: composed(rd=7), b"unsupported round dtype 7"),
        (lambda: composed(V=1 << 20, rows=2), b"too large for the shared-memory row stage"),
        (lambda: composed(mix=None, w=None, rd=7), b"unsupported round dtype 7"),
    ]:
        assert call() < 0, msg
        assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
