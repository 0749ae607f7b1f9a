"""CPU: image-completion requests in serve.LLM with the device calls stubbed (the join of a request that brings its first P image
tokens, c2i and t2i: its slot, prefix, P and seed, out[:P] == prefix, depths and step counts, slot reuse, a join that draws the last
token, CFG twins, the ValueErrors), and the argument checks of lg_prefill_slot_prefix / lg_slot_prefix_workspace_bytes through the
C-ABI without a GPU."""
import ctypes
import types

import numpy as np
import pytest
import torch

from llamagen_b200 import serve
from test_serve_t2i import _TINY, _engine

T, C, V = 6, 4, 64


def _model(model_type):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=V,
                                 cls_token_num=T if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None)


class _Device:
    """Stand-ins for the device calls. Every draw writes one out index, which the stub asserts lies in [0, max_tokens).
    * A completion join records what it was given and draws token P = prefix[-1] + 1.
    * c2i: a decode draws input + 1 at index pos[slot] for every slot (a plain request's input at position 0 is its class id).
    * t2i: a caption join draws token 0 = 10 * (valid caption tokens); a decode checks that every running slot sits at position
      T + step - 1 and draws input + 1 at index step[slot]."""

    def __init__(self, monkeypatch):
        self.joins, self.decodes = [], 0
        monkeypatch.setattr(serve.LLM, "_device_join_prefix", lambda llm, *a: self.join_prefix(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_step", lambda llm, *a: self.decode_c2i(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_join_t2i", lambda llm, *a: self.join_t2i(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_decode_t2i", lambda llm, *a: self.decode_t2i(llm, *a))

    @staticmethod
    def _write(st, slot, k, tok):
        assert 0 <= k < st["S"], (slot, k, st["S"])
        st["out"][slot, k] = tok
        st["tok"][slot] = tok

    def join_prefix(self, llm, st, params, slot, P):
        assert 1 <= P <= st["S"] - 1
        pf = st["out"][slot, :P].clone()
        self.joins.append(dict(slot=slot, P=P, prefix=pf.tolist(), seed=int(st["seeds"][slot]), step=llm.steps_run,
                               cls=None if llm.t2i else int(st["tok"][slot]), cond=st["cond"][slot].clone() if llm.t2i else None))
        self._write(st, slot, P, int(pf[-1]) + 1)

    def decode_c2i(self, llm, st, params):
        self.decodes += 1
        nxt = st["tok"] + 1
        for b in range(llm.max_num_seqs):
            self._write(st, b, int(st["pos"][b]), int(nxt[b]))

    def join_t2i(self, llm, st, params, slot):
        self.joins.append(dict(slot=slot, P=0, seed=int(st["seeds"][slot]), step=llm.steps_run))
        self._write(st, slot, 0, 10 * int(st["mask"][slot].sum()))

    def decode_t2i(self, llm, st, params):
        self.decodes += 1
        B, R = llm.max_num_seqs, st["R"]
        for b in range(B):
            if llm._slots[b] is not None:
                assert int(st["pos"][b]) == T + int(st["step"][b]) - 1 and int(st["active"][b]) == 1
                if R == 2 * B:
                    assert int(st["pos"][B + b]) == int(st["pos"][b]) and int(st["active"][B + b]) == 1
        nxt = st["tok"] + 1
        for b in range(B):
            self._write(st, b, int(st["step"][b]), int(nxt[b]))


def _feats(n, seed):
    return torch.randn(n, C, generator=torch.Generator().manual_seed(seed))


def _tokens(outs):
    return {o.request_id: o.outputs[0].token_ids for o in outs}


@pytest.mark.parametrize("cfg", [1.0, 4.0])
def test_c2i_completion_joins_mid_sequence_and_reuses_its_slot(monkeypatch, cfg):
    dev = _Device(monkeypatch)
    sp = serve.SamplingParams(top_k=10, max_tokens=6)
    llm = serve.LLM(_model("c2i"), cfg_scale=cfg, max_num_seqs=3, seed=100)
    llm.add_request([5], sp)
    llm.add_request([6], sp)
    outs = llm.step()                                       # r0, r1 draw token 0 in the decode
    assert outs == [] and llm._depth[:2] == [1, 1]
    llm.add_request([7], sp, prefix=[30, 31, 32])           # a list
    outs += llm.step()                                      # r2 joins slot 2 and draws token 3; the decode draws its token 4
    assert llm._depth == [2, 2, 5]
    st, B = llm._state, 3
    rows = [2, B + 2] if cfg > 1 else [2]
    assert st["pos"][rows].tolist() == [1 + 3 + 1] * len(rows) and st["active"][rows].tolist() == [1] * len(rows)
    outs += llm.step()                                      # r2 finishes; slot 2 is free
    assert [o.request_id for o in outs] == ["2"]
    llm.add_request([8], sp, prefix=np.array([50, 51], dtype=np.int32))
    while llm.has_unfinished_requests():
        outs += llm.step()
    # r3 joins slot 2 at step 3 (rows at 1 + 2, token 2 from the join), finishes at step 5 with r0, r1 done at step 5 too
    assert [(j["slot"], j["P"], j["prefix"], j["seed"], j["step"], j["cls"]) for j in dev.joins] == [
        (2, 3, [30, 31, 32], 102, 1, 7), (2, 2, [50, 51], 103, 3, 8)]
    assert llm.steps_run == dev.decodes == 6
    assert _tokens(outs) == {"0": [6, 7, 8, 9, 10, 11], "1": [7, 8, 9, 10, 11, 12], "2": [30, 31, 32, 33, 34, 35],
                             "3": [50, 51, 52, 53, 54, 55]}
    assert not llm.has_unfinished_requests() and llm.get_num_unfinished_requests() == 0


@pytest.mark.parametrize("cfg", [1.0, 4.0])
def test_t2i_completion_joins_mid_sequence_and_reuses_its_slot(monkeypatch, cfg):
    dev = _Device(monkeypatch)
    sp = serve.SamplingParams(top_k=10, max_tokens=5)
    llm = serve.LLM(_model("t2i"), cfg_scale=cfg, max_num_seqs=2, seed=40)
    llm.add_request(prompt_embeds=_feats(2, 0), sampling_params=sp)
    outs = llm.step()                                       # r0 joins, token 0 from its join
    llm.add_request(prompt_embeds=_feats(3, 1), sampling_params=sp, prefix=torch.tensor([7, 8], dtype=torch.int16))
    outs += llm.step()                                      # r0 decodes token 1, then r1 joins slot 1 and draws token 2
    st, B = llm._state, 2
    assert llm._depth == [2, 3] and st["step"].tolist() == [2, 3]
    rows = [1, B + 1] if cfg > 1 else [1]
    assert st["pos"][rows].tolist() == [T + 2] * len(rows)
    llm.add_request(prompt_embeds=_feats(4, 2), sampling_params=sp, prefix=[1, 2, 3])
    while llm.has_unfinished_requests():
        outs += llm.step()
    # r1 finishes at step 3; r2 joins slot 1 (still holding r1's rows) at step 4, when r0 finishes, and finishes at step 5
    assert [(j["slot"], j["P"], j["seed"], j["step"]) for j in dev.joins] == [(0, 0, 40, 0), (1, 2, 41, 1), (1, 3, 42, 4)]
    assert [j["prefix"] for j in dev.joins[1:]] == [[7, 8], [1, 2, 3]]
    c, _ = serve.LLM(_model("t2i"))._caption(_feats(4, 2))
    assert torch.equal(dev.joins[2]["cond"], c)
    assert llm.steps_run == 6
    assert _tokens(outs) == {"0": [20, 21, 22, 23, 24], "1": [7, 8, 9, 10, 11], "2": [1, 2, 3, 4, 5]}
    assert all(o.prompt_token_ids == [] for o in outs)


def test_c2i_join_that_draws_the_last_token_finishes_at_its_join(monkeypatch):
    dev = _Device(monkeypatch)
    sp = serve.SamplingParams(max_tokens=4)
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2, seed=0)
    llm.add_request([3], sp)
    llm.step()
    llm.add_request([4], sp, prefix=[10, 11, 12])           # P = max_tokens - 1
    outs = llm.step()                                       # the join draws token 3: r1 is done before the decode
    assert _tokens(outs) == {"1": [10, 11, 12, 13]} and llm._slots[1] is None
    st = llm._state
    assert st["active"].tolist() == [1, 0, 1, 0] and st["pos"][[1, 3]].tolist() == [0, 0] and int(st["tok"][1]) == 0
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert llm.steps_run == dev.decodes == 4
    llm.add_request([5], sp, prefix=[20, 21, 22])           # alone: finishes at its join, and no decode runs
    outs += llm.step()
    assert _tokens(outs) == {"0": [4, 5, 6, 7], "1": [10, 11, 12, 13], "2": [20, 21, 22, 23]}
    assert llm.steps_run == 5 and dev.decodes == 4 and not llm.has_unfinished_requests()


def test_t2i_join_that_draws_the_last_token_finishes_at_its_join(monkeypatch):
    dev = _Device(monkeypatch)
    sp = serve.SamplingParams(max_tokens=3)
    llm = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=2, seed=0)
    llm.add_request(prompt_embeds=_feats(1, 0), sampling_params=sp)
    llm.add_request(prompt_embeds=_feats(1, 1), sampling_params=sp, prefix=[5, 6])
    outs = llm.step()
    assert _tokens(outs) == {"1": [5, 6, 7]} and llm._slots[1] is None
    assert llm._state["step"].tolist() == [1, 0] and llm._state["active"].tolist() == [1, 0, 1, 0]
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert _tokens(outs) == {"0": [10, 11, 12], "1": [5, 6, 7]} and dev.decodes == 2


def test_c2i_cfg_twins_mirror_the_prefix(monkeypatch):
    _Device(monkeypatch)
    sp = serve.SamplingParams(max_tokens=4)
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2, seed=0)
    outs = llm.generate(prompt_token_ids=[[3], [4], [1000], [1000]], sampling_params=sp, prefixes=[[40, 41], None])
    got = [o.outputs[0].token_ids for o in outs]
    assert got == [[40, 41, 42, 43], [5, 6, 7, 8], [40, 41, 42, 43], [5, 6, 7, 8]]
    # add_request: a twin without a prefix takes its conditional request's, the same prefix is accepted, another one is not
    rid = llm.add_request([3], sp, prefix=[1, 2])
    llm.add_request([1000], sp, twin_of=rid, prefix=torch.tensor([1, 2]))
    assert torch.equal(llm._twins[rid].prefix, torch.tensor([1, 2]))
    rid2 = llm.add_request([5], sp)
    for twin_prefix in ([1, 3], [1, 2, 3]):
        with pytest.raises(ValueError, match="mirrors the prefix"):
            llm.add_request([1000], sp, twin_of=rid, prefix=twin_prefix)
    with pytest.raises(ValueError, match="mirrors the prefix"):
        llm.add_request([1000], sp, twin_of=rid2, prefix=[1, 2])
    assert llm.get_num_unfinished_requests() == 3


def test_value_errors_leave_nothing_queued():
    sp = serve.SamplingParams(max_tokens=4)
    c2i = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=2)
    t2i = serve.LLM(_model("t2i"), cfg_scale=1.0, max_num_seqs=2)
    f = _feats(2, 0)
    bad_prefixes = [
        [1.0, 2.0],                                          # non-integer dtype
        torch.tensor([1.0, 2.0]),
        np.array([True, False]),
        torch.tensor([[1, 2]]),                              # 2-D
        np.zeros((2, 1), np.int64),
        7,                                                   # 0-D
        [1, V],                                              # ids outside [0, V)
        [-1, 2],
        torch.zeros(0, dtype=torch.long),                    # P = 0
        [1, 2, 3, 4],                                        # P = max_tokens
        list(range(9)),
    ]
    for pf in bad_prefixes:
        for call in (lambda: c2i.add_request([3], sp, prefix=pf),
                     lambda: t2i.add_request(prompt_embeds=f, sampling_params=sp, prefix=pf),
                     lambda: c2i.generate(prompt_token_ids=[[3], [4], [1000], [1000]], sampling_params=sp, prefixes=[[1], pf]),
                     lambda: t2i.generate(prompt_embeds=[f, f], sampling_params=sp, prefixes=[[1], pf])):
            with pytest.raises(ValueError):
                call()
    for call in (lambda: c2i.generate(prompt_token_ids=[[3], [4], [1000], [1000]], sampling_params=sp, prefixes=[[1]]),
                 lambda: c2i.generate(prompt_token_ids=[[3], [4], [1000], [1000]], sampling_params=sp, prefixes=[[1], [2], [1], [2]]),
                 lambda: t2i.generate(prompt_embeds=[f, f], sampling_params=sp, prefixes=[[1]]),
                 lambda: t2i.generate(prompt_embeds=[f], sampling_params=sp, prefixes=[[1], [2]])):
        with pytest.raises(ValueError, match="prefixes holds"):
            call()
    assert c2i.get_num_unfinished_requests() == 0 and t2i.get_num_unfinished_requests() == 0
    assert next(c2i.request_counter) == 0 and next(t2i.request_counter) == 0      # no request id was taken


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_prefill_slot_prefix_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no check below lets a call reach a launch
    Tc, blk = _TINY["cls_token_num"], _TINY["block_size"]
    c2i = _engine(lib, _lib, _lib.LG_MODEL_C2I)
    bare = _engine(lib, _lib, _lib.LG_MODEL_T2I)
    ready = _engine(lib, _lib, _lib.LG_MODEL_T2I, bind=True)        # 2 rows, max_seq Tc + 8
    try:
        def ws_bytes(e, use_cfg, P):
            n = ctypes.c_size_t()
            rc = lib.lg_slot_prefix_workspace_bytes(e, use_cfg, P, ctypes.byref(n))
            return n.value if rc == 0 else None

        # P = 0 is lg_slot_workspace_bytes' size; the size grows with P; c2i engines have one too
        for use_cfg in (0, 1):
            n0 = ctypes.c_size_t()
            assert lib.lg_slot_workspace_bytes(ready, use_cfg, ctypes.byref(n0)) == 0
            assert ws_bytes(ready, use_cfg, 0) == n0.value
            assert n0.value < ws_bytes(ready, use_cfg, 4) < ws_bytes(ready, use_cfg, blk - 1)
        assert ws_bytes(ready, 0, 4) < ws_bytes(ready, 1, 4) and ws_bytes(c2i, 1, 4) > 0
        for e, P, msg in [(ready, -1, b"outside [0, block_size - 1 = 15]"), (ready, blk, b"outside [0, block_size - 1 = 15]"),
                          (None, 0, b"null argument")]:
            assert ws_bytes(e, 1, P) is None and msg in lib.lg_last_error(), msg
        assert lib.lg_slot_prefix_workspace_bytes(ready, 1, 0, None) < 0

        two4 = ws_bytes(ready, 1, 4)

        def prefill(e, cond=p, mask=p, T=Tc, prefix=p, P=4, slot=0, B=1, use_cfg=1, ws=p, nbytes=two4, logits=p):
            return lib.lg_prefill_slot_prefix(e, cond, mask, T, prefix, P, slot, B, use_cfg, ws, nbytes, logits, None)

        for rc_call, msg in [
            (lambda: prefill(None), b"lg_prefill_slot_prefix: null engine"),
            (lambda: prefill(ready, cond=None), b"null cond or logits_out"),
            (lambda: prefill(ready, logits=None), b"null cond or logits_out"),
            (lambda: prefill(ready, T=Tc - 1), b"must equal cls_token_num"),
            (lambda: prefill(ready, prefix=None), b"null prefix with P=4"),
            (lambda: prefill(ready, P=-1), b"prefix length P=-1 outside [0, block_size - 1 = 15]"),
            (lambda: prefill(ready, P=blk), b"prefix length P=16 outside [0, block_size - 1 = 15]"),
            (lambda: prefill(ready, slot=-1), b"outside [0, B=1)"),
            (lambda: prefill(ready, slot=1, B=1), b"outside [0, B=1)"),
            (lambda: prefill(ready, B=0), b"outside"),
            (lambda: prefill(c2i), b"emb_mask only applies to t2i models"),
            (lambda: prefill(c2i, mask=None), b"not finalized"),
            (lambda: prefill(ready, ws=ctypes.c_void_p((1 << 20) + 128)), b"256-byte aligned"),
            (lambda: prefill(ready, ws=None), b"256-byte aligned"),
            (lambda: prefill(bare), b"not finalized"),
            (lambda: prefill(ready, slot=1, B=2), b"rows 4 exceed workspace rows 2"),       # nh * B = 4 rows, the workspace has 2
            (lambda: prefill(ready, P=9), b"sequence 17 exceeds workspace max_seq 16"),     # T + P outgrows the cache
            (lambda: prefill(ready, nbytes=two4 - 1), b"too small"),
            (lambda: prefill(ready, use_cfg=0, nbytes=ws_bytes(ready, 0, 4) - 256), b"too small"),
            (lambda: prefill(ready, P=6, nbytes=two4), b"too small"),                       # a longer prefix needs more scratch
        ]:
            assert rc_call() < 0, msg
            assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
        # lg_prefill_slot is the P = 0 case: a prefix pointer is neither needed nor checked there
        assert lib.lg_prefill_slot(ready, p, p, Tc, 0, 1, 1, p, two4, None, None) < 0
        assert b"lg_prefill_slot: null cond or logits_out" in lib.lg_last_error()
    finally:
        for h in (c2i, bare, ready):
            lib.lg_engine_destroy(h)
