"""CPU: speculative Jacobi decoding in serve.LLM (sjd_window=L) with the device calls stubbed: a stub pass advances every started slot
by a random 1..L tokens. Depths and finishing one step after the pass that completed a request, slot reuse, joins that write the seed
and guidance before the slot starts, c2i twins, the drain on a top_k / max_tokens change, the ValueErrors, and the argument checks of
the per-slot SJD entries through the C-ABI without a GPU."""
import ctypes
import random

import pytest
import torch

from llamagen_b200 import serve
from test_serve_guidance import _add, _model

SP = serve.SamplingParams


class _Device:
    """Stand-ins for the device calls of an SJD LLM. The device state is a list of final counts per slot; a pass advances every started,
    unfinished slot by 1..L and records the counts after it (what the pinned copy would hold)."""

    def __init__(self, monkeypatch, llm, seed=0):
        self.llm, self.rng = llm, random.Random(seed)
        self.events = []           # ("join" | "start" | "pass", step, slot or None)
        self.after = []            # final counts after every pass
        self.nfin = [10 ** 9] * llm.max_num_seqs
        self.passes = {}           # request id -> passes of its slot so far
        self.owners = {}           # (step, slot) -> request id of the join at that step into that slot
        monkeypatch.setattr(serve.LLM, "_device_sjd_reset", lambda llm, st: None)
        monkeypatch.setattr(serve.LLM, "_device_join_prefix", lambda llm, st, params, slot, P: self.join(llm, st, slot, P))
        monkeypatch.setattr(serve.LLM, "_device_join_t2i", lambda llm, st, params, slot: self.join(llm, st, slot, 0))
        monkeypatch.setattr(serve.LLM, "_device_sjd_start", lambda llm, st, slot, req: self.start(llm, st, slot, req))
        monkeypatch.setattr(serve.LLM, "_device_sjd_pass", lambda llm, st, params, dbg=None: self.run(llm, st))
        monkeypatch.setattr(serve.LLM, "_sjd_nfin", lambda llm, st, p: list(self.after[p]))
        monkeypatch.setattr(serve.LLM, "_sjd_rows", lambda llm, st, done, p: st["out"][done].tolist())

    def join(self, llm, st, slot, P):
        assert P == 0
        self.events.append(("join", llm.steps_run, slot))
        self.owners[(llm.steps_run, slot)] = llm._slots[slot].request_id
        st["out"][slot, 0] = 1000 + int(llm._slots[slot].request_id)

    def start(self, llm, st, slot, req):
        assert self.events[-1] == ("join", llm.steps_run, slot)            # token 0 is drawn before the start
        assert req is llm._slots[slot]
        p = req.params                                                     # the join wrote the request's seed and guidance
        assert int(st["seeds"][slot]) == (llm._seed + int(req.request_id) if p.seed is None else p.seed)
        if "cfg" in st:
            assert float(st["cfg"][slot]) == (llm.cfg_scale if p.cfg_scale is None else p.cfg_scale)
            assert int(st["interval"][slot]) == (-1 if p.cfg_interval is None else p.cfg_interval)
        self.events.append(("start", llm.steps_run, slot))
        self.nfin[slot] = 1
        self.passes[req.request_id] = 0

    def run(self, llm, st):
        S, L = st["S"], st["L"]
        assert L == min(llm.sjd_window, S - 1)
        self.events.append(("pass", llm.steps_run, None))
        for b, req in enumerate(llm._slots):
            if self.nfin[b] < S:
                n = min(S, self.nfin[b] + self.rng.randint(1, L))
                st["out"][b, self.nfin[b]:n] = int(req.request_id)
                self.nfin[b] = n
                self.passes[req.request_id] += 1
        self.after.append(list(self.nfin))


def _drive(llm):
    """Run to the end; returns ({request id: (step of its output, tokens)}, steps)."""
    outs = {}
    while llm.has_unfinished_requests():
        step = llm.steps_run
        for o in llm.step():
            outs[o.request_id] = (step, o.outputs[0].token_ids)
    return outs


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("L", [2, 5, 64])
def test_requests_finish_one_step_after_their_last_pass_and_slots_are_reused(monkeypatch, kind, L):
    S = 9
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=3, seed=100, sjd_window=L)
    dev = _Device(monkeypatch, llm, seed=L)
    sps = [SP(top_k=10, max_tokens=S, cfg_scale=c, cfg_interval=k, seed=s)
           for c, k, s in [(1.0, None, None), (7.5, 3, 12345), (None, 0, None), (2.0, None, 5), (0.5, 5, 7), (4.0, -1, None), (7.5, None, 0)]]
    for i, sp in enumerate(sps[:5]):
        _add(llm, i, sp)
    llm.step()
    for i, sp in enumerate(sps[5:], start=5):
        _add(llm, i, sp)
    outs = _drive(llm)
    assert sorted(outs, key=int) == [str(i) for i in range(7)]
    for rid, (step, toks) in outs.items():
        assert len(toks) == S and toks[0] == 1000 + int(rid) and toks[1:] == [int(rid)] * (S - 1)
        # the request's start, its passes, and its output one step after the pass that completed it
        start = next(s for (s, _), r in dev.owners.items() if r == rid)
        assert step == start + llm.sjd_request_passes[rid]
        assert llm.sjd_request_passes[rid] == dev.passes[rid] and 1 <= dev.passes[rid] <= S - 1
    # three slots, seven requests: every slot is reused, and a slot freed in a step takes a waiting request in the next one
    starts = [(s, b) for e, s, b in dev.events if e == "start"]
    assert len(starts) == 7 and {b for _, b in starts} == {0, 1, 2}
    for b in range(3):
        mine = sorted(s for s, bb in starts if bb == b)
        ends = sorted(outs[dev.owners[(s, b)]][0] for s in mine)
        for nxt, end in zip(mine[1:], ends[:-1]):
            assert nxt == end + 1
    assert llm.sjd_passes == sum(1 for e, _, _ in dev.events if e == "pass") and llm.sjd_tokens == 7 * (S - 1)
    assert llm.steps_run == llm.sjd_passes


def test_one_step_per_pass_and_the_lag_of_one_pass(monkeypatch):
    """One slot, L = S - 1 (every pass completes the request it starts): a request takes two steps, its pass and the read."""
    S = 5
    llm = serve.LLM(_model("t2i"), cfg_scale=1.0, max_num_seqs=1, seed=0, sjd_window=64)
    dev = _Device(monkeypatch, llm)
    dev.rng.randint = lambda a, b: b
    for i in range(3):
        _add(llm, i, SP(max_tokens=S))
    outs = _drive(llm)
    assert {r: s for r, (s, _) in outs.items()} == {"0": 1, "1": 3, "2": 5}
    assert [e for e, _, _ in dev.events] == ["join", "start", "pass", "pass"] * 3
    assert llm.sjd_request_passes == {"0": 1, "1": 1, "2": 1} and llm.sjd_passes == 6


def test_c2i_twins_mirror_their_request(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=2, seed=0, sjd_window=4)
    _Device(monkeypatch, llm)
    sp = [SP(max_tokens=6, cfg_scale=7.5, cfg_interval=0, seed=31), SP(max_tokens=6, cfg_scale=1.0)]
    outs = llm.generate(prompt_token_ids=[[3], [4], [10], [10]], sampling_params=sp + sp)
    assert [o.request_id for o in outs] == ["0", "1", "2", "3"]
    assert outs[2].outputs[0].token_ids == outs[0].outputs[0].token_ids and outs[3].outputs[0].token_ids == outs[1].outputs[0].token_ids
    assert outs[2].prompt_token_ids == [10] and sorted(llm.sjd_request_passes) == ["0", "1"]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_top_k_or_max_tokens_change_still_drains(monkeypatch, kind):
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=2, seed=0, sjd_window=3)
    dev = _Device(monkeypatch, llm)
    a, b, c = SP(top_k=10, max_tokens=4, seed=1), SP(top_k=20, max_tokens=4, seed=1), SP(top_k=10, max_tokens=7)
    for i, sp in enumerate([a, b, a, c]):
        _add(llm, i, sp)
    outs = _drive(llm)
    starts = [s for e, s, _ in dev.events if e == "start"]
    # every request differs from the one before it: it joins the step after the previous one's output
    assert starts[0] == 0 and [starts[i + 1] for i in range(3)] == [outs[str(i)][0] + 1 for i in range(3)]
    assert len(outs["3"][1]) == 7


def test_value_errors():
    f = torch.randn(3, 4)
    for bad in (1, 65, 0, -2, 4.0, 2.5, "8", True, None.__class__):
        with pytest.raises(ValueError, match="sjd_window"):
            serve.LLM(_model("c2i"), sjd_window=bad)
    for kind in ("c2i", "t2i"):
        llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=2, sjd_window=8)
        with pytest.raises(ValueError, match="prefix cannot be combined with sjd_window"):
            _add(llm, 0, SP(max_tokens=8), prefix=[1, 2])
        with pytest.raises(ValueError, match="prefix cannot be combined with sjd_window"):
            if kind == "t2i":
                llm.generate(prompt_embeds=[f], sampling_params=SP(max_tokens=8), prefixes=[[1]])
            else:
                llm.generate(prompt_token_ids=[[1], [1000]], sampling_params=SP(max_tokens=8), prefixes=[[1]])
        for S in (1, 2):
            with pytest.raises(ValueError, match="max_tokens >= 3"):
                _add(llm, 0, SP(max_tokens=S))
        assert llm.get_num_unfinished_requests() == 0
        _add(llm, 0, SP(max_tokens=3))                                   # the smallest accepted: window 2
    # without sjd_window nothing changes: short requests and prefixes are accepted
    plain = serve.LLM(_model("c2i"), max_num_seqs=2)
    plain.add_request([1], SP(max_tokens=2), prefix=[1])
    assert plain.sjd_window is None and plain.sjd_passes == 0


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_sjd_slot_entries_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no call below reaches a launch
    sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 0, 0)
    nbytes = ctypes.c_size_t()

    def start(e=None, slot=0, B=2, L=4, S=16, cfg=4.0, interval=-1, out=p, ws=p):
        return lib.lg_sjd_slot_start(e, slot, B, 1, L, S, 5, cfg, interval, out, ws, 1 << 30, None)

    def pas(e=None, sc=ctypes.byref(sc), em=p, nm=p, B=2, cfg=1, S=16, L=4, ws=p, out=p, nfin=p):
        return lib.lg_sjd_pass_slots(e, sc, em, nm, B, cfg, S, L, ws, 1 << 30, out, nfin, None, None)

    for rc_call, msg in [
        (lambda: lib.lg_sjd_slots_workspace_bytes(None, 2, 1, 4, ctypes.byref(nbytes)), b"lg_sjd_slots_workspace_bytes: bad argument"),
        (lambda: lib.lg_sjd_slots_reset(None, 2, 1, 1, p, 1 << 30, None), b"lg_sjd_slots_reset: window L=1 outside [2, 64]"),
        (lambda: lib.lg_sjd_slots_reset(None, 0, 1, 4, p, 1 << 30, None), b"lg_sjd_slots_reset: B=0"),
        (lambda: lib.lg_sjd_slots_reset(None, 2, 1, 4, ctypes.c_void_p(1 << 20 | 16), 1 << 30, None), b"256-byte aligned"),
        (lambda: lib.lg_sjd_slots_reset(None, 2, 1, 4, p, 1 << 30, None), b"lg_sjd_slots_reset: engine not finalized"),
        (lambda: start(out=None), b"lg_sjd_slot_start: null out_tokens"),
        (lambda: start(slot=2), b"lg_sjd_slot_start: slot 2 outside [0, B=2)"),
        (lambda: start(slot=-1), b"slot -1 outside"),
        (lambda: start(cfg=float("nan")), b"must be finite"),
        (lambda: start(interval=-2), b"cfg_interval -2 >= -1"),
        (lambda: start(L=65), b"lg_sjd_slot_start: window L=65 outside [2, 64]"),
        (lambda: start(S=4), b"lg_sjd_slot_start: S=4 must exceed the window L=4"),
        (lambda: start(ws=None), b"lg_sjd_slot_start: scratch must be non-null"),
        (lambda: start(), b"lg_sjd_slot_start: engine not finalized"),
        (lambda: pas(sc=None), b"lg_sjd_pass_slots: null argument"),
        (lambda: pas(out=None), b"lg_sjd_pass_slots: null argument"),
        (lambda: pas(nfin=None), b"lg_sjd_pass_slots: null argument"),
        (lambda: pas(cfg=0), b"lg_sjd_pass_slots: neg_mask masks the unconditional CFG rows and needs use_cfg"),
        (lambda: pas(em=None), b"lg_sjd_pass_slots: neg_mask needs emb_mask"),
        (lambda: pas(L=1), b"lg_sjd_pass_slots: window L=1 outside [2, 64]"),
        (lambda: pas(S=3), b"lg_sjd_pass_slots: S=3 must exceed the window L=4"),
        (lambda: pas(B=0), b"lg_sjd_pass_slots: B=0"),
        (lambda: pas(), b"lg_sjd_pass_slots: engine not finalized"),
        (lambda: lib.lg_test_sjd_slots(2, 16, 4, 8, 0, *([p] * 11), None, None), b"lg_test_sjd_slots: null argument"),
        (lambda: lib.lg_test_sjd_slots(2, 4, 4, 8, 0, *([p] * 12), None), b"lg_test_sjd_slots: bad shape"),
    ]:
        assert rc_call() < 0, msg
        assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
