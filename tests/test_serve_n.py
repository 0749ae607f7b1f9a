"""CPU: parallel sampling in serve.LLM (SamplingParams(n=k)) with the device calls stubbed: one prefill and one fan-out per t2i, prefix or
SJD request (none for a plain c2i request), every slot's image index, seed and guidance before its first draw, admission that waits for
k free slots without being overtaken, outputs ordered by index, staggered SJD finishes, null-class twins, the ValueErrors, and the
argument checks of lg_sample_rows_keyed, lg_sjd_slot_start_image and lg_copy_slot_kv through the C-ABI without a GPU."""
import ctypes
import random

import numpy as np
import pytest
import torch

from llamagen_b200 import serve
from test_serve_guidance import _add, _feats, _model

SP = serve.SamplingParams


class _Device:
    """Stand-ins for the device calls of a plain or SJD LLM. Every draw checks that the slots it draws for hold their request's seed,
    guidance and image index; a slot's tokens are 1000 * (request id + 1) + 100 * image + token index, so outputs show where they came
    from. Under SJD a pass advances every started, unfinished slot by a random 1..L tokens."""

    def __init__(self, monkeypatch, llm, seed=0):
        self.llm, self.rng = llm, random.Random(seed)
        self.events = []               # (kind, step, detail)
        self.drawn = set()             # slots that have drawn since their join
        self.nfin, self.after = [10 ** 9] * llm.max_num_seqs, []
        for name, fn in [("_device_join_t2i", lambda llm, st, params, slot: self.prefill(st, slot, 0)),
                         ("_device_join_prefix", lambda llm, st, params, slot, P: self.prefill(st, slot, P)),
                         ("_device_copy_kv", lambda llm, st, src, dsts, length: self.events.append(("copy", llm.steps_run,
                                                                                                   (src, list(dsts), length)))),
                         ("_device_join_draws", lambda llm, st, params, slots, P: [self.draw(st, s, P, "join_draw") for s in slots]),
                         ("_device_step", lambda llm, st, params: self.decode(st)),
                         ("_device_decode_t2i", lambda llm, st, params: self.decode(st)),
                         ("_device_sjd_reset", lambda llm, st: None),
                         ("_device_sjd_start", lambda llm, st, slot, req: self.start(st, slot, req)),
                         ("_device_sjd_pass", lambda llm, st, params, dbg=None: self.sjd_pass(st)),
                         ("_sjd_nfin", lambda llm, st, p: list(self.after[p])),
                         ("_sjd_rows", lambda llm, st, done, p: st["out"][done].tolist())]:
            monkeypatch.setattr(serve.LLM, name, fn)

    def check(self, st, slot):
        llm = self.llm
        req = llm._slots[slot]
        j = llm._img[slot]
        assert 0 <= j < req.n and int(st["img"][slot]) == j and int(st["seeds"][slot]) == req.seed, (slot, req.request_id)
        if "cfg" in st:
            assert float(st["cfg"][slot]) == req.cfg and int(st["interval"][slot]) == req.interval
        if llm.t2i:
            assert torch.equal(st["mask"][slot], req.mask.to(st["mask"].dtype))

    def token(self, slot, k):
        return 1000 * (int(self.llm._slots[slot].request_id) + 1) + 100 * self.llm._img[slot] + k

    def draw(self, st, slot, k, kind):
        self.check(st, slot)
        self.events.append((kind, self.llm.steps_run, slot))
        self.drawn.add(slot)
        st["out"][slot, k] = self.token(slot, k)
        st["tok"][slot] = 1

    def prefill(self, st, slot, P):
        self.events.append(("prefill", self.llm.steps_run, (slot, P)))
        self.drawn.discard(slot)
        self.draw(st, slot, P, "join_draw")

    def decode(self, st):
        llm = self.llm
        self.events.append(("decode", llm.steps_run, None))
        k = st["step"] if llm.t2i else st["pos"][:llm.max_num_seqs]
        for b, req in enumerate(llm._slots):
            if req is not None:
                self.check(st, b)
                st["out"][b, int(k[b])] = self.token(b, int(k[b]))

    def start(self, st, slot, req):
        assert req is self.llm._slots[slot] and slot in self.drawn          # token 0 is drawn before the start
        self.check(st, slot)
        self.events.append(("start", self.llm.steps_run, slot))
        self.nfin[slot] = 1

    def sjd_pass(self, st):
        S, L = st["S"], st["L"]
        self.events.append(("pass", self.llm.steps_run, None))
        for b, req in enumerate(self.llm._slots):
            if self.nfin[b] < S:
                n = min(S, self.nfin[b] + self.rng.randint(1, L))
                for k in range(self.nfin[b], n):
                    st["out"][b, k] = self.token(b, k)
                self.nfin[b] = n
        self.after.append(list(self.nfin))


def _drive(llm):
    """Run to the end; returns {request id: (step of its output, RequestOutput)}; every request is returned once."""
    outs = {}
    while llm.has_unfinished_requests():
        step = llm.steps_run
        for o in llm.step():
            assert o.request_id not in outs
            outs[o.request_id] = (step, o)
    return outs


def _expect(rid, n, S, P=0, prefix=None):
    """The token rows the stub makes for request rid's n samples (a prefix's tokens first)."""
    rows = [[1000 * (int(rid) + 1) + 100 * j + k for k in range(S)] for j in range(n)]
    for r in rows:
        r[:P] = [] if prefix is None else list(prefix)
    return rows


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("sjd", [False, True])
def test_one_prefill_and_one_fan_out_per_request(monkeypatch, kind, sjd):
    S = 6
    llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=6, seed=100, sjd_window=4 if sjd else None)
    dev = _Device(monkeypatch, llm)
    pf = None if sjd else [7, 8]
    P = 0 if pf is None else 2
    _add(llm, 0, SP(max_tokens=S, n=1))
    _add(llm, 1, SP(max_tokens=S, n=4, cfg_scale=7.5, cfg_interval=2, seed=9), prefix=pf)
    _add(llm, 2, SP(max_tokens=S, n=1, cfg_scale=2.0))
    outs = _drive(llm)
    T = llm.model.cls_token_num
    prefills = [d for e, _, d in dev.events if e == "prefill"]
    copies = [d for e, _, d in dev.events if e == "copy"]
    # request 1 takes slots 1 .. 4: one prefill into slot 1, one copy of its T + P positions to slots 2, 3, 4
    assert (1, P) in prefills and copies == [(1, [2, 3, 4], T + P)]
    assert sorted(s for e, _, s in dev.events if e == "join_draw" and s in (1, 2, 3, 4)) == [1, 2, 3, 4]
    if kind == "t2i" or sjd:
        assert sorted(s for s, _ in prefills) == [0, 1, 5]
    assert [o.index for o in outs["1"][1].outputs] == [0, 1, 2, 3]
    assert [o.token_ids for o in outs["1"][1].outputs] == _expect("1", 4, S, P, pf)
    assert [o.token_ids for o in outs["0"][1].outputs] == _expect("0", 1, S)
    assert len(outs) == 3


def test_plain_c2i_request_has_no_prefill_and_no_fan_out(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, max_num_seqs=4, seed=1)
    dev = _Device(monkeypatch, llm)
    rid = llm.add_request([3], SP(max_tokens=5, n=3, seed=77))
    outs = _drive(llm)
    assert not [e for e, _, _ in dev.events if e in ("prefill", "copy", "join_draw")]
    assert [o.token_ids for o in outs[rid][1].outputs] == _expect(rid, 3, 5)
    st = llm._state
    assert st["img"][:3].tolist() == [0, 1, 2] and st["seeds"][:3].tolist() == [77] * 3 and st["tok"][:3].tolist() == [0, 0, 0]


def test_waits_for_k_free_slots_and_is_not_overtaken(monkeypatch):
    S = 4
    llm = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=4, seed=1)
    dev = _Device(monkeypatch, llm)
    _add(llm, 0, SP(max_tokens=S))                 # slot 0, joins at step 0
    _add(llm, 1, SP(max_tokens=S))                 # slot 1, step 0
    llm.step()
    _add(llm, 2, SP(max_tokens=S, n=3))            # needs 3 slots: waits until r0 and r1 free theirs
    _add(llm, 3, SP(max_tokens=S))                 # a free slot exists, but r3 may not overtake r2
    outs = _drive(llm)
    prefills = [(s, d[0]) for e, s, d in dev.events if e == "prefill"]
    # r0 and r1 return at step S - 1; at step S r2 joins slots 0, 1, 2 and r3, behind it, slot 3 (slot 2 was free all along)
    assert prefills == [(0, 0), (0, 1), (S, 0), (S, 3)]
    assert [d for e, _, d in dev.events if e == "copy"] == [(0, [1, 2], llm.model.cls_token_num)]
    assert outs["0"][0] == outs["1"][0] == S - 1 and outs["2"][0] == outs["3"][0] == 2 * S - 1
    assert [o.index for o in outs["2"][1].outputs] == [0, 1, 2]


def test_staggered_sjd_finishes_free_slots_early_and_return_once(monkeypatch):
    S, L = 10, 3
    llm = serve.LLM(_model("t2i"), cfg_scale=4.0, max_num_seqs=4, seed=3, sjd_window=L)
    dev = _Device(monkeypatch, llm, seed=5)
    _add(llm, 0, SP(max_tokens=S, n=4, seed=4))
    _add(llm, 1, SP(max_tokens=S))
    freed = []
    outs = {}
    while llm.has_unfinished_requests():
        step = llm.steps_run
        out = llm.step()
        freed.append(sum(r is None for r in llm._slots))
        for o in out:
            assert o.request_id not in outs
            outs[o.request_id] = (step, o)
    first = next(i for i, a in enumerate(dev.after) if any(n >= S for n in a))
    last = next(i for i, a in enumerate(dev.after) if all(n >= S for n in a[:4]))
    assert first < last                                     # the four samples finish at different passes (seed 5)
    # a finished sample frees its slot one step after its pass, while the request still runs; r1 takes the first freed slot
    assert outs["0"][0] == last + 1 and outs["1"][0] > first
    assert [o.token_ids for o in outs["0"][1].outputs] == _expect("0", 4, S)
    assert llm.sjd_request_passes["0"] == last + 1 and llm.sjd_tokens == 5 * (S - 1)


def test_twins_mirror_n_outputs(monkeypatch):
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=6, seed=0)
    _Device(monkeypatch, llm)
    sp = [SP(max_tokens=3, n=2, seed=5), SP(max_tokens=3, n=3)]
    outs = llm.generate(prompt_token_ids=[[3], [4], [10], [10]], sampling_params=sp + sp)
    assert [o.request_id for o in outs] == ["0", "1", "2", "3"]
    for r, t in ((0, 2), (1, 3)):
        assert [(c.index, c.token_ids) for c in outs[t].outputs] == [(c.index, c.token_ids) for c in outs[r].outputs]
        assert len(outs[r].outputs) == sp[r].n and outs[t].prompt_token_ids == [10]
    llm = serve.LLM(_model("c2i"), cfg_scale=4.0, num_classes=10, max_num_seqs=4, seed=0)
    rid = llm.add_request([3], SP(max_tokens=3, n=2))
    with pytest.raises(ValueError, match="twin"):
        llm.add_request([10], SP(max_tokens=3, n=3), twin_of=rid)


def test_value_errors():
    f = _feats(3, 0)
    for kind in ("c2i", "t2i"):
        llm = serve.LLM(_model(kind), cfg_scale=4.0, max_num_seqs=4)
        for n in (0, -1, 5, 2.0, 1.5, "2", True, False, None, np.float32(2)):
            sp = SP(max_tokens=4, n=n)
            with pytest.raises(ValueError, match="SamplingParams.n"):
                _add(llm, 0, sp)
            with pytest.raises(ValueError, match="SamplingParams.n"):
                if kind == "t2i":
                    llm.generate(prompt_embeds=[f, f], sampling_params=[SP(max_tokens=4), sp])
                else:
                    llm.generate(prompt_token_ids=[[1], [2]], sampling_params=[SP(max_tokens=4), sp])
        assert llm.get_num_unfinished_requests() == 0
        _add(llm, 0, SP(max_tokens=4, n=np.int64(4)))                    # accepted: numpy integers, n = max_num_seqs
        _add(llm, 1, SP(max_tokens=4, n=1))
        assert [r.n for r in llm._waiting] == [4, 1] and llm.get_num_unfinished_requests() == 2


def test_positional_sampling_params_keep_their_meaning():
    sp = SP(0.0, 0.9, 50, 16, 2.0, 3, 7)
    assert (sp.temperature, sp.top_p, sp.top_k, sp.max_tokens, sp.cfg_scale, sp.cfg_interval, sp.seed, sp.n) == (0.0, 0.9, 50, 16, 2.0, 3,
                                                                                                                  7, 1)


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_new_entry_points_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no call below reaches a launch
    sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 0, 0)

    def keyed(logits=p, B=1, mix=1, sc=ctypes.byref(sc), seeds=p, steps=p, cfg=p, interval=p, img=p, idx=p, seq=p):
        return lib.lg_sample_rows_keyed(logits, B, 64, mix, _lib.LG_DTYPE_F32, sc, seeds, steps, cfg, interval, img, idx, seq, 1, None)

    def start(slot=0, B=2, L=4, S=16, image=1, out=p, ws=p):
        return lib.lg_sjd_slot_start_image(None, slot, B, 1, L, S, 5, 4.0, -1, image, out, ws, 1 << 30, None)

    def copy(src=0, dst=(1, 2), n=None, B=4, cfg=1, length=8):
        arr = (ctypes.c_int32 * max(1, len(dst)))(*dst)
        return lib.lg_copy_slot_kv(None, src, arr if dst else None, len(dst) if n is None else n, B, cfg, length, None)

    for rc_call, msg in [
        (lambda: keyed(logits=None), b"lg_sample_rows_keyed: null argument"),
        (lambda: keyed(seeds=None), b"lg_sample_rows_keyed: null argument"),
        (lambda: keyed(steps=None), b"lg_sample_rows_keyed: null argument"),
        (lambda: keyed(idx=None, seq=None), b"lg_sample_rows_keyed: null argument"),
        (lambda: keyed(mix=0), b"lg_sample_rows_keyed: per-row cfg_rows / interval_rows need mix_cfg"),
        (lambda: keyed(B=0, mix=0, cfg=None, interval=None), b"bad shape B=0"),
        (lambda: start(out=None), b"lg_sjd_slot_start_image: null out_tokens"),
        (lambda: start(slot=2), b"lg_sjd_slot_start_image: slot 2 outside [0, B=2)"),
        (lambda: start(image=-1), b"lg_sjd_slot_start_image: image -1 outside"),
        (lambda: start(L=1), b"lg_sjd_slot_start_image: window L=1 outside [2, 64]"),
        (lambda: start(ws=None), b"lg_sjd_slot_start_image: scratch must be non-null"),
        (lambda: start(), b"lg_sjd_slot_start_image: engine not finalized"),
        (lambda: copy(src=4), b"lg_copy_slot_kv: source slot 4 outside [0, B=4)"),
        (lambda: copy(src=-1), b"source slot -1 outside"),
        (lambda: copy(dst=(1, 4)), b"lg_copy_slot_kv: destination slot 4 outside [0, B=4)"),
        (lambda: copy(dst=(-1,)), b"destination slot -1 outside"),
        (lambda: copy(dst=(1, 0)), b"lg_copy_slot_kv: destination slot 0 is the source"),
        (lambda: copy(dst=(1, 2, 1)), b"lg_copy_slot_kv: destination slot 1 repeated"),
        (lambda: copy(dst=(), n=2), b"lg_copy_slot_kv: n_dst=2 with null dst_slots"),
        (lambda: copy(n=-1), b"lg_copy_slot_kv: n_dst=-1"),
        (lambda: copy(B=0, src=0), b"source slot 0 outside [0, B=0)"),
        (lambda: copy(length=-1), b"lg_copy_slot_kv: len -1 < 0"),
        (lambda: copy(), b"lg_copy_slot_kv: engine not finalized"),
    ]:
        assert rc_call() < 0, msg
        assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
