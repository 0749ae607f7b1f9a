"""CPU: inpainting requests in serve.LLM (add_request(..., given=, given_mask=)) with the engine replaced by a recording library that
draws on the host: the argument checks and refusals of add_request and LLM.generate (twins included), the argument errors of
lg_extend_slot, lg_slot_extend_workspace_bytes and lg_sample_rows_given through the C-ABI without a GPU, every request's extends
(a, K) and finish step against lg_test_given_plan, no given token ever drawn over, and requests without given tokens making the calls
they make without inpainting."""
import ctypes
import types

import numpy as np
import pytest
import torch

from llamagen_b200 import _lib, serve

T2I_T, C, V = 6, 4, 64
SP = serve.SamplingParams
DRAWS = ("lg_sample_rows", "lg_sample_rows_guided", "lg_sample_rows_keyed", "lg_sample_rows_logprobs", "lg_sample_rows_given")


def _model(model_type):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=V,
                                 cls_token_num=T2I_T if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None, engine=lambda: None,
                                 _slot_scratch=lambda use_cfg: (None, 0), _slot_prefix_scratch=lambda use_cfg, P: (None, 0),
                                 _slot_extend_scratch=lambda use_cfg, K: (None, 0))


def _token(seed, img, k):
    """The token the host draw makes for image img of a request with this seed at index k (never a given id below: ids >= 32)."""
    return 32 + (seed * 7 + img * 13 + k) % 32


class _Lib:
    """The engine's entry points serve.LLM calls, recorded as (name, step, detail); every draw is made on the host from the pointers
    it is given: slot rows from the seed pointer, the step from the step pointer, the given select from the given pointer. Anything
    else (lg_test_given_plan) is the real library's."""

    def __init__(self, llm):
        self.llm, self.real, self.calls = llm, _lib.load(), []

    def __getattr__(self, name):
        if name in DRAWS:
            return lambda *a: self.draw(name, *a)
        if name == "lg_extend_slot":
            return lambda h, tokens, S, a, K, slot, *rest: self.rec(name, (slot, a, K))
        if name.startswith(("lg_decode", "lg_prefill", "lg_copy")):
            return lambda *a: self.rec(name, None)
        return getattr(self.real, name)

    def rec(self, name, detail):
        self.calls.append((name, self.llm.steps_run, detail))
        return 0

    def draw(self, name, logits, n, V_, use_cfg, dt, sc, seeds, steps, *rest):
        st = self.llm._state
        given = rest[-6] if name == "lg_sample_rows_given" else None
        out_idx, out_seq = rest[-4], rest[-3]
        s0 = (seeds.value - st["seeds"].data_ptr()) // 8
        src = next(t for t in (st["pos"], st["join_step"], st.get("step"), st.get("step0")) if t is not None and
                   0 <= steps.value - t.data_ptr() < t.numel() * 4)
        step = src.view(-1)[(steps.value - src.data_ptr()) // 4:][:n if src.numel() > 1 else 1]
        row0 = (out_seq.value - st["out"].data_ptr()) // (4 * st["S"])
        for j in range(n):
            slot, k = s0 + j, int(step[j if step.numel() > 1 else 0])
            req = self.llm._slots[slot]
            t = 0 if req is None else _token(req.seed, self.llm._img[slot], k)
            if given is not None and given.value:
                g = int(st["given"][slot, k])
                t = g if g >= 0 else t
            elif req is not None and req.given is not None and int(req.given[k]) >= 0:
                raise AssertionError(f"slot {slot}: a draw without the given select at given token {k}")
            st["out"][row0 + j, k] = t
            st["tok"][s0 + j] = t
        self.calls.append((name, self.llm.steps_run, (s0, n)))
        return 0


def _llm(monkeypatch, kind, cfg_scale=4.0, **kw):
    llm = serve.LLM(_model(kind), cfg_scale=cfg_scale, num_classes=10, seed=5, **kw)
    lib = _Lib(llm)
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(_lib, "current_stream", lambda dev: None)
    return llm, lib


def _add(llm, i, sp, **kw):
    if llm.t2i:
        feats = torch.randn(2 + i % 3, C, generator=torch.Generator().manual_seed(i))
        return llm.add_request(prompt_embeds=feats, sampling_params=sp, **kw)
    return llm.add_request([i % 10], sp, **kw)


def _mask(S, runs):
    m = torch.zeros(S, dtype=torch.bool)
    for a, b in runs:
        m[a:b] = True
    return m


def _ids(S, seed):
    return torch.randint(0, 32, (S,), generator=torch.Generator().manual_seed(seed))


def _plan(ids, mask):
    row = np.where(mask.numpy(), ids.numpy(), -1).astype(np.int32)
    segs = np.zeros((len(row) + 1, 3), dtype=np.int32)
    n = _lib.load().real.lg_test_given_plan(row.ctypes.data_as(ctypes.c_void_p), 1, len(row), segs.ctypes.data_as(ctypes.c_void_p),
                                            len(row) + 1)
    return [tuple(s) for s in segs[:n].tolist()]


def _drive(llm):
    outs = {}
    while llm.has_unfinished_requests():
        step = llm.steps_run
        for o in llm.step():
            assert o.request_id not in outs
            outs[o.request_id] = (step, o)
    return outs


S = 160
MASKS = {
    "box_hole": _mask(S, [(0, 40), (44, 56), (60, 72), (76, 88), (92, S)]),   # rows of 16 with a 4-wide hole in four rows
    "runs_of_one": _mask(S, [(k, k + 1) for k in range(1, S - 1, 2)]),
    "run_longer_than_64": _mask(S, [(10, 150)]),
    "leading_run_only": _mask(S, [(0, 70)]),
    "trailing_run": _mask(S, [(5, 9), (100, S)]),
    "all_false": _mask(S, []),
}


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("name", list(MASKS))
def test_extends_and_finish_follow_the_engine_plan(monkeypatch, kind, name):
    mask = MASKS[name]
    ids = _ids(S, 3)
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=3)
    _add(llm, 0, SP(max_tokens=S, top_k=1))                                   # a plain request beside it
    rid = _add(llm, 1, SP(max_tokens=S, top_k=1), given=ids, given_mask=mask)
    outs = _drive(llm)
    plan = _plan(ids, mask)
    P = plan[0][2]
    ext = [(a, K) for kind_, a, K in plan if kind_ == 2]
    assert [d[1:] for n, _, d in lib.calls if n == "lg_extend_slot"] == ext
    # one drawn token per step: the LEAD's draw, every DECODE token and every EXTEND's last draw; a c2i prefix join draws in the
    # same step as the first decode
    drawn = 1 + sum(K for kind_, _, K in plan if kind_ == 1) + len(ext)
    assert drawn == S - int(mask.sum())
    assert outs[rid][0] == max(0, drawn - 1 - (1 if kind == "c2i" and P > 0 else 0))
    toks = outs[rid][1].outputs[0].token_ids
    seed = llm._seed + int(rid)
    assert toks == [int(ids[k]) if mask[k] else _token(seed, 0, k) for k in range(S)]
    other = outs["0"][1].outputs[0].token_ids
    assert other == [_token(llm._seed, 0, k) for k in range(S)]
    if ext:   # each extend runs right after the decode of its step, and its draw of token a + K with the slot's key
        i = next(j for j, c in enumerate(lib.calls) if c[0] == "lg_extend_slot")
        assert lib.calls[i - 1][0] == "lg_sample_rows_given" and lib.calls[i + 1][0] == "lg_sample_rows_given"
        assert lib.calls[i + 1][2][1] == 1


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_no_given_token_is_drawn_over_with_n_and_twins(monkeypatch, kind):
    llm, lib = _llm(monkeypatch, kind, max_num_seqs=6)
    Sx = 40
    masks = [_mask(Sx, [(0, 3), (10, 20), (25, 26), (30, Sx)]), _mask(Sx, [(1, 2), (5, 39)])]
    ids = [_ids(Sx, 7), _ids(Sx, 8)]
    sp = [SP(max_tokens=Sx, n=3, seed=11), SP(max_tokens=Sx, cfg_scale=2.0)]
    if kind == "c2i":
        outs = llm.generate(prompt_token_ids=[[3], [4], [10], [10]], sampling_params=sp + sp, givens=ids, given_masks=masks)
        assert [o.outputs[0].token_ids for o in outs[2:]] == [o.outputs[0].token_ids for o in outs[:2]]     # twins mirror
    else:
        f = [torch.randn(3, C, generator=torch.Generator().manual_seed(i)) for i in range(2)]
        outs = llm.generate(prompt_embeds=f, sampling_params=sp, givens=ids, given_masks=masks)
    for r in range(2):
        assert len(outs[r].outputs) == sp[r].n
        for c in outs[r].outputs:
            toks = torch.tensor(c.token_ids)
            assert torch.equal(toks[masks[r]], ids[r][masks[r]]), (r, c.index)
            seed = llm._seed + r if sp[r].seed is None else sp[r].seed
            assert [int(t) for t, g in zip(toks, masks[r]) if not g] == [_token(seed, c.index, k) for k in range(Sx) if not masks[r][k]]
    assert all(n != "lg_sample_rows_logprobs" for n, _, _ in lib.calls)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_requests_without_given_make_the_same_calls(monkeypatch, kind):
    def run(with_given):
        llm, lib = _llm(monkeypatch, kind, max_num_seqs=2)
        _add(llm, 0, SP(max_tokens=12, top_k=1))
        _add(llm, 1, SP(max_tokens=12, top_k=1), prefix=[1, 2])
        _drive(llm)
        assert "given" not in llm._state
        if with_given:   # then an inpainting request runs through, and the plain requests after it draw as before it
            _add(llm, 2, SP(max_tokens=12, top_k=1), given=_ids(12, 1), given_mask=_mask(12, [(4, 8)]))
            _drive(llm)
            n = len(lib.calls)
            _add(llm, 3, SP(max_tokens=12, top_k=1))
            _add(llm, 4, SP(max_tokens=12, top_k=1), prefix=[1, 2])
            _drive(llm)
            return [(c[0], c[2]) for c in lib.calls[n:]]
        return [(c[0], c[2]) for c in lib.calls]
    plain, after = run(False), run(True)
    assert not any(n in ("lg_sample_rows_given", "lg_extend_slot") for n, _ in plain)
    assert [n for n, _ in after] == [n for n, _ in plain]


def test_value_errors(monkeypatch):
    ids, mask = _ids(8, 0), _mask(8, [(2, 4)])
    for kind in ("c2i", "t2i"):
        llm, _ = _llm(monkeypatch, kind, max_num_seqs=4)
        sp = SP(max_tokens=8)
        for kw, msg in [
            (dict(given=ids), "given and given_mask go together"),
            (dict(given_mask=mask), "given and given_mask go together"),
            (dict(given=ids.float(), given_mask=mask), "given must be an integer tensor"),
            (dict(given=ids, given_mask=mask.int()), "given_mask must be a bool tensor"),
            (dict(given=ids[:7], given_mask=mask), "given must be"),
            (dict(given=ids, given_mask=mask[:7]), "given_mask must be"),
            (dict(given=ids[None], given_mask=mask), "given is 1-D"),
            (dict(given=ids, given_mask=mask[None]), "given_mask is 1-D"),
            (dict(given=ids, given_mask=torch.ones(8, dtype=torch.bool)), "at least one token must be drawn"),
            (dict(given=torch.full((8,), V), given_mask=mask), "given token ids must lie in"),
            (dict(given=ids, given_mask=mask, prefix=[1, 2]), "cannot be combined with prefix"),
        ]:
            with pytest.raises(ValueError, match=msg):
                _add(llm, 0, sp, **kw)
        for bad in (SP(max_tokens=8, logprobs=2), SP(max_tokens=8, best_of=2)):
            with pytest.raises(ValueError, match="logprobs or best_of"):
                _add(llm, 0, bad, given=ids, given_mask=mask)
        _add(llm, 0, sp, given=torch.full((8,), V), given_mask=torch.zeros(8, dtype=torch.bool))   # ids are read only where given
        _add(llm, 1, sp, given=ids.tolist(), given_mask=mask.numpy())                               # lists and arrays
        assert llm.get_num_unfinished_requests() == 2
        f = [torch.randn(3, C)] * 2
        gen = (dict(prompt_embeds=f) if kind == "t2i" else dict(prompt_token_ids=[[1], [2], [10], [10]]))
        with pytest.raises(ValueError, match="givens / given_masks hold"):
            llm.generate(sampling_params=sp, givens=[ids], given_masks=[mask], **gen)
        with pytest.raises(ValueError, match="cannot be combined with prefix"):
            llm.generate(sampling_params=sp, givens=[ids, None], given_masks=[mask, None], prefixes=[[1], None], **gen)
        llm, _ = _llm(monkeypatch, kind, max_num_seqs=4, sjd_window=4)
        with pytest.raises(ValueError, match="sjd_window"):
            _add(llm, 0, sp, given=ids, given_mask=mask)
    llm, _ = _llm(monkeypatch, "c2i", max_num_seqs=4)
    rid = llm.add_request([3], SP(max_tokens=8), given=ids, given_mask=mask)
    llm.add_request([10], SP(max_tokens=8), twin_of=rid, given=ids, given_mask=mask)                # the same given: accepted
    with pytest.raises(ValueError, match="mirrors the given tokens"):
        llm.add_request([10], SP(max_tokens=8), twin_of=rid, given=ids, given_mask=_mask(8, [(1, 4)]))
    rid2 = llm.add_request([4], SP(max_tokens=8))
    with pytest.raises(ValueError, match="mirrors the given tokens"):
        llm.add_request([10], SP(max_tokens=8), twin_of=rid2, given=ids, given_mask=mask)


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
def test_new_entry_points_argument_checks():
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no call below reaches a launch
    sc = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 0, 0)
    cfg = _lib.ModelCfg(2, 2, 128, 256, 512, 8, 64, 0, 16, _lib.LG_MODEL_T2I, _lib.LG_DTYPE_BF16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
    c2i = _lib.ModelCfg(2, 2, 128, 256, 512, 1, 64, 10, 0, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_BF16, 1e-5)
    hc = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(c2i), 0, ctypes.byref(hc)) == 0, lib.lg_last_error()

    def given(seq=p, stride=16, g=p):
        return lib.lg_sample_rows_given(p, 1, 64, 1, _lib.LG_DTYPE_F32, ctypes.byref(sc), p, p, p, p, None, g, None, p, seq, stride, None)

    def extend(e=h, tokens=p, S=32, a=4, K=3, slot=0, B=2, cfg=1, em=p, nm=None, ws=p, logits=p):
        return lib.lg_extend_slot(e, tokens, S, a, K, slot, B, cfg, em, nm, ws, 1 << 30, logits, None)

    def nbytes(e=h, K=3):
        n = ctypes.c_size_t()
        return lib.lg_slot_extend_workspace_bytes(e, 1, K, ctypes.byref(n))

    try:
        for rc_call, msg in [
            (lambda: given(seq=None), b"lg_sample_rows_given: given tokens are indexed as out_seq and need it"),
            (lambda: given(stride=0), b"lg_sample_rows_given: given tokens are indexed as out_seq and need it"),
            (lambda: extend(e=None), b"lg_extend_slot: null engine"),
            (lambda: extend(tokens=None), b"lg_extend_slot: null tokens or logits_out"),
            (lambda: extend(logits=None), b"lg_extend_slot: null tokens or logits_out"),
            (lambda: extend(S=2), b"lg_extend_slot: S=2 outside [3, block_size=64]"),
            (lambda: extend(S=65), b"lg_extend_slot: S=65 outside"),
            (lambda: extend(a=0), b"lg_extend_slot: extend [a=0, a + K=3) must lie in [1, S - 1 = 31)"),
            (lambda: extend(K=0), b"lg_extend_slot: extend [a=4, a + K=4)"),
            (lambda: extend(a=29), b"lg_extend_slot: extend [a=29, a + K=32) must lie in [1, S - 1 = 31)"),
            (lambda: extend(slot=2), b"lg_extend_slot: slot 2 outside [0, B=2)"),
            (lambda: extend(slot=-1), b"lg_extend_slot: slot -1 outside"),
            (lambda: extend(B=0, slot=0), b"slot 0 outside [0, B=0)"),
            (lambda: extend(e=hc, em=p), b"lg_extend_slot: emb_mask only applies to t2i models"),
            (lambda: extend(cfg=0, nm=p), b"lg_extend_slot: neg_mask masks the unconditional CFG row and needs use_cfg"),
            (lambda: extend(em=None, nm=p), b"lg_extend_slot: neg_mask needs emb_mask"),
            (lambda: extend(ws=None), b"lg_extend_slot: scratch must be non-null and 256-byte aligned"),
            (lambda: extend(ws=ctypes.c_void_p((1 << 20) + 16)), b"scratch must be non-null and 256-byte aligned"),
            (lambda: extend(), b"lg_extend_slot: engine not finalized"),
            (lambda: nbytes(e=None), b"lg_slot_extend_workspace_bytes: null argument"),
            (lambda: nbytes(K=0), b"lg_slot_extend_workspace_bytes: K=0 outside [1, block_size - 2 = 62]"),
            (lambda: nbytes(K=63), b"K=63 outside"),
        ]:
            assert rc_call() < 0, msg
            assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
        assert nbytes(K=62) == 0 and nbytes(K=1) == 0
    finally:
        lib.lg_engine_destroy(h)
        lib.lg_engine_destroy(hc)
