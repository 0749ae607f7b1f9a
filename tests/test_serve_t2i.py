"""CPU: serve.LLM on text-conditional models with the device calls stubbed (joins, slot reuse, token 0 from the join, the
conditions and masks a join is given, truncation at T, the drain on a change of sampling parameters, the ValueErrors), and the
argument checks of lg_prefill_slot / lg_decode_rows_t2i through the C-ABI without a GPU."""
import ctypes
import types

import numpy as np
import pytest
import torch

from llamagen_b200 import serve
from llamagen_b200.cond import pack_t5_features, prepare_condition

T, C = 6, 4


def _model(model_type="t2i"):
    return types.SimpleNamespace(model_type=model_type, tok_embeddings=types.SimpleNamespace(weight=torch.zeros(1)), vocab_size=64,
                                 cls_token_num=T if model_type == "t2i" else 1, config=types.SimpleNamespace(caption_dim=C),
                                 setup_caches=lambda **kw: None)


class _Device:
    """Stand-ins for the two device calls. A join records what it was given and draws token 0 = 10 * (valid caption tokens); a decode
    checks that every running slot's rows sit at position T + step - 1 (the input of token `step`) and draws input + 1 at that step."""

    def __init__(self, monkeypatch):
        self.joins = []
        monkeypatch.setattr(serve.LLM, "_device_join_t2i", lambda llm, *a: self.join(llm, *a))
        monkeypatch.setattr(serve.LLM, "_device_decode_t2i", lambda llm, *a: self.decode(llm, *a))

    def join(self, llm, st, params, slot):
        self.joins.append(dict(slot=slot, step=llm.steps_run, cond=st["cond"][slot].clone(), mask=st["mask"][slot].clone(),
                               seed=int(st["seeds"][slot]), params=params))
        t0 = 10 * int(st["mask"][slot].sum())
        st["out"][slot, 0] = t0
        st["tok"][slot] = t0

    def decode(self, llm, st, params):
        B, R = llm.max_num_seqs, st["R"]
        for b in range(B):
            if llm._slots[b] is not None:
                assert int(st["pos"][b]) == T + int(st["step"][b]) - 1 and int(st["active"][b]) == 1
                if R == 2 * B:
                    assert int(st["pos"][B + b]) == int(st["pos"][b]) and int(st["active"][B + b]) == 1
        nxt = st["tok"] + 1
        for b in range(B):
            st["out"][b, int(st["step"][b])] = nxt[b]
        st["tok"].copy_(nxt)


def _feats(n, seed):
    return torch.randn(n, C, generator=torch.Generator().manual_seed(seed))


def _expected(f):
    c, m = prepare_condition(*pack_t5_features([f], max_len=T, dim=C), left_padding=True)
    return c[0], m[0]


def test_joins_mid_sequence_and_into_reused_slots(monkeypatch):
    dev = _Device(monkeypatch)
    sp = serve.SamplingParams(top_k=10, max_tokens=3)
    llm = serve.LLM(_model(), cfg_scale=4.0, max_num_seqs=3, seed=100)
    f = [_feats(2, 0), _feats(3, 1).numpy()[None], _feats(5, 2), _feats(8, 3)]      # [n, C] tensors and the .npy layout [1, n, C]
    llm.add_request(prompt_embeds=f[0], sampling_params=sp)
    llm.add_request(None, sp, prompt_embeds=f[1])
    outs = llm.step()                                       # r0, r1 join; token 0 comes from the join
    assert outs == [] and llm._depth[:2] == [1, 1]
    llm.add_request(prompt_embeds=f[2], sampling_params=sp)
    outs += llm.step()                                      # r0, r1 decode token 1, then r2 joins mid-sequence
    assert llm._depth == [2, 2, 1]
    llm.add_request(prompt_embeds=f[3], sampling_params=sp)  # 8 > T valid tokens: truncated at T
    while llm.has_unfinished_requests():
        outs += llm.step()
    # r0, r1 finish at step 3, r3 joins slot 0 (still holding r0's rows) at step 4, r2 finishes then, r3 at step 6
    assert llm.steps_run == 6
    assert [(j["slot"], j["step"]) for j in dev.joins] == [(0, 0), (1, 0), (2, 1), (0, 3)]
    assert [j["seed"] for j in dev.joins] == [100, 101, 102, 103]
    got = {o.request_id: o.outputs[0].token_ids for o in outs}
    assert got == {"0": [20, 21, 22], "1": [30, 31, 32], "2": [50, 51, 52], "3": [60, 61, 62]}
    assert all(o.prompt_token_ids == [] and o.finished for o in outs)
    for j, fi, n in zip(dev.joins, f, (2, 3, 5, T)):
        c, m = _expected(torch.as_tensor(fi))
        assert torch.equal(j["cond"], c) and torch.equal(j["mask"], m)
        assert j["mask"].tolist() == [0.0] * (T - n) + [1.0] * n          # left padding, truncated at T
    assert not llm.has_unfinished_requests() and llm.get_num_unfinished_requests() == 0


def test_generate_surface_and_the_drain_on_a_parameter_change(monkeypatch):
    dev = _Device(monkeypatch)
    a, b = serve.SamplingParams(top_k=10, max_tokens=2), serve.SamplingParams(top_k=20, max_tokens=3)
    llm = serve.LLM(_model(), cfg_scale=1.0, max_num_seqs=2, seed=7)
    feats = [_feats(1, 10), _feats(4, 11), _feats(T, 12)]
    outs = llm.generate(prompt_embeds=feats, sampling_params=[a, b, a])
    assert [o.request_id for o in outs] == ["0", "1", "2"]
    assert [o.outputs[0].token_ids for o in outs] == [[10, 11], [40, 41, 42], [60, 61]]
    # r0 runs alone (2 steps); r1 has other parameters, so it and r2 behind it wait for the drain; r2 waits for r1 (3 steps)
    assert [(j["slot"], j["step"], j["params"]) for j in dev.joins] == [(0, 0, a), (0, 2, b), (0, 5, a)]
    assert llm.steps_run == 7


def test_value_errors():
    t2i, c2i = serve.LLM(_model(), cfg_scale=4.0, max_num_seqs=2), serve.LLM(_model("c2i"), cfg_scale=1.0, max_num_seqs=2)
    bad = [
        lambda: t2i.add_request([3]),                                        # prompt_token_ids on a t2i LLM
        lambda: t2i.add_request(prompt_embeds=None),
        lambda: t2i.add_request(prompt_embeds=torch.zeros(3, C + 1)),        # wrong feature width
        lambda: t2i.add_request(prompt_embeds=np.zeros((1, 3, C + 1), np.float32)),
        lambda: t2i.add_request(prompt_embeds=torch.zeros(2, 3, C)),         # two captions in one request
        lambda: t2i.add_request(prompt_embeds=torch.zeros(0, C)),            # empty caption
        lambda: t2i.add_request(prompt_embeds=torch.zeros(1, 0, C)),
        lambda: t2i.add_request(prompt_embeds=torch.zeros(3, C), twin_of="0"),
        lambda: t2i.generate(prompt_token_ids=[[1]]),
        lambda: t2i.generate(prompt_embeds=[torch.zeros(3, C), torch.zeros(0, C)]),
        lambda: c2i.add_request(prompt_embeds=torch.zeros(3, C)),            # prompt_embeds on a c2i LLM
        lambda: c2i.add_request(),
        lambda: c2i.generate(prompt_embeds=[torch.zeros(3, C)]),
        lambda: serve.LLM(types.SimpleNamespace(model_type="x2i")),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    assert t2i.get_num_unfinished_requests() == 0 and c2i.get_num_unfinished_requests() == 0   # nothing was queued


# ------------------------------------------------------------------------------------------------------------ C-ABI, no GPU
_TINY = dict(n_layer=2, n_head=4, dim=256, ffn_dim=704, vocab_size=1024, cls_token_num=8, block_size=16, caption_dim=64)


def _engine(lib, _lib, model_type, bind=False):
    """A fp32 engine of the tiny shape. bind: every weight bound to a fake 256-aligned address (finalize checks names, shapes and
    alignment on the host only) and a 2-row workspace set, so the checks that need a ready engine run; nothing is ever launched."""
    m = _TINY
    cfg = _lib.ModelCfg(m["n_layer"], m["n_head"], m["dim"], m["ffn_dim"], m["vocab_size"], m["cls_token_num"], m["block_size"], 10,
                        m["caption_dim"], model_type, _lib.LG_DTYPE_F32, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0, lib.lg_last_error()
    if bind:
        D, F, V, Tc, Cd = m["dim"], m["ffn_dim"], m["vocab_size"], m["cls_token_num"], m["caption_dim"]
        shapes = {"tok_embeddings.weight": (V, D), "norm.weight": (D,), "output.weight": (V, D),
                  "cls_embedding.cap_proj.fc1.weight": (D, Cd), "cls_embedding.cap_proj.fc2.weight": (D, D),
                  "cls_embedding.uncond_embedding": (Tc, Cd)}
        for l in range(m["n_layer"]):
            p = f"layers.{l}."
            shapes.update({p + "attention.wqkv.weight": (3 * D, D), p + "attention.wo.weight": (D, D), p + "feed_forward.w1.weight": (F, D),
                           p + "feed_forward.w3.weight": (F, D), p + "feed_forward.w2.weight": (D, F), p + "attention_norm.weight": (D,),
                           p + "ffn_norm.weight": (D,)})
        for name, shape in shapes.items():
            assert lib.lg_engine_bind_weight(h, name.encode(), ctypes.c_void_p(1 << 20), _lib.shape_array(shape), len(shape),
                                             _lib.LG_DTYPE_F32) == 0
        fr = (Tc + m["block_size"], D // m["n_head"] // 2, 2)
        assert lib.lg_engine_bind_weight(h, b"freqs_cis", ctypes.c_void_p(1 << 20), _lib.shape_array(fr), 3, _lib.LG_DTYPE_F32) == 0
        assert lib.lg_engine_finalize(h) == 0, lib.lg_last_error()
        n = ctypes.c_size_t()
        assert lib.lg_engine_workspace_bytes(h, 2, Tc + 8, ctypes.byref(n)) == 0
        assert lib.lg_engine_set_workspace(h, ctypes.c_void_p(1 << 20), n.value, 2, Tc + 8) == 0, lib.lg_last_error()
    return h


def test_prefill_slot_and_decode_rows_t2i_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)          # a non-null, 256-byte aligned address: no check below lets a call reach a launch
    Tc = _TINY["cls_token_num"]
    c2i = _engine(lib, _lib, _lib.LG_MODEL_C2I)
    bare = _engine(lib, _lib, _lib.LG_MODEL_T2I)
    ready = _engine(lib, _lib, _lib.LG_MODEL_T2I, bind=True)
    try:
        one, two, nb = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
        assert lib.lg_slot_workspace_bytes(ready, 0, ctypes.byref(one)) == 0 and lib.lg_slot_workspace_bytes(ready, 1, ctypes.byref(two)) == 0
        assert 0 < one.value < two.value and one.value % 256 == 0
        assert lib.lg_slot_workspace_bytes(c2i, 1, ctypes.byref(nb)) < 0 and b"text-conditional" in lib.lg_last_error()
        assert lib.lg_slot_workspace_bytes(None, 1, ctypes.byref(nb)) < 0

        def prefill(e, cond=p, T=Tc, slot=0, B=1, use_cfg=1, ws=p, ws_bytes=two.value, logits=p):
            return lib.lg_prefill_slot(e, cond, p, T, slot, B, use_cfg, ws, ws_bytes, logits, None)

        for rc_call, msg in [
            (lambda: prefill(None), b"null engine"),
            (lambda: prefill(c2i), b"text-conditional models only"),
            (lambda: prefill(ready, cond=None), b"null cond"),
            (lambda: prefill(ready, logits=None), b"null cond or logits_out"),
            (lambda: prefill(ready, T=Tc - 1), b"must equal cls_token_num"),
            (lambda: prefill(ready, slot=-1), b"outside [0, B=1)"),
            (lambda: prefill(ready, slot=1, B=1), b"outside [0, B=1)"),
            (lambda: prefill(ready, B=0), b"outside"),
            (lambda: prefill(ready, ws=ctypes.c_void_p((1 << 20) + 128)), b"256-byte aligned"),
            (lambda: prefill(ready, ws=None), b"256-byte aligned"),
            (lambda: prefill(bare), b"not finalized"),
            (lambda: prefill(ready, slot=1, B=2), b"rows 4 exceed workspace rows 2"),       # nh * B = 4 rows, the workspace has 2
            (lambda: prefill(ready, ws_bytes=two.value - 1), b"too small"),
            (lambda: prefill(ready, use_cfg=0, ws_bytes=one.value - 256), b"too small"),
        ]:
            assert rc_call() < 0, msg
            assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())

        def decode(e, tok=p, pos=p, B=1, use_cfg=1, logits=p):
            return lib.lg_decode_rows_t2i(e, tok, pos, p, B, use_cfg, logits, None)

        for rc_call, msg in [
            (lambda: decode(None), b"null engine"),
            (lambda: decode(c2i), b"text-conditional models only"),
            (lambda: decode(ready, tok=None), b"bad argument"),
            (lambda: decode(ready, pos=None), b"bad argument"),
            (lambda: decode(ready, logits=None), b"bad argument"),
            (lambda: decode(ready, B=0), b"bad argument"),
            (lambda: decode(bare), b"not finalized"),
            (lambda: decode(ready, B=2), b"rows 4 exceed workspace rows 2"),
        ]:
            assert rc_call() < 0, msg
            assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())
    finally:
        for h in (c2i, bare, ready):
            lib.lg_engine_destroy(h)
