"""CPU: negative prompts without a GPU. generate()'s ValueErrors, serve.LLM's host logic with the device calls stubbed (the negative's
prepared condition and mask reach the join, requests with and without one share the running batch, per-request lists are checked
before anything is queued, a negative_prompt needs a text_encoder), the argument checks of the *_neg C-ABI siblings, and the
sample_t2i flags."""
import ctypes

import pytest
import torch

from llamagen_b200 import serve
from llamagen_b200.cond import pack_t5_features, prepare_condition
from test_serve_t2i import C, T, _Device, _engine, _feats, _model, _TINY


def _gpt(model_type):
    from llamagen_b200.gpt import ModelArgs, Transformer
    return Transformer(ModelArgs(n_layer=1, n_head=2, dim=64, vocab_size=32, block_size=16, cls_token_num=4, model_type=model_type,
                                 caption_dim=16))


def test_generate_value_errors():
    from llamagen_b200 import generate
    t2i, c2i = _gpt("t2i"), _gpt("c2i")
    cond, em = torch.zeros(2, 4, 16), torch.ones(2, 4)
    neg = torch.zeros(1, 4, 16)
    bad = [
        lambda: generate(c2i, torch.tensor([1, 2]), 4, cfg_scale=4.0, negative_cond=neg),            # c2i: no negative class
        lambda: generate(t2i, cond, 4, em, cfg_scale=1.0, negative_cond=neg),                        # no CFG
        lambda: generate(t2i, cond, 4, em, cfg_scale=0.5, negative_cond=neg),
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_emb_masks=em),                   # a mask without a negative
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=torch.zeros(3, 4, 16)),     # neither 1 nor B
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=torch.zeros(2, 5, 16)),     # T
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=torch.zeros(2, 4, 8)),      # C
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=torch.zeros(4, 16)),        # not 3-D
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=neg, negative_emb_masks=torch.ones(2, 5)),
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=neg, negative_emb_masks=torch.ones(3, 4)),
        lambda: generate(t2i, cond, 4, em, cfg_scale=4.0, negative_cond=neg, teacher=torch.zeros(2, 4, dtype=torch.long)),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()


def _prepared(f):
    c, m = prepare_condition(*pack_t5_features([f], max_len=T, dim=C), left_padding=True)
    return c[0], m[0]


class _NegDevice(_Device):
    """_Device that also records the negative state of a joining slot."""

    def join(self, llm, st, params, slot):
        super().join(llm, st, params, slot)
        self.joins[-1].update(has_neg=st["has_neg"][slot], neg=st["neg"][slot].clone(), neg_mask=st["neg_mask"][slot].clone())


def test_negatives_reach_the_join_and_share_the_batch(monkeypatch):
    dev = _NegDevice(monkeypatch)
    sp = serve.SamplingParams(top_k=10, max_tokens=3)
    llm = serve.LLM(_model(), cfg_scale=4.0, max_num_seqs=3, seed=100)
    f = [_feats(2, 0), _feats(3, 1), _feats(5, 2), _feats(4, 3)]
    negs = [_feats(4, 10), None, _feats(1, 12).numpy()[None], None]
    outs = llm.generate(prompt_embeds=f, sampling_params=sp, negative_prompt_embeds=negs)
    assert [o.outputs[0].token_ids for o in outs] == [[20, 21, 22], [30, 31, 32], [50, 51, 52], [40, 41, 42]]
    # all three slots join at step 0 (no drain between requests with and without a negative); the fourth takes a freed slot
    assert [(j["slot"], j["step"]) for j in dev.joins] == [(0, 0), (1, 0), (2, 0), (0, 3)]
    for j, fi, ng in zip(dev.joins, f, negs):
        c, m = _prepared(torch.as_tensor(fi))
        assert torch.equal(j["cond"], c) and torch.equal(j["mask"], m)
        assert j["has_neg"] == (ng is not None)
        if ng is None:
            assert torch.equal(j["neg_mask"], m)                # the unconditional row keeps its caption's mask
        else:
            nc, nm = _prepared(torch.as_tensor(ng))
            assert torch.equal(j["neg"], nc) and torch.equal(j["neg_mask"], nm)


def test_value_errors_before_anything_is_queued():
    t2i = serve.LLM(_model(), cfg_scale=4.0, max_num_seqs=2)
    no_cfg = serve.LLM(_model(), cfg_scale=1.0, max_num_seqs=2)
    c2i = serve.LLM(_model("c2i"), cfg_scale=1.0, max_num_seqs=2)
    good = torch.zeros(3, C)
    bad = [
        lambda: t2i.add_request(prompt_embeds=good, negative_prompt_embeds=torch.zeros(3, C + 1)),
        lambda: t2i.add_request(prompt_embeds=good, negative_prompt_embeds=torch.zeros(0, C)),
        lambda: t2i.add_request(prompt_embeds=good, negative_prompt="blurry"),                 # no text_encoder
        lambda: no_cfg.add_request(prompt_embeds=good, negative_prompt_embeds=good),           # a negative needs CFG
        lambda: t2i.generate(prompt_embeds=[good, good], negative_prompt_embeds=[good]),       # one per request
        lambda: t2i.generate(prompt_embeds=[good, good], negative_prompt_embeds=[good, torch.zeros(2, C + 1)]),
        lambda: t2i.generate(prompt_embeds=[good, good], negative_prompts=["a", None]),        # no text_encoder
        lambda: t2i.generate(prompt_embeds=[good], negative_prompts=["a"], negative_prompt_embeds=[good]),
        lambda: c2i.add_request([3], negative_prompt_embeds=good),
        lambda: c2i.generate(prompt_token_ids=[[1]], negative_prompt_embeds=[good]),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
    assert all(x.get_num_unfinished_requests() == 0 for x in (t2i, no_cfg, c2i))


def test_negative_prompts_go_through_one_encoder_call(monkeypatch):
    calls = []

    def encoder(prompts):
        calls.append(list(prompts))
        n = len(prompts)
        embs = torch.arange(n, dtype=torch.float32)[:, None, None].expand(n, T, C).clone()
        mask = torch.zeros(n, T)
        mask[:, :2] = 1
        return embs, mask

    encoder.d_model = C
    got = []
    monkeypatch.setattr(serve.LLM, "_enqueue_t2i", lambda self, c, p, pf, ng=None: got.append((c, ng)))
    llm = serve.LLM(_model(), cfg_scale=4.0, max_num_seqs=2, text_encoder=encoder)
    llm.generate(prompts=["a", "b", "c"], negative_prompts=["x", None, "z"])
    assert calls == [["a", "b", "c", "x", "z"]]
    assert [g[0][0][-1, 0].item() for g in got] == [0.0, 1.0, 2.0]
    assert got[1][1] is None and got[0][1][0][-1, 0].item() == 3.0 and got[2][1][0][-1, 0].item() == 4.0
    calls.clear()
    llm.add_request(prompt="a", negative_prompt="x")
    assert calls == [["a", "x"]]


def test_neg_siblings_argument_checks():
    from llamagen_b200 import _lib
    lib = _lib.load()
    p = ctypes.c_void_p(1 << 20)
    Tc = _TINY["cls_token_num"]
    c2i = _engine(lib, _lib, _lib.LG_MODEL_C2I)
    ready = _engine(lib, _lib, _lib.LG_MODEL_T2I, bind=True)
    try:
        cfg = _lib.SampleCfg(4.0, -1, 1.0, 0, 1.0, 0, 0)
        nocfg = _lib.SampleCfg(1.0, -1, 1.0, 0, 1.0, 0, 0)

        def gen(e, em=p, neg=p, nm=p, sc=cfg):
            return lib.lg_generate_neg(e, p, em, neg, nm, 1, Tc, 4, ctypes.byref(sc), p, None, None, None)

        def pre(e, em=p, neg=p, nm=p, sc=cfg):
            return lib.lg_generate_prefix_neg(e, p, em, neg, nm, 1, Tc, 4, ctypes.byref(sc), p, 1, p, 1 << 30, p, None, None)

        def sjd(e, em=p, neg=p, nm=p, sc=cfg):
            return lib.lg_generate_sjd_neg(e, p, em, neg, nm, 1, Tc, 4, ctypes.byref(sc), 2, p, 1 << 30, p, p, None, None)

        def slot(e, em=p, neg=p, nm=p, use_cfg=1):
            return lib.lg_prefill_slot_prefix_neg(e, p, em, neg, nm, Tc, None, 0, 0, 1, use_cfg, p, 1 << 30, p, None)

        for fn, name in ((gen, b"lg_generate_neg"), (pre, b"lg_generate_prefix_neg"), (sjd, b"lg_generate_sjd_neg")):
            for rc_call, msg in [
                (lambda: fn(None), b"null engine" if fn is gen else b"not finalized"),
                (lambda: fn(c2i), b"t2i models only" if fn is gen else b"not finalized"),
                (lambda: fn(ready, sc=nocfg), b"needs CFG"),
                (lambda: fn(ready, neg=None), b"neg_mask without neg_cond"),
                (lambda: fn(ready, em=None), b"neg_mask needs emb_mask"),
            ]:
                assert rc_call() < 0, msg
                err = lib.lg_last_error()
                assert msg in err and name in err, (name, msg, err)
        for rc_call, msg in [
            (lambda: slot(None), b"null engine"),
            (lambda: slot(ready, use_cfg=0), b"needs CFG"),
            (lambda: slot(ready, neg=None), b"neg_mask without neg_cond"),
            (lambda: slot(ready, em=None), b"neg_mask needs emb_mask"),
        ]:
            assert rc_call() < 0, msg
            assert msg in lib.lg_last_error(), (msg, lib.lg_last_error())

        def dec(e, em=p, nm=p, use_cfg=1):
            return lib.lg_decode_rows_t2i_neg(e, p, p, em, nm, 1, use_cfg, p, None)

        for rc_call, msg in [
            (lambda: dec(None), b"null engine"),
            (lambda: dec(c2i), b"text-conditional models only"),
            (lambda: dec(ready, use_cfg=0), b"needs use_cfg"),
            (lambda: dec(ready, em=None), b"neg_mask needs emb_mask"),
        ]:
            assert rc_call() < 0, msg
            assert b"lg_decode_rows_t2i_neg" in lib.lg_last_error() and msg in lib.lg_last_error(), (msg, lib.lg_last_error())
        # the test sibling of lg_test_attention: a second mask needs the first
        rc = lib.lg_test_attention_neg(_lib.LG_DTYPE_F32, _lib.LG_DTYPE_F32, 1.0, 1.0, 2, 1, 1, 64, 64, 8, p, p, 1, 0, 0, None, None, None,
                                       p, 1, 4, p, None, 0, None, 0, None, p, None, None)
        assert rc < 0 and b"emb_mask_uncond needs emb_mask" in lib.lg_last_error()
    finally:
        for h in (c2i, ready):
            lib.lg_engine_destroy(h)


def test_sample_t2i_flags():
    from llamagen_b200.sample import sample_t2i
    parse = sample_t2i.build_parser().parse_args
    a = parse(["--negative-prompt", "blurry, low quality"])
    assert a.negative_prompt == "blurry, low quality" and a.negative_cond_npy is None
    sample_t2i.check_negative_args(a)
    b = parse(["--synthetic-cond", "--negative-cond-npy", "neg.npy"])
    assert b.negative_cond_npy == "neg.npy" and b.negative_prompt is None
    for argv in (["--negative-prompt", "x", "--negative-cond-npy", "n.npy"], ["--negative-prompt", "x", "--cfg-scale", "1.0"]):
        with pytest.raises(SystemExit):
            sample_t2i.check_negative_args(parse(argv))
