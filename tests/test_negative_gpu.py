"""GPU: negative prompts, a caption in place of the null condition of classifier-free guidance.

* Identity anchor: the negative uncond_embedding with negative_emb_masks = emb_masks gives the tokens and logits of no negative, bit for
  bit: fp32 and bf16, plain / prefix / sjd_window, one and two chains (LG_SPLIT), R <= 8 and batched decode, 16-bit and fp8 KV caches.
* fp32 greedy tokens bit-exact against the negative oracle (tests/negative_oracle.py), logits within 1e-4; bf16 / fp16 teacher-forced
  logits against it within 1.5 x the oracle's own 16-bit spread plus the dtype floor.
* The mask is per row: every attention kernel through lg_test_attention_neg equals lg_test_attention with the two masks stacked as 2B
  mask rows; end to end, features under mask 0 are never read, and the caption's mask in place of the negative's changes the logits.
* serve.LLM: mixed running sets give the same tokens under three schedules, fp32 greedy tokens match the oracle in waves, and
  negative_prompts strings equal negative_prompt_embeds of the encoder's features.
* sample_t2i --negative-cond-npy writes its image."""
import ctypes

import numpy as np
import pytest
import torch

from negative_oracle import negative_oracle
from oracle import GPTOracle
from util import build_gpt, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

XL2 = dict(n_layer=2, n_head=20, dim=1280, vocab_size=16384, block_size=256, cls_token_num=120, model_type="t2i", caption_dim=2048)
FLOORS = {torch.bfloat16: 0.02, torch.float16: 0.0025}


def _model(dt, kv="auto", **cfg):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(1234)
    m = Transformer(ModelArgs(**cfg))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dt).eval()
    m.set_kv_cache(kv)
    return m


def _cond(B, T, C, lens, seed, dt=torch.float32):
    """Prepared conditions (left-padded, padding zeroed) of random features with valid lengths `lens`, and their masks."""
    from llamagen_b200.cond import prepare_condition
    g = torch.Generator().manual_seed(seed)
    masks = torch.stack([(torch.arange(T) < n).float() for n in lens])
    c, m = prepare_condition(torch.randn(B, T, C, generator=g) * masks[:, :, None], masks)
    return c.to(dt), m


def _gen(m, cond, S, em, **kw):
    from llamagen_b200 import generate
    out = generate(m, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), **kw)
    torch.cuda.synchronize()
    return tuple(o.cpu() for o in out) if isinstance(out, tuple) else out.cpu()


def _uncond(m):
    return m.cls_embedding.uncond_embedding.detach()[None]


# ------------------------------------------------------------------------------------------------------------ identity anchor
@pytest.mark.parametrize("dt, kv, B, split", [
    (torch.float32, "auto", 2, "1"), (torch.bfloat16, "auto", 3, "1"), (torch.bfloat16, "auto", 16, "1"), (torch.bfloat16, "auto", 16, "2"),
    (torch.bfloat16, "fp8", 16, "2"), (torch.bfloat16, "fp8", 4, "1"),
], ids=["f32_small", "bf16_small", "bf16_batched", "bf16_two_chains", "bf16_kv_fp8_two_chains", "bf16_kv_fp8_small"])
def test_identity_anchor(dt, kv, B, split, monkeypatch):
    monkeypatch.setenv("LG_SPLIT", split)
    m = _model(dt, kv, **XL2)
    S, T, C = 24, 120, 2048
    cond, em = _cond(B, T, C, [(17 * b + 5) % 120 + 1 for b in range(B)], 3, dt)
    neg = _uncond(m).cpu()
    kw = dict(cfg_scale=7.5, sample_logits=False)
    a_t, a_l = _gen(m, cond, S, em, return_logits=True, **kw)
    b_t, b_l = _gen(m, cond, S, em, return_logits=True, negative_cond=neg, negative_emb_masks=em, **kw)
    assert torch.equal(a_t, b_t) and torch.equal(a_l, b_l)
    pf = a_t[:, :5].clone()
    a_t, a_l = _gen(m, cond, S, em, return_logits=True, prefix=pf, **kw)
    b_t, b_l = _gen(m, cond, S, em, return_logits=True, prefix=pf, negative_cond=neg.expand(B, T, C).clone(), negative_emb_masks=em, **kw)
    assert torch.equal(a_t, b_t) and torch.equal(a_l, b_l)
    a = _gen(m, cond, S, em, sjd_window=6, seed=9, cfg_scale=7.5)
    b = _gen(m, cond, S, em, sjd_window=6, seed=9, cfg_scale=7.5, negative_cond=neg, negative_emb_masks=em)
    assert torch.equal(a, b)
    # without emb_masks a negative gives both halves all-ones masks: the same visibility as no mask
    a = _gen(m, cond, S, None, seed=4, cfg_scale=7.5, top_k=100)
    b = _gen(m, cond, S, None, seed=4, cfg_scale=7.5, top_k=100, negative_cond=neg)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ against the oracle
def test_fp32_exact_against_negative_oracle():
    g = load_golden("gpt_t2i.pt")
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    T, C, S = g["cfg"]["cls_token_num"], g["cfg"]["caption_dim"], g["S"]
    cond, em = g["cond"], g["emb_masks"]
    B = cond.shape[0]
    valid = em.sum(-1).long().tolist()
    neg, nm = _cond(B, T, C, [max(1, T - v) if v < T else T // 2 for v in valid], 11)   # valid lengths that differ from the caption's
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for cfg_scale, neg_in, nm_in in ((4.0, neg, nm), (7.5, neg[:1], nm[:1])):
        out, logits = _gen(m, cond, S, em, cfg_scale=cfg_scale, sample_logits=False, return_logits=True, negative_cond=neg_in,
                           negative_emb_masks=nm_in)
        want, wl = negative_oracle(orc, cond, neg_in, S, emb_masks=em, negative_emb_masks=nm_in, cfg_scale=cfg_scale, sample_logits=False)
        assert torch.equal(out, want.cpu()), f"cfg {cfg_scale}: greedy tokens differ from the negative oracle"
        assert (logits - wl.cpu()).abs().max().item() <= 1e-4


def _generate_neg_teacher(m, cond, em, neg, nm, S, teacher, cfg_scale):
    """lg_generate_neg with a teacher: the mixed logits [S, B, V] of every step fed the teacher's tokens."""
    from llamagen_b200 import _lib
    lib, h = _lib.load(), m.engine()
    B, T = cond.shape[:2]
    dt = m.tok_embeddings.weight.dtype
    m.setup_caches(max_batch_size=2 * B, max_seq_length=T + S, dtype=dt)
    c, n = cond.cuda().to(dt).contiguous(), neg.cuda().to(dt).expand(B, -1, -1).contiguous()
    e, nmd = em.cuda().float().contiguous(), nm.cuda().float().contiguous()
    tf = teacher.cuda().to(torch.int32).contiguous()
    out = torch.empty(B, S, dtype=torch.int32, device="cuda")
    dbg = torch.empty(S, B, m.vocab_size, dtype=torch.float32, device="cuda")
    sc = _lib.SampleCfg(float(cfg_scale), -1, 1.0, 0, 1.0, 1, 0)
    _lib.check(lib.lg_generate_neg(h, _lib.ptr(c), _lib.ptr(e), _lib.ptr(n), _lib.ptr(nmd), B, T, S, ctypes.byref(sc), _lib.ptr(out),
                                   _lib.ptr(dbg), _lib.ptr(tf), _lib.current_stream("cuda")), "lg_generate_neg")
    torch.cuda.synchronize()
    return dbg.cpu()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_16bit_teacher_forced_against_negative_oracle(dt):
    m = _model(dt, **XL2)
    S, T, C = 12, 120, 2048
    cond, em = _cond(3, T, C, [40, 120, 7], 21)
    neg, nm = _cond(3, T, C, [90, 3, 60], 22)
    sd16 = {k: v.detach() for k, v in m.state_dict().items()}
    sd32 = {k: v.float() for k, v in sd16.items()}
    kw = dict(emb_masks=em.cuda(), negative_emb_masks=nm.cuda(), cfg_scale=7.5, sample_logits=False)
    ref_t, ref_l = negative_oracle(GPTOracle(sd32, oracle_cfg(m)), cond.cuda(), neg.cuda(), S, **kw)
    _, h_l = negative_oracle(GPTOracle(sd16, oracle_cfg(m)), cond.cuda().to(dt), neg.cuda().to(dt), S, teacher=ref_t, **kw)
    ref_t, ref_l, h_l = ref_t.cpu(), ref_l.cpu(), h_l.cpu()
    tol = 1.5 * (h_l - ref_l).abs().max().item() + FLOORS[dt]
    lg = _generate_neg_teacher(m, cond, em, neg, nm, S, ref_t, 7.5)
    err = (lg - ref_l).abs().max().item()
    assert err <= tol, f"|engine - ref32| {err:.4g} > bound {tol:.4g}"
    sure = top2_gap(ref_l) > 2 * tol
    assert torch.equal(lg.argmax(-1)[sure], ref_l.argmax(-1)[sure])
    print(f"{dt}: err {err:.4g} bound {tol:.4g}")


# ------------------------------------------------------------------------------------------------------------ the mask is per row
def _attn(neg_mask, dtype, kv_dtype, R, Tq, H, hd, max_seq, pos_value, pos_rows, emb_mask, B, Tc, seed):
    """One call of lg_test_attention_neg (neg_mask not None) or lg_test_attention on seeded buffers; returns (out, kernel)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    tdt = {_lib.LG_DTYPE_F32: torch.float32, _lib.LG_DTYPE_BF16: torch.bfloat16}[dtype]
    k = torch.randn(R, H, max_seq, hd, generator=g)
    v = torch.randn(R, H, max_seq, hd, generator=g)
    if kv_dtype == _lib.LG_DTYPE_E4M3:
        k, v = (x.to(torch.float8_e4m3fn).view(torch.uint8).cuda() for x in (k, v))
    else:
        k, v = k.to(tdt).cuda(), v.to(tdt).cuda()
    q = torch.randn(R * Tq, H * hd, generator=g).to(tdt).cuda()
    out = torch.empty(R * Tq, H * hd, dtype=tdt, device="cuda")
    path = (ctypes.c_int * 3)()
    pr = None if pos_rows is None else torch.tensor(pos_rows, dtype=torch.int32, device="cuda")
    em = emb_mask.cuda().contiguous()
    args = [dtype, kv_dtype, 1.0, 1.0, R, Tq, H, hd, hd, max_seq, _lib.ptr(k), _lib.ptr(v), 1, 0, pos_value, None, _lib.ptr(pr), _lib.ptr(em)]
    tail = [B, Tc, _lib.ptr(q), None, 0, None, 0, None, _lib.ptr(out), path, _lib.current_stream("cuda")]
    if neg_mask is None:
        _lib.check(lib.lg_test_attention(*args, *tail), "lg_test_attention")
    else:
        nm = neg_mask.cuda().contiguous()
        _lib.check(lib.lg_test_attention_neg(*args, _lib.ptr(nm), *tail), "lg_test_attention_neg")
    torch.cuda.synchronize()
    return out.float().cpu(), path[0]


def test_every_attention_kernel_reads_the_unconditional_mask_per_row():
    from llamagen_b200 import _lib
    B, Tc, H, hd = 2, 120, 4, 64
    g = torch.Generator().manual_seed(0)
    em = (torch.rand(B, Tc, generator=g) > 0.4).float()
    nm = (torch.rand(B, Tc, generator=g) > 0.6).float()
    f32, b16, e4 = _lib.LG_DTYPE_F32, _lib.LG_DTYPE_BF16, _lib.LG_DTYPE_E4M3
    cases = [   # (dtype, kv, Tq, max_seq, pos_value, pos_rows)
        (b16, b16, 1, 136, 125, None),                # 1 attn_tma_kernel (decode)
        (b16, e4, 1, 136, 125, None),
        (b16, b16, 120, 128, 0, None),                # 3 attn_prefill_tc_kernel (the condition prefill)
        (b16, b16, 130, 136, 0, None),                # 2 attn_causal_tc_kernel (prefix prefills)
        (b16, e4, 130, 136, 0, None),                 # 2 attn_causal_tc_f8_kernel
        (b16, b16, 6, 136, 0, [121, 118, 125, 122]),  # 4 attn_window_tc_kernel (speculative windows)
        (f32, f32, 1, 128, 121, None),                # 0 attention_kernel (CUDA cores)
        (f32, f32, 120, 128, 0, None),
    ]
    kernels = set()
    for i, (dt, kv, Tq, ms, pv, pr) in enumerate(cases):
        common = (dt, kv, 2 * B, Tq, H, hd, ms, pv, pr)
        got, kern = _attn(nm, *common, em, B, Tc, 100 + i)
        stacked, k2 = _attn(None, *common, torch.cat([em, nm]), 2 * B, Tc, 100 + i)   # 2B mask rows: row r reads row r
        plain, _ = _attn(None, *common, em, B, Tc, 100 + i)
        same, _ = _attn(em, *common, em, B, Tc, 100 + i)
        kernels.add(kern)
        assert kern == k2 and torch.equal(got, stacked), f"case {i} (kernel {kern}): the unconditional rows do not read neg_mask"
        assert torch.equal(same, plain), f"case {i}: emb_mask_uncond = emb_mask is not the sibling's result"
        assert torch.equal(got[: B * Tq], plain[: B * Tq]), f"case {i}: the conditional rows changed"
        assert not torch.equal(got[B * Tq:], plain[B * Tq:]), f"case {i}: the unconditional rows ignore neg_mask"
    assert kernels == {0, 1, 2, 3, 4}, kernels


@pytest.mark.parametrize("dt, kv", [(torch.float32, "auto"), (torch.bfloat16, "auto"), (torch.bfloat16, "fp8")])
def test_masked_negative_features_are_never_read(dt, kv):
    m = _model(dt, kv, **XL2)
    S, T, C, B = 10, 120, 2048, 2
    cond, em = _cond(B, T, C, [50, 100], 31, dt)
    neg, nm = _cond(B, T, C, [20, 70], 32, dt)
    garbage = neg + (1 - nm)[:, :, None].to(dt) * 3.0       # non-zero features where the negative's mask is 0
    kw = dict(cfg_scale=7.5, sample_logits=False, return_logits=True)
    for extra in (dict(), dict(prefix=torch.zeros(B, 140, dtype=torch.long) + 5, max_tokens=150), dict(sjd=True)):
        S_ = extra.pop("max_tokens", S)
        if extra.pop("sjd", False):
            a = _gen(m, cond, S_, em, cfg_scale=7.5, sjd_window=4, seed=1, negative_cond=neg, negative_emb_masks=nm)
            b = _gen(m, cond, S_, em, cfg_scale=7.5, sjd_window=4, seed=1, negative_cond=garbage, negative_emb_masks=nm)
            assert torch.equal(a, b)
            continue
        a = _gen(m, cond, S_, em, negative_cond=neg, negative_emb_masks=nm, **kw, **extra)
        b = _gen(m, cond, S_, em, negative_cond=garbage, negative_emb_masks=nm, **kw, **extra)
        c = _gen(m, cond, S_, em, negative_cond=neg, negative_emb_masks=em, **kw, **extra)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), f"{extra.keys()}: features under mask 0 were read"
        P = extra["prefix"].shape[1] if "prefix" in extra else 0
        assert not torch.equal(a[1][P:], c[1][P:]), f"{extra.keys()}: the unconditional rows ignore their own mask"


# ------------------------------------------------------------------------------------------------------------ serving
def _feats(lens, C, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((n, C)).astype(np.float32) for n in lens]


def _run(llm, feats, negs, sp, waves):
    order = [i for _, w in waves for i in w]
    llm.request_counter = iter(order)
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            llm.add_request(prompt_embeds=feats[i], sampling_params=sp, negative_prompt_embeds=negs[i])
    while llm.has_unfinished_requests():
        outs += llm.step()
    return {int(o.request_id): o.outputs[0].token_ids for o in outs}


@pytest.mark.parametrize("dt, kv", [(torch.bfloat16, "auto"), (torch.bfloat16, "fp8")])
def test_serve_mixed_sets_do_not_depend_on_the_schedule(dt, kv):
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(dt, kv, **XL2)
    feats = _feats([5, 120, 37, 64, 9, 88], 2048, 1)
    negs = [f if i % 2 else None for i, f in enumerate(_feats([30, 2, 99, 120, 15, 50], 2048, 2))]
    sp = SamplingParams(temperature=1.0, top_k=100, max_tokens=12)
    runs = []
    for waves in ([(0, [0, 1, 2, 3, 4, 5])], [(0, [0, 1]), (3, [2, 3]), (4, [4, 5])], [(0, [5, 4]), (2, [3, 2, 1, 0])]):
        runs.append(_run(LLM(m, cfg_scale=7.5, max_num_seqs=3, seed=5), feats, negs, sp, waves))
    assert runs[0] == runs[1] == runs[2]


def test_serve_fp32_exact_against_oracle_in_three_waves():
    from llamagen_b200.cond import pack_t5_features, prepare_condition
    from llamagen_b200.serve import LLM, SamplingParams
    g = load_golden("gpt_t2i.pt")
    T, C, S = g["cfg"]["cls_token_num"], g["cfg"]["caption_dim"], g["S"]
    feats = _feats([5, 37, 64, 120, 9, 88], C, 7)
    negs = [None, *_feats([3, 120], C, 8), None, *_feats([60, 11], C, 9)]
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    got = _run(LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=3), feats, negs, SamplingParams(temperature=0.0, max_tokens=S),
               [(0, [0, 1]), (3, [2, 3, 4]), (S + 5, [5])])
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for i, f in enumerate(feats):
        c, mk = prepare_condition(*pack_t5_features([f], T, C))
        if negs[i] is None:
            ref, _ = orc.generate(c, S, emb_masks=mk, cfg_scale=4.0, sample_logits=False)
        else:
            nc, nmk = prepare_condition(*pack_t5_features([negs[i]], T, C))
            ref, _ = negative_oracle(orc, c, nc, S, emb_masks=mk, negative_emb_masks=nmk, cfg_scale=4.0, sample_logits=False)
        assert got[i] == ref[0].tolist(), f"caption {i}"


def test_serve_negative_prompts_equal_their_features():
    from llamagen_b200.gpt import ModelArgs, Transformer
    from llamagen_b200.serve import LLM, SamplingParams
    from test_t5_gpu import TINY, _encoder, _StubTokenizer
    gd = load_golden("t5_tiny.pt")
    enc = _encoder(TINY, gd["state_dict"], torch.bfloat16, max_length=12, tokenizer=_StubTokenizer())
    torch.manual_seed(5)
    gpt = Transformer(ModelArgs(n_layer=2, n_head=2, dim=128, vocab_size=256, block_size=16, cls_token_num=12, model_type="t2i",
                                caption_dim=128))
    gpt.output.weight.data.normal_(std=0.02)
    gpt = gpt.to(device="cuda", dtype=torch.bfloat16).eval()
    prompts = ["a red cube on a table", "two cats", "sun"]
    negatives = ["blurry", None, "a dark and grainy picture"]
    embs, mk = enc(prompts + [negatives[0], negatives[2]])
    feats = [embs[i][mk[i] != 0] for i in range(5)]
    sp = SamplingParams(temperature=1.0, top_k=0, max_tokens=16)
    a = LLM(gpt, cfg_scale=4.0, max_num_seqs=2, seed=11, text_encoder=enc).generate(prompts=prompts, sampling_params=sp,
                                                                                   negative_prompts=negatives)
    b = LLM(gpt, cfg_scale=4.0, max_num_seqs=2, seed=11).generate(prompt_embeds=feats[:3], sampling_params=sp,
                                                                  negative_prompt_embeds=[feats[3], None, feats[4]])
    c = LLM(gpt, cfg_scale=4.0, max_num_seqs=2, seed=11).generate(prompt_embeds=feats[:3], sampling_params=sp)
    ta, tb, tc = ([o.outputs[0].token_ids for o in x] for x in (a, b, c))
    assert ta == tb and tb[1] == tc[1] and tb != tc
    llm = LLM(gpt, cfg_scale=4.0, max_num_seqs=2, seed=11, text_encoder=enc)
    llm.request_counter = iter([0])
    llm.add_request(prompt=prompts[0], negative_prompt=negatives[0], sampling_params=sp)
    outs = []
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert outs[0].outputs[0].token_ids == ta[0]


# ------------------------------------------------------------------------------------------------------------ CLI
def test_sample_t2i_negative_cond_npy(tmp_path, monkeypatch):
    from llamagen_b200.sample import sample_t2i
    monkeypatch.chdir(tmp_path)
    np.save(tmp_path / "neg.npy", np.random.default_rng(0).standard_normal((1, 17, 2048)).astype(np.float32))
    args = sample_t2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--image-size", "256", "--synthetic-cond",
                                                 "--negative-cond-npy", str(tmp_path / "neg.npy")])
    sample_t2i.main(args)
    assert (tmp_path / "sample_t2i.png").stat().st_size > 10000
