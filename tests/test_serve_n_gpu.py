"""GPU: parallel sampling in serve.LLM (SamplingParams(n=k)), lg_sample_rows_keyed and lg_copy_slot_kv.

* Kernel: random logits, B in {1, 8, 64}, per-row image indices, seeds, steps and guidance, round dtype f32 / bf16 / f16, every filter:
  row b with img_rows[b] = j draws what image j of a per-call lg_sample with that seed, step and guidance draws, bit for bit; with
  img_rows NULL the call equals lg_sample_rows_guided.
* Fan-out: after the join of an n = 3 request beside two running ones, every destination's K / V bytes over positions [0, T + P) equal the source's in every
  layer, unconditional rows included, and every other byte of the cache is what it was (bf16, fp16, an fp8 cache; with and without a
  negative; with a prefix).
* Against generate(): with max_num_seqs = 4, sample j of an n = 4 request equals image j of generate(cond repeated 4 times, seed=s)
  token for token (c2i and t2i, cfg 1.0 and 4.0, a prefix, a negative, sjd_window=4). In fp32 everywhere; in bf16 where generate()
  prefills the batch as the join does. A t2i generate() without a prefix prefills all 4k rows in one batch, whose GEMMs round
  differently from the one-row prefill of a join in bf16: the evidence test shows generate()'s own token-0 logits change from B = 1 to
  B = 4 while sample 0 still equals generate() at B = 1.
* In a busy batch: an n = 3 request among requests joining in waves with mixed guidance, prefixes and negatives returns exactly what
  it returns alone (bf16, fp16, an fp8 KV cache, fp8 weights; plain and sjd_window)."""
import ctypes

import pytest
import torch

from test_serve_guidance_gpu import FILTERS, RD, _rows
from test_serve_prefix_gpu import C2I, _oracle_cond, _prefix
from test_serve_t2i_gpu import XL3, _captions, _model

pytestmark = pytest.mark.gpu

V = 16384


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("B", [1, 8, 64])
def test_keyed_rows_equal_the_per_call_draw_of_their_image(B, rd):
    from llamagen_b200 import _lib
    lib = _lib.load()
    stream = _lib.current_stream("cuda")
    g = torch.Generator().manual_seed(2000 * B + RD[rd])
    x = (3.0 * torch.randn(2 * B, V, generator=g)).cuda()
    scales, intervals, steps, seeds = _rows(B, 3 * B + RD[rd])
    imgs = torch.randint(0, 9, (B,), generator=g, dtype=torch.int32)
    imgs[0] = 0
    if B > 1:
        imgs[1] = 5
    cfg_d, int_d, step_d, seed_d, img_d = scales.cuda(), intervals.cuda(), steps.cuda(), seeds.cuda(), imgs.cuda()
    for f in FILTERS:
        sc = _lib.SampleCfg(99.0, 1, 1.0, f["top_k"], f["top_p"], f["greedy"], 0)
        got = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.lg_sample_rows_keyed(_lib.ptr(x), B, V, 1, RD[rd], ctypes.byref(sc), _lib.ptr(seed_d), _lib.ptr(step_d),
                                            _lib.ptr(cfg_d), _lib.ptr(int_d), _lib.ptr(img_d), _lib.ptr(got), None, 0, stream),
                   "lg_sample_rows_keyed")
        want = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        for b in range(B):
            # image j of a per-call lg_sample: j + 1 images, row b of x as image j (the other images are copies of it)
            j, s, k = int(imgs[b]), float(scales[b]), int(intervals[b])
            call = torch.cat([x[b].expand(j + 1, V), x[B + b].expand(j + 1, V)]).contiguous()
            sc1 = _lib.SampleCfg(s, k, 1.0, f["top_k"], f["top_p"], f["greedy"], int(seeds[b]) & (2 ** 64 - 1))
            out = torch.full((j + 1,), -1, dtype=torch.int32, device="cuda")
            _lib.check(lib.lg_sample(_lib.ptr(call), j + 1, V, int(s > 1.0), RD[rd], ctypes.byref(sc1), int(steps[b]), _lib.ptr(out), None,
                                     stream), "lg_sample")
            want[b] = out[j]
        assert torch.equal(got.cpu(), want.cpu()), (f, (got != want).nonzero().flatten().tolist())
        # img_rows NULL: lg_sample_rows_guided
        null = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.lg_sample_rows_keyed(_lib.ptr(x), B, V, 1, RD[rd], ctypes.byref(sc), _lib.ptr(seed_d), _lib.ptr(step_d),
                                            _lib.ptr(cfg_d), _lib.ptr(int_d), None, _lib.ptr(null), None, 0, stream), "lg_sample_rows_keyed")
        guided = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.lg_sample_rows_guided(_lib.ptr(x), B, V, 1, RD[rd], ctypes.byref(sc), _lib.ptr(seed_d), _lib.ptr(step_d),
                                             _lib.ptr(cfg_d), _lib.ptr(int_d), _lib.ptr(guided), None, 0, stream), "lg_sample_rows_guided")
        assert torch.equal(null.cpu(), guided.cpu()), f


# ------------------------------------------------------------------------------------------------------------ fan-out
def _kv_views(m):
    """(K, V) byte views [layers, rows, H, max_seq, row_bytes] of the model's workspace cache (K first, V from the next 256 bytes)."""
    cfg, buf = m.config, m._workspace
    rows, seq = m._ws_shape
    hd = cfg.dim // cfg.n_head
    eb = 1 if m._kv_cache[0] == "fp8" else m.tok_embeddings.weight.element_size()
    nb = cfg.n_layer * rows * cfg.n_head * seq * hd * eb
    off = (buf.data_ptr() + 255) // 256 * 256 - buf.data_ptr()
    voff = off + (nb + 255) // 256 * 256
    shape = (cfg.n_layer, rows, cfg.n_head, seq, hd * eb)
    return buf[off:off + nb].view(shape), buf[voff:voff + nb].view(shape)


@pytest.mark.parametrize("dt, kv", [(torch.bfloat16, "auto"), (torch.float16, "auto"), (torch.bfloat16, "fp8")], ids=["bf16", "f16", "kv_fp8"])
@pytest.mark.parametrize("neg, P", [(False, 0), (True, 0), (False, 5)], ids=["plain", "negative", "prefix"])
def test_fan_out_copies_the_join_and_nothing_else(dt, kv, neg, P):
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(dt, kv, **XL3)
    S, B, T = 12, 6, XL3["cls_token_num"]
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=B, seed=3)
    cap = _captions([40], XL3["caption_dim"], 1)[0]
    llm.generate(prompt_embeds=[cap], sampling_params=SamplingParams(max_tokens=S))       # the workspace exists and is zero-filled
    for _ in range(2):                                       # slots 0 and 1 run n = 1 requests
        llm.add_request(prompt_embeds=cap, sampling_params=SamplingParams(max_tokens=S))
    llm.step()
    torch.cuda.synchronize()
    K, Vc = _kv_views(m)
    g = torch.Generator(device="cuda").manual_seed(7)
    for t in (K, Vc):                                        # random bytes in the rows of the free slots 2 .. 5
        for half in (0, 1):
            r = t[:, half * B + 2:half * B + B]
            r.copy_(torch.randint(0, 256, r.shape, generator=g, device="cuda", dtype=torch.int32).to(torch.uint8))
    before = (K.clone(), Vc.clone())
    negative = _captions([90], XL3["caption_dim"], 2)[0] if neg else None
    llm.add_request(prompt_embeds=_captions([77], XL3["caption_dim"], 3)[0], sampling_params=SamplingParams(max_tokens=S, n=3),
                    prefix=_prefix(P, m.vocab_size, 4), negative_prompt_embeds=negative)
    pos = llm._state["pos"].tolist()
    llm.step()                                               # decodes every slot (one position each), then the join of slots 2, 3, 4
    torch.cuda.synchronize()
    slots = [i for i in range(B) if llm._slots[i] is not None and llm._slots[i].n == 3]
    assert slots == [2, 3, 4]
    src, dsts, n = slots[0], slots[1:], T + P
    for t, old in zip((K, Vc), before):
        for half in (0, 1):
            r0 = half * B
            assert not torch.equal(t[:, r0 + src, :, :n], old[:, r0 + src, :, :n])          # the prefill wrote the source
            for d in dsts:
                assert torch.equal(t[:, r0 + d, :, :n], t[:, r0 + src, :, :n]), (half, d)
                assert torch.equal(t[:, r0 + d, :, n:], old[:, r0 + d, :, n:]), (half, d)
            assert torch.equal(t[:, r0 + src, :, n:], old[:, r0 + src, :, n:])
            for i in (0, 1, 5):         # the step's decode runs every slot, free ones too (their rows are never read): one position each
                p = pos[r0 + i]
                assert torch.equal(t[:, r0 + i, :, :p], old[:, r0 + i, :, :p]), (half, i)
                assert torch.equal(t[:, r0 + i, :, p + 1:], old[:, r0 + i, :, p + 1:]), (half, i)


# ------------------------------------------------------------------------------------------------------------ against generate()
def _gen_case(kind, dt, case):
    """(model, S, cond for the LLM, prefix or None, negative or None, cfg_scale, sjd_window)."""
    cfg = 1.0 if case == "cfg1" else 4.0
    L = 4 if case == "sjd" else None
    if kind == "t2i":
        m, S = _model(dt, **XL3), 24
        cond = _captions([37], XL3["caption_dim"], 21)[0]
        neg = _captions([64], XL3["caption_dim"], 22)[0] if case == "negative" else None
    else:
        m, S, cond, neg = _model(dt, **C2I), 32, 387, None
    pf = _prefix(6, m.vocab_size, 23) if case == "prefix" else None
    return m, S, cond, pf, neg, cfg, L


GEN_CASES = [("c2i", "cfg1"), ("c2i", "cfg4"), ("c2i", "prefix"), ("c2i", "sjd"),
             ("t2i", "cfg1"), ("t2i", "cfg4"), ("t2i", "prefix"), ("t2i", "negative"), ("t2i", "sjd")]


# t2i without a prefix in bf16: generate() prefills the batch in one pass (see test_bf16_t2i_batched_prefill_rounds_differently)
BATCHED_PREFILL = {("t2i", "cfg1"), ("t2i", "cfg4"), ("t2i", "negative"), ("t2i", "sjd")}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("kind, case", GEN_CASES, ids=[f"{k}_{c}" for k, c in GEN_CASES])
def test_samples_equal_generate_images(kind, case, dt):
    if dt == torch.bfloat16 and (kind, case) in BATCHED_PREFILL:
        pytest.skip("bf16 t2i without a prefix: generate()'s batched prefill rounds differently at B = 4 (evidence test); fp32 covers it")
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m, S, c, pf, neg, cfg, L = _gen_case(kind, dt, case)
    k, seed = 4, 987654321
    llm = LLM(m, cfg_scale=cfg, max_num_seqs=k, seed=1, sjd_window=L)
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, seed=seed, n=k)
    if kind == "t2i":
        rid = llm.add_request(prompt_embeds=c, sampling_params=sp, prefix=pf, negative_prompt_embeds=neg)
    else:
        rid = llm.add_request([c], sp, prefix=pf)
    outs = []
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert [o.request_id for o in outs] == [rid] and [o.index for o in outs[0].outputs] == list(range(k))
    cond, em = _oracle_cond(llm, c)
    kw = dict(cfg_scale=cfg, temperature=1.0, top_k=1000, seed=seed)
    if pf is not None:
        kw["prefix"] = pf[None].expand(k, -1).cuda()
    if neg is not None:
        nc, nm = llm._caption(neg)
        kw.update(negative_cond=nc[None].cuda(), negative_emb_masks=nm[None].cuda())
    if L is not None:
        kw["sjd_window"] = L
    ref = generate(m, cond.expand(k, *cond.shape[1:]).cuda(), S, emb_masks=None if em is None else em.expand(k, -1).cuda(), **kw).cpu()
    for j in range(k):
        assert outs[0].outputs[j].token_ids == ref[j].tolist(), f"sample {j}"
    assert len({tuple(o.token_ids) for o in outs[0].outputs}) == k


@pytest.mark.parametrize("case", ["cfg1", "cfg4"])
def test_bf16_t2i_batched_prefill_rounds_differently(case):
    """Why bf16 t2i without a prefix is compared in fp32: generate()'s token-0 logits of image 0 are not the same bits at B = 1 and
    B = 4 (its prefill is one batched pass of 4 rows), while an n = 4 request's sample 0 equals generate() at B = 1, whose prefill is
    the one-row pass a join runs."""
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m, S, c, _, _, cfg, _ = _gen_case("t2i", torch.bfloat16, case)
    seed = 987654321
    llm = LLM(m, cfg_scale=cfg, max_num_seqs=4, seed=1)
    cond, em = _oracle_cond(llm, c)
    kw = dict(cfg_scale=cfg, temperature=1.0, top_k=1000, seed=seed, return_logits=True)
    t1, l1 = generate(m, cond.cuda(), S, emb_masks=em.cuda(), **kw)
    t4, l4 = generate(m, cond.expand(4, *cond.shape[1:]).cuda(), S, emb_masks=em.expand(4, -1).cuda(), **kw)
    assert not torch.equal(l1[0, 0], l4[0, 0])                                   # token 0's logits: B = 1 and B = 4 round differently
    assert torch.equal(l4[0, 0], l4[0, 1]) and torch.equal(l4[0, 0], l4[0, 3])   # the same bits for every image of the batch
    llm.add_request(prompt_embeds=c, sampling_params=SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, seed=seed, n=4))
    outs = []
    while llm.has_unfinished_requests():
        outs += llm.step()
    assert outs[0].outputs[0].token_ids == t1[0].tolist()


# ------------------------------------------------------------------------------------------------------------ in a busy batch
GUIDES = [(4.0, -1, 11), (2.0, 3, 22), (1.0, -1, 33), (7.5, 0, 44), (4.0, 10, 55), (2.0, -1, 66)]


def _busy_requests(kind, dt, kv, w, sjd):
    from llamagen_b200.serve import SamplingParams
    if kind == "t2i":
        m, S = _model(dt, kv, **XL3), 16
        C = XL3["caption_dim"]
        conds = _captions([5, 37, 64, 120, 17, 90], C, 31)
        negs = [None, _captions([9], C, 3)[0], None, _captions([120], C, 4)[0], None, None]
        Ps = [0, 4, 0, 2, 0, 9]
    else:
        m, S = _model(dt, kv, **C2I), 24
        conds, negs, Ps = [207, 360, 387, 974, 88, 979], [None] * 6, [0, 3, 0, 0, 11, 2]
    if w == "fp8":
        m.set_weight_dtype("fp8")
    reqs = []
    for i, (c, k, s) in enumerate(GUIDES):
        sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, cfg_scale=c, cfg_interval=k, seed=s * 1000 + 7, n=3 if i == 1 else 1)
        reqs.append((conds[i], sp, None if sjd else _prefix(Ps[i], m.vocab_size, 60 + i), negs[i] if c > 1.0 else None))
    return m, S, reqs


def _run_all(llm, reqs, waves):
    """reqs: [(cond, SamplingParams, prefix, negative)]; waves: [(steps to run before the wave, [request indices])]. Returns {index: [tokens
    of every sample]}."""
    llm.request_counter = iter([i for _, w in waves for i in w])
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            c, sp, pf, neg = reqs[i]
            if llm.t2i:
                llm.add_request(prompt_embeds=c, sampling_params=sp, prefix=pf, negative_prompt_embeds=neg)
            else:
                llm.add_request([c], sp, prefix=pf)
    while llm.has_unfinished_requests():
        outs += llm.step()
    return {int(o.request_id): [c.token_ids for c in o.outputs] for o in outs}


@pytest.mark.parametrize("sjd", [False, True], ids=["plain", "sjd"])
@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("dt, kv, w", [(torch.bfloat16, "auto", "auto"), (torch.float16, "auto", "auto"), (torch.bfloat16, "fp8", "auto"),
                                       (torch.bfloat16, "auto", "fp8")], ids=["bf16", "f16", "kv_fp8", "w_fp8"])
def test_n3_in_a_busy_batch_equals_alone(kind, dt, kv, w, sjd):
    from llamagen_b200.serve import LLM
    m, S, reqs = _busy_requests(kind, dt, kv, w, sjd)
    L = 4 if sjd else None
    got = _run_all(LLM(m, cfg_scale=4.0, max_num_seqs=5, seed=5, sjd_window=L), reqs, [(0, [0, 2, 3]), (0, [1]), (3, [4]), (2, [5])])
    assert sorted(got) == list(range(len(reqs))) and len(got[1]) == 3 and all(len(t) == S for o in got.values() for t in o)
    alone = _run_all(LLM(m, cfg_scale=4.0, max_num_seqs=5, seed=5, sjd_window=L), reqs, [(0, [1])])
    assert alone[1] == got[1]
    assert len({tuple(t) for t in got[1]}) == 3
