"""GPU: token log-probabilities of the sample kernel (lg_sample_rows_logprobs), of generate(return_logprobs=True) and of serve.LLM
(SamplingParams(logprobs=, best_of=)).

* Kernel, one call at a time over test_sample_kernel_gpu's case matrix, each case with its own rounding, with fp32 / bf16 / fp16
  rounding, with CFG at per-row scales and intervals, and greedy: the picks equal lg_sample_rows_keyed's; rank and the top-N ids are
  exact against the fp32 row restated from the logits (over the kernel's own kept set, which differs from the float64 filter's only in
  the top-p band); the logprobs lie within LP_ABS + |x - max| 2^-22 of the float64 oracle (the kernel rounds x - max once and
  log(Z), an fp32 sum of V terms, once); exp(logprob of the pick) equals out_probs[pick] within 1e-5 relative.
* generate(): the tokens are bit-identical with and without return_logprobs (c2i, t2i, CFG, a negative, a prefix, an fp8 KV cache, one
  and two chains; S large enough for the captured graph), and one and two chains give the same logprobs.
* Against score(): at temperature 1 without top-k / top-p, generate's logprobs equal -score(tokens) at cfg 1 and 4: fp32 within 1e-3,
  bf16 within 3 times the spread between bf16 and fp32 score() of the same tokens, plus 1e-3.
* serve.LLM: every request's per-token dicts and cumulative_logprob equal generate(return_logprobs=True, top_logprobs=N) of its images
  (fp32 golden models: c2i twins, t2i, per-request guidance, n, prefix, staggered arrivals; a bf16 model with fp8 weights), and
  best_of = m returns the n images of generate(cond repeated m times) with the largest row sums, in that order."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

import logprob_oracle as lo
import test_sample_kernel_gpu as sk
from util import build_gpt, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda"
LP_ABS = 2e-5
N_TOP = 20
WORST = {"lp": 0.0}


# ------------------------------------------------------------------------------------------------------------ kernel
def _rows_call(lib, logits, B, V, mix, rd, sc, seeds, steps, cfg_rows, int_rows, S, lp_spec):
    """lg_sample_rows_logprobs (lp_spec: an lg_logprobs or None) -> (picks, token rows [B, S])."""
    from llamagen_b200 import _lib
    idx = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    seq = torch.full((B, S), -5, dtype=torch.int32, device=DEV)
    _lib.check(lib.lg_sample_rows_logprobs(_lib.ptr(logits), B, V, int(mix), sk.RD[rd], ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                           _lib.ptr(cfg_rows), _lib.ptr(int_rows), None, ctypes.byref(lp_spec) if lp_spec else None,
                                           _lib.ptr(idx), _lib.ptr(seq), S, _lib.current_stream(DEV)), "lg_sample_rows_logprobs")
    return idx, seq


VARIANTS = ["own", "f32", "bf16", "f16", "cfg_rows", "greedy"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("cid", list(sk.CASE_BY_ID))
def test_kernel_logprobs_against_the_float64_oracle(cid, variant):
    from dataclasses import replace

    from llamagen_b200 import _lib
    lib = _lib.load()
    c = sk.CASE_BY_ID[cid]
    if variant in ("f32", "bf16", "f16"):
        c = replace(c, rd=variant)
    elif variant == "cfg_rows":
        c = replace(c, mix=True, cfg=4.0, interval=3)
    elif variant == "greedy":
        c = replace(c, greedy=True)
    seed = zlib.crc32((c.id + variant).encode())
    x = sk.make_logits(c, torch.Generator().manual_seed(seed))
    B, V, step = c.B, c.V, c.step
    logits = torch.from_numpy(x.reshape(-1)).to(DEV)
    g = torch.Generator().manual_seed(seed)
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64)
    steps = torch.full((B,), step, dtype=torch.int32)
    cfg_rows = int_rows = None
    scales = np.full(B, c.cfg, np.float32)
    intervals = np.full(B, c.interval)
    if variant == "cfg_rows":
        scales = np.array([0.5, 1.0, 2.5, 4.0, 7.5], np.float32)[torch.randint(0, 5, (B,), generator=g).numpy()]
        intervals = np.array([-1, 0, 3, 10 ** 6])[torch.randint(0, 4, (B,), generator=g).numpy()]
        steps = torch.randint(0, 8, (B,), generator=g, dtype=torch.int32)
        cfg_rows = torch.from_numpy(scales).to(DEV)
        int_rows = torch.from_numpy(intervals.astype(np.int32)).to(DEV)
    S = int(steps.max()) + 1
    sc = _lib.SampleCfg(c.cfg, c.interval, c.temp, c.top_k, c.top_p, 1 if c.greedy else 0, 0)
    seeds_d, steps_d = seeds.to(DEV), steps.to(DEV)
    lp = torch.full((B, S), float("nan"), device=DEV)
    rk = torch.full((B, S), -9, dtype=torch.int32, device=DEV)
    tid = torch.full((B, S, N_TOP), -9, dtype=torch.int32, device=DEV)
    tlp = torch.full((B, S, N_TOP), float("nan"), device=DEV)
    spec = _lib.Logprobs(lp.data_ptr(), rk.data_ptr(), tid.data_ptr(), tlp.data_ptr(), N_TOP)
    if V * 8 + 32 * N_TOP * 8 > 200 * 1024:      # the row and its copy outgrow the shared-memory stage (V = 51200)
        with pytest.raises(_lib.LgError, match="with logprobs"):
            _rows_call(lib, logits, B, V, c.mix, c.rd, sc, seeds_d, steps_d, cfg_rows, int_rows, S, spec)
        return
    pick, seq = _rows_call(lib, logits, B, V, c.mix, c.rd, sc, seeds_d, steps_d, cfg_rows, int_rows, S, spec)
    # the same call without logprobs (lg_sample_rows_keyed) draws the same tokens
    ref = torch.full((B, S), -5, dtype=torch.int32, device=DEV)
    ref_idx = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    _lib.check(lib.lg_sample_rows_keyed(_lib.ptr(logits), B, V, int(c.mix), sk.RD[c.rd], ctypes.byref(sc), _lib.ptr(seeds_d),
                                        _lib.ptr(steps_d), _lib.ptr(cfg_rows), _lib.ptr(int_rows), None, _lib.ptr(ref_idx), _lib.ptr(ref), S,
                                        _lib.current_stream(DEV)), "lg_sample_rows_keyed")
    assert torch.equal(pick, ref_idx) and torch.equal(seq, ref)
    # out_probs and the top-k path of the same row (lg_test_sample; a per-row scale is not a test-hook argument)
    probs = path = None
    if variant != "cfg_rows":
        _, probs, path, _ = sk.sample_call(logits, B, V, mix=c.mix, rd=c.rd, cfg_scale=c.cfg, interval=c.interval, temperature=c.temp,
                                           top_k=c.top_k, top_p=c.top_p, greedy=c.greedy, seed=1, step=step)
    pick, lp, rk, tid, tlp = (t.cpu().numpy() for t in (pick, lp, rk, tid, tlp))
    for b in range(B):
        k = int(steps[b])
        mix = sk.mix_on(c.mix and (cfg_rows is None or scales[b] > 1.0), k, int(intervals[b]))
        xs = sk.stage(sk.restate_row(x[b], x[B + b] if c.mix else None, mix, scales[b], c.rd), c.temp)
        keep, amb = sk.ref_filter(xs, c.top_k, c.top_p)
        if probs is not None:
            if c.expect_topk is not None and variant == "own":
                assert path[b, 0] == c.expect_topk, (b, path[b])
            kept = (keep & ~amb) | (amb & (probs[b] > 0))      # the kernel's kept set: the float64 one outside the top-p band
        else:
            kept = keep & ~amb
            if amb.any():
                continue                                        # no out_probs to settle a token in the band
        v = int(pick[b])
        assert kept[v], (b, v)
        ref_lp = lo.logprobs(xs, kept)
        bound = LP_ABS + np.abs(np.where(kept, xs.astype(np.float64), 0) - xs[kept].max()) * 2.0 ** -22
        err = abs(float(lp[b, k]) - ref_lp[v])
        WORST["lp"] = max(WORST["lp"], err)
        assert err <= bound[v], ("logprob", b, lp[b, k], ref_lp[v])
        assert rk[b, k] == lo.rank(xs, kept, v), (b, rk[b, k])
        ids, tl = lo.top(xs, kept, N_TOP)
        assert np.array_equal(tid[b, k], ids), (b, tid[b, k], ids)
        ok = ids >= 0
        assert np.all(np.abs(tlp[b, k][ok] - tl[ok]) <= bound[ids[ok]]) and np.all(np.isneginf(tlp[b, k][~ok])), b
        if c.greedy:
            assert rk[b, k] == 1
        if probs is not None and probs[b, v] > 2.0 ** -100:
            assert abs(math.exp(float(lp[b, k])) - probs[b, v]) <= 1e-5 * probs[b, v], (b, math.exp(float(lp[b, k])), probs[b, v])
        others = np.ones(S, bool)
        others[k] = False
        assert np.isnan(lp[b, others]).all() and (rk[b, others] == -9).all()


def test_kernel_logprob_error_report():
    """The largest logprob error the kernel matrix above saw (it runs first in file order), against LP_ABS."""
    print(f"largest |logprob - float64| over the kernel matrix: {WORST['lp']:.3g} (bound {LP_ABS} + |x - max| 2^-22)")
    assert WORST["lp"] <= 1.0


def test_top_n_bounds_are_refused():
    from llamagen_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(2, 64, device=DEV)
    lp = torch.zeros(2, 1, device=DEV)
    sc = _lib.SampleCfg(1.0, -1, 1.0, 0, 1.0, 0, 0)
    z = torch.zeros(2, dtype=torch.int64, device=DEV)
    for spec in (_lib.Logprobs(lp.data_ptr(), 0, lp.data_ptr(), lp.data_ptr(), 21), _lib.Logprobs(lp.data_ptr(), 0, 0, 0, 3)):
        with pytest.raises(_lib.LgError):
            _lib.check(lib.lg_sample_rows_logprobs(_lib.ptr(x), 2, 64, 0, 0, ctypes.byref(sc), _lib.ptr(z), _lib.ptr(z.int()), None, None,
                                                   None, ctypes.byref(spec), None, _lib.ptr(z.int()), 1, _lib.current_stream(DEV)), "lp")


# ------------------------------------------------------------------------------------------------------------ generate()
def _golden(name, dt, kv="auto"):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], dt)
    if kv != "auto":
        m.set_kv_cache(kv)
    return g, m


def _gen(m, g, B, **kw):
    from llamagen_b200 import generate
    cond = g["cond"][:B].cuda() if m.model_type == "t2i" else (torch.arange(B) % 10).cuda()
    em = g["emb_masks"][:B].cuda() if m.model_type == "t2i" else None
    return generate(m, cond, g["S"], emb_masks=em, **kw)


CASES = [("gpt_c2i.pt", torch.float32, "auto", 1.0, None, 0), ("gpt_c2i.pt", torch.bfloat16, "auto", 4.0, None, 0),
         ("gpt_c2i.pt", torch.bfloat16, "fp8", 4.0, None, 3), ("gpt_t2i.pt", torch.float32, "auto", 4.0, "neg", 0),
         ("gpt_t2i.pt", torch.bfloat16, "auto", 4.0, None, 5), ("gpt_t2i.pt", torch.float16, "fp8", 4.0, "neg", 2),
         ("gpt_t2i.pt", torch.bfloat16, "auto", 1.0, None, 0)]


@pytest.mark.parametrize("name, dt, kv, cfg, neg, P", CASES)
def test_generate_tokens_unchanged_by_logprobs(name, dt, kv, cfg, neg, P):
    g, m = _golden(name, dt, kv)
    B, S = 3, g["S"]
    assert S - P - 2 >= 3      # the captured decode graph runs
    kw = dict(cfg_scale=cfg, cfg_interval=3 if cfg > 1 else -1, temperature=1.0, top_k=100, top_p=0.95, seed=77)
    if neg:
        kw.update(negative_cond=g["cond"][:B].flip(0).cuda())
    if P:
        kw.update(prefix=torch.randint(0, 512, (B, P), generator=torch.Generator().manual_seed(P)))
    base = _gen(m, g, B, **kw).cpu()
    toks, lp = _gen(m, g, B, return_logprobs=True, **kw)
    toks2, lp2, ex = _gen(m, g, B, return_logprobs=True, top_logprobs=7, **kw)
    assert torch.equal(toks.cpu(), base) and torch.equal(toks2.cpu(), base)
    assert torch.equal(lp, lp2)
    lp, ranks, ids, tl = lp.cpu(), ex["ranks"].cpu(), ex["top_ids"].cpu(), ex["top_logprobs"].cpu()
    if P:
        assert (lp[:, :P] == 0).all() and (ranks[:, :P] == 0).all() and (ids[:, :P] == -1).all() and torch.isneginf(tl[:, :P]).all()
    lp, ranks, ids, tl, tk = lp[:, P:], ranks[:, P:], ids[:, P:], tl[:, P:], base[:, P:]
    assert (lp <= 0).all() and (ranks >= 1).all() and (ranks <= 100).all()
    # the alternative at the drawn token's rank has its logprob: it is the token itself, or a tie of it with a lower id
    inside = ranks <= 7
    at = tl.gather(2, (ranks.clamp(1, 7) - 1).long().unsqueeze(2)).squeeze(2)
    assert torch.equal(at[inside], lp[inside])
    assert (tl[..., :-1] >= tl[..., 1:]).all()


def test_two_chains_give_the_same_tokens_and_logprobs(monkeypatch):
    outs = {}
    for split in ("1", "2"):
        monkeypatch.setenv("LG_SPLIT", split)
        g, m = _golden("gpt_c2i.pt", torch.bfloat16)
        from llamagen_b200 import generate
        cond = torch.randint(0, 10, (48,), generator=torch.Generator().manual_seed(3)).cuda()
        kw = dict(cfg_scale=4.0, temperature=1.0, top_k=50, seed=5)
        plain = generate(m, cond, g["S"], **kw).cpu()
        toks, lp, ex = generate(m, cond, g["S"], return_logprobs=True, top_logprobs=3, **kw)
        assert torch.equal(toks.cpu(), plain)
        outs[split] = (toks.cpu(), lp.cpu(), ex["top_ids"].cpu(), ex["top_logprobs"].cpu(), ex["ranks"].cpu())
    for a, b in zip(outs["1"], outs["2"]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------ score()
@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg", [1.0, 4.0])
def test_generate_logprobs_equal_minus_score(name, cfg):
    from llamagen_b200 import score
    res = {}
    for dt in (torch.float32, torch.bfloat16):
        g, m = _golden(name, dt)
        B = 4
        toks, lp = _gen(m, g, B, cfg_scale=cfg, temperature=1.0, top_k=0, top_p=1.0, seed=11, return_logprobs=True)
        cond = g["cond"][:B].cuda() if m.model_type == "t2i" else (torch.arange(B) % 10).cuda()
        em = g["emb_masks"][:B].cuda() if m.model_type == "t2i" else None
        res[dt] = (m, cond, em, toks, lp.cpu(), g)
    m32, cond, em, toks, lp32, _ = res[torch.float32]
    err32 = (lp32 + score(m32, cond, toks.long(), emb_masks=em, cfg_scale=cfg).cpu()).abs().max().item()
    assert err32 <= 1e-3, err32
    m16, cond, em, toks16, lp16, _ = res[torch.bfloat16]
    nll16 = score(m16, cond, toks16.long(), emb_masks=em, cfg_scale=cfg).cpu()
    spread = (nll16 - score(m32, cond, toks16.long(), emb_masks=em, cfg_scale=cfg).cpu()).abs().max().item()
    err16 = (lp16 + nll16).abs().max().item()
    print(f"{name} cfg {cfg}: fp32 |lp + nll| {err32:.3g}; bf16 {err16:.3g} against bf16-vs-fp32 score spread {spread:.3g}")
    assert err16 <= 3 * spread + 1e-3, (err16, spread)


# ------------------------------------------------------------------------------------------------------------ serve.LLM
def _ref(m, cond, em, S, sp, scale, interval, seed, k, prefix=None, N=None, **kw):
    """generate() of cond repeated k times with a request's parameters: (tokens, lp, extras) on the host."""
    from llamagen_b200 import generate
    rep = (lambda t: None if t is None else t.expand(k, *t.shape[1:]).contiguous())
    pf = None if prefix is None else torch.as_tensor(prefix)[None].expand(k, -1)
    out = generate(m, rep(cond).cuda(), S, emb_masks=None if em is None else rep(em).cuda(), cfg_scale=scale, cfg_interval=interval,
                   temperature=sp.temperature, top_k=max(0, sp.top_k), top_p=sp.top_p, seed=seed, prefix=pf, return_logprobs=True,
                   top_logprobs=N or 1, **kw)
    return out[0].cpu(), out[1].cpu(), {k_: v.cpu() for k_, v in out[2].items()}


def _check_output(o, ref, sp, P, images=None):
    toks, lp, ex = ref
    images = list(range(len(o.outputs))) if images is None else images
    assert [c.index for c in o.outputs] == images
    for c in o.outputs:
        j = c.index
        assert c.token_ids == toks[j].tolist(), j
        want = float(np.sum(lp[j, P:].numpy().astype(np.float64)))
        assert abs(c.cumulative_logprob - want) <= 1e-4 * max(1.0, abs(want)), (c.cumulative_logprob, want)
        if sp.logprobs is not None:
            ref_d = lo.completion_logprobs(toks[j].tolist(), lp[j].numpy(), ex["ranks"][j].numpy(), ex["top_ids"][j].numpy(),
                                           ex["top_logprobs"][j].numpy(), sp.logprobs, P)
            assert len(c.logprobs) == len(ref_d)
            for k, (d, r) in enumerate(zip(c.logprobs, ref_d)):
                if r is None:
                    assert d is None
                    continue
                assert set(d) == set(r), (k, d, r)
                for t in d:
                    assert d[t].rank == r[t][1] and abs(d[t].logprob - r[t][0]) <= 1e-4, (k, t, d[t], r[t])


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_serve_logprobs_equal_generate_fp32(kind):
    from llamagen_b200.serve import LLM, SamplingParams as SP
    from test_serve_t2i_gpu import _captions
    g, m = _golden(f"gpt_{kind}.pt", torch.float32)
    S, slots = g["S"], 4
    llm = LLM(m, cfg_scale=4.0, num_classes=10, max_num_seqs=slots, seed=21)
    conds = [3, 7, 1, 5, 9] if kind == "c2i" else _captions([40, 120, 7, 64, 90], 64, 5)
    params = [SP(max_tokens=S, top_k=100, logprobs=5), SP(max_tokens=S, top_k=100, logprobs=0, cfg_scale=2.5, cfg_interval=4, seed=99),
              SP(max_tokens=S, top_k=100), SP(max_tokens=S, top_k=100, n=2, logprobs=3, seed=7),
              SP(max_tokens=S, top_k=100, logprobs=20, seed=3)]
    prefixes = [None, None, None, None, [5, 6, 7]]
    ids, outs = [], {}

    def add(i):
        kw = dict(prompt_embeds=conds[i]) if kind == "t2i" else dict(prompt_token_ids=[conds[i]])
        rid = llm.add_request(sampling_params=params[i], prefix=prefixes[i], **kw)
        if kind == "c2i" and i == 0:     # a null-class twin mirrors request 0
            ids.append(llm.add_request(prompt_token_ids=[10], sampling_params=params[i], twin_of=rid))
        return rid

    rids = [add(0), add(1)]
    for _ in range(3):
        outs.update({o.request_id: o for o in llm.step()})
    rids += [add(2), add(3), add(4)]
    while llm.has_unfinished_requests():
        outs.update({o.request_id: o for o in llm.step()})
    from test_serve_prefix_gpu import _oracle_cond
    for i, rid in enumerate(rids):
        sp, req_seed = params[i], (21 + int(rid) if params[i].seed is None else params[i].seed)
        cond, em = _oracle_cond(llm, conds[i])
        scale = 4.0 if sp.cfg_scale is None else sp.cfg_scale
        interval = -1 if sp.cfg_interval is None else sp.cfg_interval
        P = len(prefixes[i]) if prefixes[i] else 0
        ref = _ref(m, cond, em, S, sp, scale, interval, req_seed, max(sp.n, slots) if kind == "c2i" else sp.n, prefixes[i],
                   sp.logprobs)
        o = outs[rid]
        if sp.logprobs is None:
            assert all(c.logprobs is None and c.cumulative_logprob is None for c in o.outputs)
            assert [c.token_ids for c in o.outputs] == [ref[0][j].tolist() for j in range(sp.n)]
        else:
            _check_output(o, ref, sp, P)
    if ids:
        twin = outs[ids[0]]
        assert [(c.token_ids, c.logprobs, c.cumulative_logprob) for c in twin.outputs] == \
            [(c.token_ids, c.logprobs, c.cumulative_logprob) for c in outs[rids[0]].outputs]


def test_serve_best_of_returns_the_largest_cumulative_logprobs():
    from llamagen_b200.serve import LLM, SamplingParams as SP
    g, m = _golden("gpt_c2i.pt", torch.float32)
    S = g["S"]
    llm = LLM(m, cfg_scale=4.0, num_classes=10, max_num_seqs=6, seed=4)
    sp = SP(max_tokens=S, top_k=50, n=2, best_of=5, seed=123, logprobs=2)
    rid = llm.add_request([4], sp)
    outs = {}
    while llm.has_unfinished_requests():
        outs.update({o.request_id: o for o in llm.step()})
    o = outs[rid]
    toks, lp, ex = _ref(m, torch.tensor([4]), None, S, sp, 4.0, -1, 123, 6, N=2)
    sums = lp[:5].double().sum(1)
    order = sorted(range(5), key=lambda j: (-float(sums[j]), j))[:2]
    _check_output(o, (toks, lp, ex), sp, 0, images=order)
    assert o.outputs[0].cumulative_logprob >= o.outputs[1].cumulative_logprob


def test_serve_fp8_weights_logprobs_equal_generate():
    from llamagen_b200.serve import LLM, SamplingParams as SP
    from test_weight_fp8_gpu import _gpt_b
    gpt = _gpt_b()
    S, slots = 32, 4
    sp = SP(temperature=1.0, top_k=2000, max_tokens=S, logprobs=4)
    llm = LLM(gpt, cfg_scale=4.0, num_classes=1000, max_num_seqs=slots, seed=11, weight_dtype="fp8")
    outs = {}
    llm.add_request([207], sp)
    outs.update({o.request_id: o for o in llm.step()})
    llm.add_request([360], sp)
    while llm.has_unfinished_requests():
        outs.update({o.request_id: o for o in llm.step()})
    for rid, c in enumerate([207, 360]):
        ref = _ref(gpt, torch.tensor([c]), None, S, sp, 4.0, -1, 11 + rid, slots, N=4)
        _check_output(outs[str(rid)], ref, sp, 0)
