"""GPU: per-request guidance and seeds in serve.LLM (SamplingParams(cfg_scale=, cfg_interval=, seed=)) and lg_sample_rows_guided.

* Kernel: random logits [2B, 16384], B in {1, 8, 64}, per-row scales in {0.5, 1.0, 1.5, 4.0, 7.5}, intervals in {-1, 0, 3, 10**6},
  assorted steps and seeds, round dtype f32 / bf16 / f16, top-k and top-p on and off, sampled and greedy: every row's id equals a
  separate lg_sample_rows call with that row's scalar config (mix_cfg iff its scale is > 1), seed and step, bit for bit; greedy ids
  equal the sampling oracle's after cfg_mix_oracle.
* Schedule independence, c2i and t2i, in bf16, fp16 and bf16 with an fp8 KV cache (c2i also with fp8 weights): a mixed batch of
  scales {1.0, 2.0, 4.0, 7.5} with intervals and explicit seeds, more requests than slots, prefixes (and on t2i negative prompts)
  among them; every request's tokens equal those of the request run alone in an LLM of the same max_num_seqs (for a scale c > 1 an
  LLM built with cfg_scale c and no per-request scale).
* fp32 greedy on the golden models: every request of a mixed batch equals GPTOracle.generate(cfg_scale=c_i, cfg_interval=k_i,
  sample_logits=False).
* Seed: with one slot at cfg 1.0, SamplingParams(seed=s) gives generate(seed=s)'s tokens bit for bit, sampled."""
import ctypes

import numpy as np
import pytest
import torch

from test_serve_prefix_gpu import C2I, _oracle_cond, _prefix
from test_serve_t2i_gpu import XL3, _captions, _model
from util import build_gpt, load_golden

pytestmark = pytest.mark.gpu

V = 16384
RD = {"f32": 0, "bf16": 1, "f16": 2}
FILTERS = [dict(top_k=0, top_p=1.0, greedy=0), dict(top_k=1000, top_p=1.0, greedy=0), dict(top_k=0, top_p=0.9, greedy=0),
           dict(top_k=500, top_p=0.8, greedy=0), dict(top_k=0, top_p=1.0, greedy=1), dict(top_k=200, top_p=0.9, greedy=1)]


def _rows(B, seed):
    g = torch.Generator().manual_seed(seed)
    scales = torch.tensor([0.5, 1.0, 1.5, 4.0, 7.5])[torch.randint(0, 5, (B,), generator=g)]
    intervals = torch.tensor([-1, 0, 3, 10 ** 6], dtype=torch.int32)[torch.randint(0, 4, (B,), generator=g)]
    steps = torch.randint(0, 12, (B,), generator=g, dtype=torch.int32)
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64)
    if B >= 4:                       # the step-0 draw and both sides of the interval-3 boundary
        steps[:4] = torch.tensor([0, 1, 4, 5], dtype=torch.int32)
    return scales, intervals, steps, seeds


@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("B", [1, 8, 64])
def test_guided_rows_equal_their_scalar_calls(B, rd):
    from llamagen_b200 import _lib
    from oracle.sampling_oracle import cfg_mix_oracle, sample_oracle
    lib = _lib.load()
    stream = _lib.current_stream("cuda")
    g = torch.Generator().manual_seed(1000 * B + RD[rd])
    x = (3.0 * torch.randn(2 * B, V, generator=g)).cuda()
    scales, intervals, steps, seeds = _rows(B, B + 7 * RD[rd])
    cfg_d, int_d, step_d, seed_d = scales.cuda(), intervals.cuda(), steps.cuda(), seeds.cuda()
    for f in FILTERS:
        sc = _lib.SampleCfg(99.0, 1, 1.0, f["top_k"], f["top_p"], f["greedy"], 0)    # scale and interval are the rows'
        got = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        _lib.check(lib.lg_sample_rows_guided(_lib.ptr(x), B, V, 1, RD[rd], ctypes.byref(sc), _lib.ptr(seed_d), _lib.ptr(step_d),
                                             _lib.ptr(cfg_d), _lib.ptr(int_d), _lib.ptr(got), None, 0, stream), "lg_sample_rows_guided")
        want = torch.full((B,), -1, dtype=torch.int32, device="cuda")
        for b in range(B):
            s, k = float(scales[b]), int(intervals[b])
            one = torch.stack([x[b], x[B + b]]).contiguous()        # [cond; uncond] of image b alone
            sc1 = _lib.SampleCfg(s, k, 1.0, f["top_k"], f["top_p"], f["greedy"], 0)
            _lib.check(lib.lg_sample_rows(_lib.ptr(one), 1, V, int(s > 1.0), RD[rd], ctypes.byref(sc1), _lib.ptr(seed_d[b:b + 1]),
                                          _lib.ptr(step_d[b:b + 1]), _lib.ptr(want[b:b + 1]), None, 0, stream), "lg_sample_rows")
        got, want = got.cpu(), want.cpu()
        assert torch.equal(got, want), (f, (got != want).nonzero().flatten().tolist())
        if f["greedy"]:
            xr = x.cpu() if rd == "f32" else x.cpu().to(torch.bfloat16 if rd == "bf16" else torch.float16).float()
            for b in range(B):
                s, k, st = float(scales[b]), int(intervals[b]), int(steps[b])
                mix = s > 1.0 and not (k > -1 and st >= 1 and st - 1 > k)
                row = cfg_mix_oracle(torch.stack([xr[b], xr[B + b]]), s) if mix else xr[b:b + 1]
                idx, probs = sample_oracle(row, top_k=f["top_k"], top_p=f["top_p"], sample_logits=False)
                o = int(idx[0, 0])
                assert int(got[b]) == o or probs[0, int(got[b])] == probs[0, o], (f, b, int(got[b]), o)


# ------------------------------------------------------------------------------------------------------------ serving
GUIDES = [(1.0, -1, 11), (2.0, 3, 22), (4.0, -1, 33), (7.5, 0, 44), (7.5, 10, 55), (2.0, -1, 66), (1.0, 5, 77)]


def _add(llm, cond, sp, prefix=None, neg=None):
    if llm.t2i:
        return llm.add_request(prompt_embeds=cond, sampling_params=sp, prefix=prefix, negative_prompt_embeds=neg)
    return llm.add_request([cond], sp, prefix=prefix)


def _run(llm, reqs, waves):
    """reqs: [(cond, SamplingParams, prefix, negative)]; waves: [(steps to run before the wave, [request indices])]. Request ids follow
    the indices. Returns {index: tokens}."""
    llm.request_counter = iter([i for _, w in waves for i in w])
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            _add(llm, *reqs[i])
    while llm.has_unfinished_requests():
        outs += llm.step()
    return {int(o.request_id): o.outputs[0].token_ids for o in outs}


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("dt, kv, w", [(torch.bfloat16, "auto", "auto"), (torch.float16, "auto", "auto"), (torch.bfloat16, "fp8", "auto"),
                                       (torch.bfloat16, "auto", "fp8")], ids=["bf16", "f16", "bf16_kv_fp8", "bf16_w_fp8"])
def test_each_request_draws_what_it_draws_alone(kind, dt, kv, w):
    from llamagen_b200.serve import LLM, SamplingParams
    if kind == "t2i":
        if w == "fp8":
            pytest.skip("fp8 weights: covered on the c2i shape")
        m, S = _model(dt, kv, **XL3), 24
        conds = _captions([5, 37, 64, 120, 17, 90, 1], XL3["caption_dim"], 11)
        negs = [None, _captions([9], XL3["caption_dim"], 3)[0], None, _captions([120], XL3["caption_dim"], 4)[0], None, None, None]
        Ps = [0, 0, 10, 3, 0, 0, 23]
    else:
        m, S = _model(dt, kv, **C2I), 32
        if w == "fp8":
            m.set_weight_dtype("fp8")
        conds, negs, Ps = [207, 360, 387, 974, 88, 979, 417], [None] * 7, [0, 5, 0, 0, 31, 0, 2]
    base = 4.0
    reqs = []
    for i, (c, k, s) in enumerate(GUIDES):
        sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, cfg_scale=c, cfg_interval=k, seed=s * 1000 + 7)
        reqs.append((conds[i], sp, _prefix(Ps[i], m.vocab_size, 50 + i), negs[i] if c > 1.0 else None))
    n = len(reqs)
    got = _run(LLM(m, cfg_scale=base, max_num_seqs=3, seed=5), reqs, [(0, [0, 1, 2, 3]), (4, [4, 5]), (9, [6])])
    assert sorted(got) == list(range(n)) and all(len(t) == S for t in got.values())
    assert len({tuple(t) for t in got.values()}) == n
    for i, (cond, sp, pf, neg) in enumerate(reqs):
        if sp.cfg_scale > 1.0:     # an LLM built with the request's scale, the request without one of its own
            alone = LLM(m, cfg_scale=sp.cfg_scale, max_num_seqs=3, seed=5)
            sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, cfg_interval=sp.cfg_interval, seed=sp.seed)
        else:
            alone = LLM(m, cfg_scale=base, max_num_seqs=3, seed=5)
        ref = _run(alone, [(cond, sp, pf, neg)], [(0, [0])])[0]
        assert ref == got[i], f"request {i} (cfg {GUIDES[i][0]}, interval {GUIDES[i][1]}, P {Ps[i]})"


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_fp32_greedy_equals_oracle_per_request(name):
    from llamagen_b200.serve import LLM, SamplingParams
    from oracle import GPTOracle
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    S = g["S"]
    t2i = m.model_type == "t2i"
    conds = _captions([5, 37, 64, 120, 9, 88, 17], g["cfg"]["caption_dim"], 7) if t2i else [1, 2, 3, 4, 5, 6, 7]
    guides = [(4.0, -1), (1.0, -1), (7.5, 3), (2.0, 0), (0.5, 2), (7.5, -1), (4.0, 1)]
    reqs = [(c, SamplingParams(temperature=1.0, top_k=1, max_tokens=S, cfg_scale=s, cfg_interval=k), None, None)
            for c, (s, k) in zip(conds, guides)]
    llm = LLM(m, cfg_scale=4.0, num_classes=g["cfg"]["num_classes"], max_num_seqs=3, seed=3)
    got = _run(llm, reqs, [(0, [0, 1]), (3, [2, 3, 4]), (S + 5, [5, 6])])
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for i, (c, (s, k)) in enumerate(zip(conds, guides)):
        cond, em = _oracle_cond(llm, c)
        want, _ = orc.generate(cond, S, emb_masks=em, cfg_scale=s, cfg_interval=k, sample_logits=False)
        assert got[i] == want[0].tolist(), f"request {i} (cfg {s}, interval {k})"


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_seed_is_generate_seed_bit_for_bit(kind):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    if kind == "t2i":
        m, S, conds = _model(torch.bfloat16, **XL3), 32, _captions([5, 120, 64], XL3["caption_dim"], 9)
    else:
        m, S, conds = _model(torch.bfloat16, **C2I), 64, [207, 360, 387]
    seeds = [123456789, 0, 2 ** 63 - 1]
    reqs = [(c, SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, seed=s), None, None) for c, s in zip(conds, seeds)]
    llm = LLM(m, cfg_scale=1.0, max_num_seqs=1, seed=40)
    got = _run(llm, reqs, [(0, [0, 1, 2])])
    for r, (c, s) in enumerate(zip(conds, seeds)):
        cond, em = _oracle_cond(llm, c)
        ref = generate(m, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), cfg_scale=1.0, temperature=1.0, top_k=1000, seed=s)
        assert ref[0].cpu().tolist() == got[r], f"request {r} (seed {s})"
