"""GPU: per-image temperature, top-k, top-p and greedy (lg_sample_cfg's row arrays) from the kernel up to serve.LLM.

* Kernel: B rows over the grid top_k in {0, 1, 7, 2000, V, V + 5} x temperature in {1.0, 0.7, 1.3, 0} x top_p in {1.0, 0.9, 0.0}, greedy
  mixed in, f32 / bf16 / f16 rounding, CFG on and off, through lg_sample_rows_keyed, _logprobs, _given, _composed (a table of plain
  rows), lg_sample and lg_test_sample (with dbg_path), and lg_test_sample_groups. A row with top_p = 1 equals a one-row call with its
  values as scalars bit for bit (token, logprob, rank, top ids); a row with top_p < 1 keeps the float64 restatement's set and
  probabilities within the bands of test_sample_kernel_gpu (nucleus draws use float atomics and are not bit-reproducible).
* generate(): on tiny c2i and t2i models image b of a per-image call equals image b of the scalar call with value b, bit for bit, on the
  plain, CFG, prefix, given, negative, cond_weights, logprobs and sjd_window paths, in bf16, fp16 and with an fp8 KV cache.
* serve.LLM(per_request_sampling=True): a mixed stream of c2i and t2i requests, each with its own filters (guidance, seeds, n, logprobs,
  prefixes, given tokens, cond_weights and negatives among them; a t2i request at temperature 0 beside sampled ones), and an SJD LLM:
  every request draws what it draws alone in an LLM without the flag."""
import ctypes

import numpy as np
import pytest
import torch

from test_sample_kernel_gpu import ref_filter, restate_row, stage
from test_serve_prefix_gpu import C2I, _prefix
from test_serve_t2i_gpu import XL3, _captions, _model

pytestmark = pytest.mark.gpu

V = 16384
RD = {"f32": 0, "bf16": 1, "f16": 2}
TOPK = [0, 1, 7, 2000, V, V + 5]
TEMP = [1.0, 0.7, 1.3, 0.0]
TOPP = [1.0, 0.9, 0.0]


def P(t):
    from llamagen_b200 import _lib
    return _lib.ptr(t)


def _grid():
    """Per-row (top_k, temperature, top_p, greedy): every combination of the grid, every fifth row greedy."""
    rows = [(k, t, p) for k in TOPK for t in TEMP for p in TOPP]
    return [(k, t, p, int(i % 5 == 3)) for i, (k, t, p) in enumerate(rows)]


def _cfg(rows, dev="cuda", scale=1.0):
    """SampleCfg with the scalars at values no row has (they must not be read) and the row arrays, plus the device arrays."""
    from llamagen_b200 import _lib
    arr = (torch.tensor([r[1] for r in rows], dtype=torch.float32, device=dev), torch.tensor([r[0] for r in rows], dtype=torch.int32, device=dev),
           torch.tensor([r[2] for r in rows], dtype=torch.float32, device=dev), torch.tensor([r[3] for r in rows], dtype=torch.int32, device=dev))
    sc = _lib.SampleCfg(scale, -1, 5.0, 3, 0.5, 0, 0, *(a.data_ptr() for a in arr))
    return sc, arr


def _scalar(r, scale=1.0):
    from llamagen_b200 import _lib
    k, t, p, g = r
    return _lib.SampleCfg(scale, -1, t, k, p, g, 0)


def _logits(B, mix, rd, seed):
    g = torch.Generator().manual_seed(seed)
    return (3.0 * torch.randn((2 if mix else 1) * B, V, generator=g)).cuda()


def _one(x, b, B, mix):
    return (torch.stack([x[b], x[B + b]]) if mix else x[b:b + 1]).contiguous()


def _check_nucleus(x, b, B, mix, rd, r, pick, probs=None):
    """A top_p < 1 row: pick lies in the float64 kept set (or its ambiguity band); probs (when given) keep that set and agree with the
    renormalised float64 probabilities."""
    k, t, p, g = r
    xc = x[b].cpu().numpy()
    xu = x[B + b].cpu().numpy() if mix else None
    xs = stage(restate_row(xc, xu, mix, 4.0 if mix else 1.0, rd), t)
    keep, amb = ref_filter(xs, k, p)
    assert keep[pick] or amb[pick], (r, pick)
    if g:
        assert xs[pick] == xs[keep].max() or amb[pick], (r, pick)
    if probs is not None:
        kern = probs > 0
        assert np.all(kern[keep & ~amb]) and not np.any(kern & ~(keep | amb)), r
        e = np.where(kern, np.exp(xs.astype(np.float64) - xs[kern].max()), 0.0)
        assert np.allclose(probs, e / e.sum(), rtol=1e-4, atol=1e-6), r


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "cfg"])
@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
def test_rows_equal_their_scalar_calls(rd, mix):
    from llamagen_b200 import _lib
    lib, st = _lib.load(), _lib.current_stream("cuda")
    rows = _grid()
    B = len(rows)
    x = _logits(B, mix, rd, 17 * RD[rd] + mix)
    g = torch.Generator().manual_seed(5 + RD[rd])
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64).cuda()
    steps = torch.randint(0, 9, (B,), generator=g, dtype=torch.int32).cuda()
    img = torch.randint(0, 4, (B,), generator=g, dtype=torch.int32).cuda()
    given = torch.full((B, 16), -1, dtype=torch.int32, device="cuda")
    given[::7, :] = 11                                                   # some rows take a given token instead of their draw
    scale = 4.0 if mix else 1.0
    sc, keep = _cfg(rows, scale=scale)
    N = 20

    def lp_bufs(n):
        return (torch.zeros(n, 16, device="cuda"), torch.zeros(n, 16, dtype=torch.int32, device="cuda"),
                torch.zeros(n, 16, N, dtype=torch.int32, device="cuda"), torch.zeros(n, 16, N, device="cuda"))

    def run(entry, cfg, sl, logits, n):
        """One call of `entry` over rows sl (n rows) of the per-row inputs: (tokens, logprob rows or None)."""
        out = torch.full((n,), -9, dtype=torch.int32, device="cuda")
        seq = torch.full((n, 16), -9, dtype=torch.int32, device="cuda")
        lp = lp_bufs(n) if entry in ("logprobs", "composed") else None
        spec = _lib.Logprobs(*(t.data_ptr() for t in lp), N) if lp else None
        head = (P(logits), n, V, int(mix), RD[rd], ctypes.byref(cfg), P(seeds[sl]), P(steps[sl]))
        if entry == "keyed":
            _lib.check(lib.lg_sample_rows_keyed(*head, None, None, P(img[sl]), P(out), P(seq), 16, st), entry)
        elif entry == "logprobs":
            _lib.check(lib.lg_sample_rows_logprobs(*head, None, None, P(img[sl]), ctypes.byref(spec), P(out), P(seq), 16, st), entry)
        elif entry == "given":
            _lib.check(lib.lg_sample_rows_given(*head, None, None, P(img[sl]), P(given[sl]), None, P(out), P(seq), 16, st), entry)
        else:   # composed: a gather table of plain rows (the grouped instantiation, one CTA per row)
            tab = torch.full((n, 1 + _lib.MAX_COMPOSE), -1, dtype=torch.int32, device="cuda")
            w = torch.zeros(n, _lib.MAX_COMPOSE, device="cuda")
            lgt = logits if mix else torch.cat([logits, logits]).contiguous()
            _lib.check(lib.lg_sample_rows_composed(P(lgt), 2 * n, n, V, RD[rd], ctypes.byref(cfg), P(seeds[sl]), P(steps[sl]), None, None,
                                                   P(img[sl]), None, P(tab), P(w), ctypes.byref(spec), P(out), P(seq), 16, st), entry)
        torch.cuda.synchronize()
        return out.cpu(), None if lp is None else [t.cpu() for t in lp]

    for entry in ("keyed", "logprobs", "given", "composed"):
        got, glp = run(entry, sc, slice(0, B), x, B)
        for b, r in enumerate(rows):
            if entry == "given" and b % 7 == 0:
                assert int(got[b]) == 11, (entry, b)
                continue
            if r[2] < 1.0:
                _check_nucleus(x, b, B, mix, rd, r, int(got[b]))   # composed without CFG mixes u = c: the plain row
                continue
            one, olp = run(entry, _scalar(r, scale), slice(b, b + 1), _one(x, b, B, mix), 1)
            assert int(got[b]) == int(one[0]), (entry, rd, mix, b, r)
            if glp is not None:
                s = int(steps[b])
                for t, o in zip(glp, olp):
                    assert torch.equal(t[b, s], o[0, s]), (entry, b, r)

    # lg_sample and lg_test_sample: the call's stream keys (image b keys as row b + 1), probabilities and dbg_path per row
    idx = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    pr = torch.empty(B, V, device="cuda")
    _lib.check(lib.lg_sample(P(x), B, V, int(mix), RD[rd], ctypes.byref(sc), 3, P(idx), P(pr), st), "lg_sample")
    path = torch.full((B, 3), -1, dtype=torch.int32, device="cuda")
    tidx = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    vec = ctypes.c_int(-1)

    def test_sample(cfg, logits, n, row_offset, out, pa, probs=None):
        _lib.check(lib.lg_test_sample(P(logits), n, V, int(mix), RD[rd], ctypes.byref(cfg), 3, None, row_offset, None, None, P(out), P(probs),
                                      None, 0, None, None, None, 0, None, None, None, None, ctypes.c_float(0.0), 0, 0, None, None, P(pa),
                                      ctypes.byref(vec), st), "lg_test_sample")
    test_sample(sc, x, B, 0, tidx, path)
    torch.cuda.synchronize()
    idx, pr, tidx, path = idx.cpu(), pr.cpu().numpy(), tidx.cpu(), path.cpu()
    for b, r in enumerate(rows):
        if r[2] < 1.0:
            _check_nucleus(x, b, B, mix, rd, r, int(idx[b]), pr[b])
            assert path[b, 0] == (0 if r[0] <= 0 or r[0] >= V else path[b, 0]), (b, r)
            continue
        o, opr = torch.full((1,), -9, dtype=torch.int32, device="cuda"), torch.empty(1, V, device="cuda")
        opa = torch.full((1, 3), -1, dtype=torch.int32, device="cuda")
        test_sample(_scalar(r, scale), _one(x, b, B, mix), 1, b, o, opa, opr)
        torch.cuda.synchronize()
        assert int(idx[b]) == int(o[0]) == int(tidx[b]), ("lg_sample", rd, mix, b, r)
        assert np.array_equal(pr[b], opr[0].cpu().numpy()), ("probs", b, r)
        assert torch.equal(path[b], opa[0].cpu()), ("dbg_path", b, r, path[b].tolist(), opa[0].tolist())
        assert path[b, 2] == (0 if r[3] else path[b, 2]) and (r[3] or path[b, 2] in (1, 2)), (b, r)


@pytest.mark.parametrize("rd", ["f32", "bf16"])
def test_groups_take_rows_per_image(rd):
    from llamagen_b200 import _lib
    lib, st = _lib.load(), _lib.current_stream("cuda")
    rows = [r for r in _grid() if r[2] == 1.0]
    B, K = len(rows), 2
    g = torch.Generator().manual_seed(3)
    x = (3.0 * torch.randn(2 * B * K, V, generator=g)).cuda()
    w = torch.tensor([[4.0, -1.5]] * B, device="cuda")
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64).cuda()
    steps = torch.randint(0, 9, (B,), generator=g, dtype=torch.int32).cuda()
    sc, keep = _cfg(rows)
    got = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    _lib.check(lib.lg_test_sample_groups(P(x), B, K, V, RD[rd], ctypes.byref(sc), P(w), P(seeds), P(steps), P(got), None, st), "groups")
    for b, r in enumerate(rows):
        one = torch.cat([x[b * K:(b + 1) * K], x[B * K + b * K:B * K + (b + 1) * K]]).contiguous()
        o = torch.full((1,), -9, dtype=torch.int32, device="cuda")
        _lib.check(lib.lg_test_sample_groups(P(one), 1, K, V, RD[rd], ctypes.byref(_scalar(r)), P(w[b]), P(seeds[b:b + 1]),
                                             P(steps[b:b + 1]), P(o), None, st), "groups")
        assert int(got[b]) == int(o[0]), (b, r)


# ------------------------------------------------------------------------------------------------------------ generate()
def _c2i(dt, kv="auto"):
    return _model(dt, kv, **C2I)


CASES = {
    "c2i_cfg_bf16": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0)),
    "c2i_plain_f16": dict(kind="c2i", dt=torch.float16, kw=dict()),
    "c2i_cfg_kv_fp8": dict(kind="c2i", dt=torch.bfloat16, kv="fp8", kw=dict(cfg_scale=4.0, cfg_interval=5)),
    "c2i_prefix": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0), prefix=5),
    "c2i_given": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0), given=True),
    "c2i_logprobs": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0, return_logprobs=True, top_logprobs=5)),
    "c2i_compose": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cond_weights=[4.0, -1.0]), compose=True),
    "c2i_sjd": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0, sjd_window=4)),
    "c2i_sjd_greedy": dict(kind="c2i", dt=torch.bfloat16, kw=dict(sjd_window=4, sample_logits=False)),
    "c2i_teacher": dict(kind="c2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0), teacher=True),
    "t2i_negative": dict(kind="t2i", dt=torch.bfloat16, kw=dict(cfg_scale=4.0), negative=True),
    "t2i_plain": dict(kind="t2i", dt=torch.bfloat16, kw=dict()),
}
_MODELS = {}


@pytest.mark.parametrize("case", sorted(CASES))
def test_generate_image_b_is_the_scalar_call_with_value_b(case):
    from llamagen_b200 import generate
    c = CASES[case]
    key = (c["kind"], c["dt"], c.get("kv", "auto"))
    if key not in _MODELS:
        _MODELS.clear()
        _MODELS[key] = _c2i(c["dt"], key[2]) if c["kind"] == "c2i" else _model(c["dt"], key[2], **XL3)
    m = _MODELS[key]
    S, B = 20, 4
    temps, topks, topps = [1.0, 0.7, 1.3, 0.0], [2000, 7, V + 5, 0], [1.0] * B
    kw = dict(c["kw"], seed=1234)
    if c["kind"] == "c2i":
        cond = torch.tensor([207, 360, 387, 974], device="cuda")
        if c.get("compose"):
            cond = torch.tensor([[207, 1], [360, 2], [387, 3], [974, 4]], device="cuda")
    else:
        caps = _captions([5, 37, 64, 120], XL3["caption_dim"], 3)
        from llamagen_b200.cond import pack_t5_features, prepare_condition
        embs, masks = pack_t5_features([torch.from_numpy(f[0]) for f in caps], max_len=XL3["cls_token_num"], dim=XL3["caption_dim"])
        cond, em = prepare_condition(embs, masks, left_padding=True)
        cond, kw["emb_masks"] = cond.cuda(), em.cuda()
        if c.get("negative"):
            ne, nmk = pack_t5_features([torch.from_numpy(_captions([9], XL3["caption_dim"], 4)[0][0])], max_len=XL3["cls_token_num"], dim=XL3["caption_dim"])
            nc, nm = prepare_condition(ne, nmk, left_padding=True)
            kw["negative_cond"], kw["negative_emb_masks"] = nc.cuda(), nm.cuda()
    if c.get("prefix"):
        kw["prefix"] = torch.stack([_prefix(c["prefix"], V, 9 + b) for b in range(B)]).cuda()
    if c.get("given"):
        gv = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(8))
        mask = torch.zeros(B, S, dtype=torch.bool)
        mask[:, 3:6] = True
        mask[1, 10:14] = True
        kw["given"], kw["given_mask"] = gv.cuda(), mask.cuda()
    if c.get("teacher"):
        kw["teacher"] = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(9)).cuda()
    tens = [torch.tensor(temps), np.array(topks), topps]   # a tensor, an array and a list
    got = generate(m, cond, S, temperature=tens[0], top_k=tens[1], top_p=tens[2], **kw)
    for b in range(B):
        want = generate(m, cond, S, temperature=temps[b], top_k=topks[b], top_p=topps[b], **kw)
        if isinstance(got, tuple):
            assert torch.equal(got[0][b], want[0][b]) and torch.equal(got[1][b], want[1][b]), (case, b)
            for k in got[2]:
                assert torch.equal(got[2][k][b], want[2][k][b]), (case, b, k)
        else:
            assert torch.equal(got[b], want[b]), (case, b, (got[b] != want[b]).nonzero().flatten().tolist())


def test_sample_rows():
    from llamagen_b200.generate import sample
    x = _logits(8, False, "f32", 4).view(8, 1, V)
    temps, ks = [1.0, 0.7, 1.3, 0.0] * 2, [0, 1, 7, 2000, V, V + 5, 3, 0]
    idx, probs = sample(x, temperature=temps, top_k=ks, top_p=1.0, seed=77)
    for b in range(8):
        # lg_sample keys image b as row b + 1: the same row alone would key as row 1, so compare probabilities and greedy picks
        _, pb = sample(x[b:b + 1], temperature=temps[b], top_k=ks[b], seed=77)
        assert torch.equal(probs[b], pb[0]), b


# ------------------------------------------------------------------------------------------------------------ serve.LLM
# (temperature, top_k, top_p) of the mixed stream's requests, in request order
FILTERS = [(1.0, 4000, 1.0), (1.0, 1000, 1.0), (1.3, 7, 1.0), (0.9, 2000, 0.95), (0.7, -1, 1.0), (1.0, 16384, 0.9), (1.0, 2000, 1.0),
           (1.0, 300, 1.0)]


def _serve(llm, reqs, waves):
    """reqs: [add_request kwargs]; waves: [(steps before the wave, [indices])]. Returns {index: [token lists of its outputs]}."""
    llm.request_counter = iter([i for _, w in waves for i in w])
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            llm.add_request(**reqs[i])
    while llm.has_unfinished_requests():
        outs += llm.step()
    return {int(o.request_id): [(c.token_ids, c.cumulative_logprob) for c in o.outputs] for o in outs}


def _alone(m, req, i, **llm_kw):
    """Request i alone in an LLM without per_request_sampling, under its own request id (its default seed is base + i)."""
    from llamagen_b200.serve import LLM
    return _serve(LLM(m, **llm_kw), {i: req}, [(0, [i])])[i]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_serve_mixed_filters_share_the_batch(kind):
    from llamagen_b200.serve import LLM, SamplingParams
    S = 24
    if kind == "c2i":
        m = _c2i(torch.bfloat16)
        conds = [dict(prompt_token_ids=[c]) for c in (207, 360, 387, 974, 88, 979, 417, 5)]
    else:
        m = _model(torch.bfloat16, **XL3)
        caps = _captions([5, 37, 64, 120, 17, 90, 1, 33], XL3["caption_dim"], 11)
        conds = [dict(prompt_embeds=f) for f in caps]
    extra = [dict(), dict(prefix=_prefix(4, V, 1)), dict(), dict(given=torch.arange(S) % 97, given_mask=torch.arange(S) % 5 == 2),
             dict(), dict(), dict(), dict()]
    params = [dict(cfg_scale=2.0, seed=11), dict(n=2, seed=12), dict(logprobs=3), dict(cfg_interval=3),
              dict(best_of=2, n=1), dict(), dict(cond_weights=(4.0,)), dict(cfg_scale=1.0)]
    if kind == "t2i":
        extra[5] = dict(negative_prompt_embeds=_captions([9], XL3["caption_dim"], 4)[0])
    reqs = []
    for i in range(len(conds)):
        t, k, p = FILTERS[i]
        if kind == "t2i" and i == 7:
            t = 0.0                                              # greedy beside sampled requests
        sp = SamplingParams(temperature=t, top_k=k, top_p=p, max_tokens=S, **params[i])
        reqs.append(dict(conds[i], sampling_params=sp, **extra[i]))
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=4, seed=5, per_request_sampling=True)
    got = _serve(llm, reqs, [(0, [0, 1, 2]), (3, [3, 4, 5]), (6, [6, 7])])
    assert sorted(got) == list(range(len(reqs)))
    for i, r in enumerate(reqs):
        ref = _alone(m, r, i, cfg_scale=4.0, max_num_seqs=4, seed=5)
        for (a, la), (b, lb) in zip(got[i], ref):
            # top-p draws use float atomics (not bit-reproducible): their requests are compared on what top-p cannot change
            if r["sampling_params"].top_p < 1.0:
                assert len(a) == len(b) == S
            else:
                assert a == b and la == lb, (kind, i)


def test_serve_sjd_mixed_filters():
    from llamagen_b200.serve import LLM, SamplingParams
    m, S = _c2i(torch.bfloat16), 24
    reqs = [dict(prompt_token_ids=[c], sampling_params=SamplingParams(temperature=t, top_k=k, top_p=1.0, max_tokens=S, seed=100 + i))
            for i, (c, (t, k)) in enumerate(zip((207, 360, 387, 974, 88), ((1.0, 4000), (0.7, 7), (1.3, 2000), (0.0, 1), (1.0, -1))))]
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=5, sjd_window=4, per_request_sampling=True)
    got = _serve(llm, reqs, [(0, [0, 1, 2]), (2, [3, 4])])
    for i, r in enumerate(reqs):
        assert got[i] == _alone(m, r, i, cfg_scale=4.0, max_num_seqs=3, seed=5, sjd_window=4), i
