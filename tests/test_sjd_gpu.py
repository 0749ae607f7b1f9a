"""Speculative Jacobi decoding on the GPU: the window attention kernel against a float64 reference, the acceptance kernel against the
test oracle (tests/sjd_oracle.py), and lg_generate_sjd end to end (greedy equality with generate(), replay of sampled runs from the
p rows the engine dumps, determinism, and isolation from generate() and score())."""
import math
import zlib

import numpy as np
import pytest
import torch

import sjd_oracle as so
import test_attention_gpu as ta

DEV = "cuda"


# ------------------------------------------------------------------------------------------------ window attention (path 4)
def _rows(R, Tq, S):
    """Ragged first positions: the first K / V block edges, the condition edge of t2i, and the last window that fits max_seq."""
    base = [0, 63, 64, 1, 120, 127, S - Tq, 200, 31]
    return [min(p, S - Tq) for p in base[:R]]


def _wcases():
    cs = []
    for Tq in (2, 7, 16, 17, 33, 64):
        cs.append(ta.Case(f"win_bf16_hd64_tq{Tq}", "bf16", "auto", 64, 7, 2, 301, (4, 2, 0), Tq=Tq, pos=("rows", _rows(7, Tq, 301))))
    for dt in ("bf16", "f16"):
        for hd, hdp in ((64, 64), (128, 128), (100, 112)):
            for Tq in (17, 64):
                cs.append(ta.Case(f"win_{dt}_hd{hd}_tq{Tq}", dt, "auto", hd, 5, 2, 301, (4, 2, 0), hdp=hdp, Tq=Tq,
                                  pos=("rows", _rows(5, Tq, 301))))
    cs.append(ta.Case("win_mask_bf16", "bf16", "auto", 64, 6, 2, 301, (4, 2, 0), Tq=16, pos=("rows", [120, 121, 150, 200, 285, 130]),
                      mask=("ragged", 3, 120)))
    cs.append(ta.Case("win_mask_f16_hd128", "f16", "auto", 128, 4, 2, 301, (4, 2, 0), Tq=33, pos=("rows", [120, 180, 268, 125]),
                      mask=("ragged", 2, 120)))
    off = []
    for c in (cs[3], cs[-2]):   # the same calls on attention_kernel
        off.append(ta.Case(c.id + "_tma0", c.dt, c.kv, c.hd, c.R, c.H, c.S, (0, 0, 0), hdp=c.hdp, Tq=c.Tq, pos=c.pos, mask=c.mask,
                           env={"LG_ATTN_TMA": "0"}))
    return cs + off


WCASES = {c.id: c for c in _wcases()}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(WCASES))
def test_window_attention_call(cid, monkeypatch):
    """Same inputs, references and bounds as test_attention_gpu.py (needles at block, condition and diagonal edges, poison past each
    query's position and in masked condition keys, guard bands); path 4 must run, and path 0 under LG_ATTN_TMA=0."""
    c = WCASES[cid]
    for k, v in c.env.items():
        monkeypatch.setenv(k, v)
    seed = zlib.crc32(cid.encode())
    worst = ta._one(c, "wide", None, seed)[2]
    Tc = c.mask[2] if c.mask else 0
    for i, nd in enumerate(ta._needle_specs(c, Tc)):
        worst = max(worst, ta._one(c, "needle", nd, seed + 1 + i)[2])
    if c.hdp > c.hd:
        a = ta._one(c, "needle", ("rel", 1), seed + 99, pad="zero")[0]
        b = ta._one(c, "needle", ("rel", 1), seed + 99, pad="garbage")[0]
        assert torch.equal(a, b)
    print(f"[{cid}] path {c.expect} max |out - ref| / absO {worst:.3g}")


# ------------------------------------------------------------------------------------------------ acceptance kernel
def _verify_gpu(p, q, qflag, x, win, nfin, start, S, seed, greedy):
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, L, V = p.shape
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to(device=DEV, dtype=dt).contiguous()
    dp, dq = t(p, torch.float32), t(q, torch.float32)
    dfl, dx, dw = t(qflag, torch.int32), t(x, torch.int32), t(win, torch.int32)
    dn, ds = t(nfin, torch.int32), t(start, torch.int32)
    out = torch.full((B, S), -1, dtype=torch.int32, device=DEV)
    P = _lib.ptr
    _lib.check(lib.lg_test_sjd_verify(B, S, L, V, int(greedy), seed, P(dp), P(dq), P(dfl), P(dx), P(dw), P(dn), P(ds), P(out),
                                      _lib.current_stream(DEV)), "lg_test_sjd_verify")
    torch.cuda.synchronize()
    return out.cpu().numpy(), dn.cpu().numpy(), ds.cpu().numpy()


def _rand_rows(rng, n, V, topk=None):
    x = np.exp(rng.standard_normal((n, V)) * 1.5)
    if topk:
        cut = np.sort(x, 1)[:, -topk][:, None]
        x = np.where(x >= cut, x, 0.0)
    return (x / x.sum(1, keepdims=True)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("greedy", [0, 1])
@pytest.mark.parametrize("V", [37, 1000])
def test_verify_kernel_matches_oracle(greedy, V):
    rng = np.random.default_rng(V + greedy)
    B, L, S, seed = 96, 8, 40, 1234
    p = _rand_rows(rng, B * L, V, topk=5).reshape(B, L, V)
    q = _rand_rows(rng, B * L, V, topk=7).reshape(B, L, V)
    q[::3] = p[::3]                                              # p = q: every draft of those images is accepted
    qflag = (rng.random((B, L)) < 0.2).astype(np.int32)
    qflag[::3] = 0
    x = np.array([[so.inv_cdf(p[b, i], rng.random()) for i in range(L)] for b in range(B)], np.int32)
    if greedy:
        x = p.argmax(-1).astype(np.int32)
    nfin = rng.integers(1, S, B).astype(np.int32)
    start = np.minimum(nfin, S - L).astype(np.int32)
    win = np.zeros((B, L), np.int32)
    for b in range(B):
        for i in range(1, L):
            k = start[b] + i - 1
            if k >= nfin[b]:
                src = np.full(V, 1.0 / V) if qflag[b, i - 1] else q[b, i - 1]
                win[b, i] = so.inv_cdf(src, rng.random()) if rng.random() < 0.7 or greedy == 0 else p[b, i - 1].argmax()
    out, n2, s2 = _verify_gpu(p, q, qflag, x, win, nfin, start, S, seed, greedy)
    accepted = 0
    for b in range(B):
        im = so.Image(S, L, V, seed, b, 0)
        im.n, im.s, im.win = int(nfin[b]), int(start[b]), [int(t) for t in win[b]]
        im.q = [None if qflag[b, i] else q[b, i] for i in range(L)]
        made = im.step(p[b], x[b], bool(greedy))
        k0 = int(nfin[b])
        assert list(out[b, k0:k0 + len(made)]) == made, b
        assert (out[b, :k0] == -1).all() and (out[b, k0 + len(made):] == -1).all()
        assert (n2[b], s2[b]) == (im.n, im.s)
        accepted += len(made) - 1
    assert accepted > B // 4


def _residual_uniforms(seed, B, k):
    """u_res(k) of images 0 .. B - 1 (sjd_oracle.uniform, vectorised)."""
    def sm(x):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))
    with np.errstate(over="ignore"):
        b = np.arange(1, B + 1, dtype=np.uint64)
        c1, c3 = np.uint64((so.C1 * (k + 1)) & so.M64), np.uint64((so.C3 * so.RESIDUAL) & so.M64)
        r = sm(sm(sm(np.uint64(seed) ^ c1) ^ (np.uint64(so.C2) * b)) ^ c3)
    return (r >> np.uint64(40)).astype(np.float64) * 2.0 ** -24


@pytest.mark.gpu
def test_verify_residual_draw_intervals():
    """About 1.5 million residual draws of normalize(max(0, p - q)) at V = 16384 (1024 images x 1500 seeds; every draft has p = 0 and
    is rejected): each pick's float64 CDF interval over the fp32 residual weights holds u_res within (ceil(V / 512) + 16) 2^-24, and
    its weight is > 0. The fp32 segment prefixes of the 512 threads have gaps and overlaps; a target there must still go to a
    neighbouring segment, never to an unrelated token."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, L, S, V, seeds = 1024, 2, 3, 16384, 1500
    g = torch.Generator(device=DEV).manual_seed(4)
    p = torch.softmax(torch.randn(B, L, V, device=DEV, generator=g) * 2.0, -1)
    q = torch.softmax(torch.randn(B, L, V, device=DEV, generator=g) * 2.0, -1)
    p[:, 0, 0] = 0                                     # the draft (token 0) has p = 0: rejected
    p, q = p.contiguous(), q.contiguous()
    w = torch.clamp_min(p[:, 0] - q[:, 0], 0).double()   # the kernel's fp32 weights fmaxf(0, p - q), exactly
    C = w.cumsum(1)
    C = C / C[:, -1:]
    zi = torch.zeros(B, L, dtype=torch.int32, device=DEV)
    nfin = torch.empty(B, dtype=torch.int32, device=DEV)
    start = torch.empty(B, dtype=torch.int32, device=DEV)
    out = torch.empty(B, S, dtype=torch.int32, device=DEV)
    picks = torch.empty(seeds, B, dtype=torch.long, device=DEV)
    P = _lib.ptr
    for j in range(seeds):
        nfin.fill_(1)
        start.fill_(1)
        out.fill_(-1)
        _lib.check(lib.lg_test_sjd_verify(B, S, L, V, 0, 1000 + j, P(p), P(q), P(zi), P(zi), P(zi), P(nfin), P(start), P(out),
                                          _lib.current_stream(DEV)), "lg_test_sjd_verify")
        picks[j] = out[:, 1].long()
    u = torch.from_numpy(np.stack([_residual_uniforms(1000 + j, B, 1) for j in range(seeds)])).to(DEV)   # [seeds][B]
    pk = picks.t().contiguous()                                                                          # [B][seeds]
    assert (pk >= 0).all() and (w.gather(1, pk) > 0).all()
    hi = C.gather(1, pk)
    lo = torch.where(pk > 0, C.gather(1, (pk - 1).clamp(min=0)), torch.zeros_like(hi))
    band = (math.ceil(V / 512) + 16) * 2.0 ** -24
    ut = u.t()
    bad = (ut < lo - band) | (ut > hi + band)
    print(f"[residual sweep] {B * seeds} draws, {int(bad.sum())} outside their interval")
    assert int(bad.sum()) == 0, bad.nonzero()[:10].tolist()


@pytest.mark.gpu
def test_verify_first_token_histogram_is_p():
    """65536 images share one (p, q) pair and differ only in their keys; the first token made final follows p_0 (total variation below
    1.3 times its expectation under p_0 plus 0.003)."""
    rng = np.random.default_rng(3)
    B, L, S, V = 65536, 4, 10, 16
    p0 = _rand_rows(rng, 1, V, topk=12)[0]
    q0 = _rand_rows(rng, 1, V)[0]
    p = np.broadcast_to(p0, (B, L, V))
    q = np.broadcast_to(q0, (B, L, V))
    x = np.tile(np.array([so.inv_cdf(p0, u) for u in rng.random(L)], np.int32), (B, 1))
    win = np.zeros((B, L), np.int32)
    win[:, 1:] = np.array([so.inv_cdf(q0, u) for u in rng.random(B * (L - 1))]).reshape(B, L - 1)
    nfin = np.ones(B, np.int32)
    out, _, _ = _verify_gpu(p, q, np.zeros((B, L), np.int32), x, win, nfin, nfin.copy(), S, 99, 0)
    h = np.bincount(out[:, 1], minlength=V) / B
    tv = 0.5 * np.abs(h - p0).sum()
    e_tv = np.sqrt(p0 * (1 - p0) / (2 * np.pi * B)).sum()
    assert tv < 1.3 * e_tv + 0.003, (tv, e_tv)


# ------------------------------------------------------------------------------------------------ end to end
def _model(t2i=False, dtype=torch.float32, dim=256, n_layer=2, n_head=4, kv=None, seed=0):
    from llamagen_b200 import ModelArgs, Transformer
    torch.manual_seed(seed)
    kw = dict(model_type="t2i", cls_token_num=8, caption_dim=64) if t2i else dict(num_classes=10)
    m = Transformer(ModelArgs(dim=dim, n_layer=n_layer, n_head=n_head, vocab_size=512, block_size=64, **kw))
    m.output.weight.data.normal_(std=0.05)
    if kv:
        m.set_kv_cache(kv)
    return m.to(device=DEV, dtype=dtype).eval()


def _cond(m, B, seed=1):
    g = torch.Generator().manual_seed(seed)
    if m.model_type == "c2i":
        return torch.randint(0, 10, (B,), generator=g).to(DEV), None
    cond = torch.randn(B, 8, 64, generator=g).to(device=DEV, dtype=m.tok_embeddings.weight.dtype)
    em = torch.ones(B, 8, device=DEV)
    em[0, :3] = 0
    if B > 2:
        em[2, :6] = 0
    return cond, em


def _sjd_dbg(m, cond, em, S, L, cfg, **sk):
    """lg_generate_sjd with its p rows: (tokens [B, S], passes, dbg [passes][B][L][V], L actually run)."""
    from llamagen_b200 import _lib
    from llamagen_b200.generate import _generate_sjd
    B, L = cond.shape[0], min(L, S - 1)
    T = 1 if m.model_type == "c2i" else cond.shape[1]
    rows = 2 * B if cfg > 1 else B
    m.setup_caches(max_batch_size=rows, max_seq_length=T + S)
    lib, h = _lib.load(), m.engine()
    out = torch.empty(B, S, dtype=torch.int32, device=DEV)
    dbg = torch.full((S - 1, B, L, m.vocab_size), float("nan"), device=DEV)
    sc = _lib.SampleCfg(float(cfg), int(sk.get("cfg_interval", -1)), float(sk.get("temperature", 1.0)), int(sk.get("top_k", 0)),
                        float(sk.get("top_p", 1.0)), 0 if sk.get("sample_logits", True) else 1, int(sk["seed"]))
    cd = cond.to(torch.int32).contiguous() if m.model_type == "c2i" else cond.contiguous()
    toks, st = _generate_sjd(m, lib, h, cond, cd, em, B, T, S, out, L, cfg > 1, True, sc, dbg)
    return toks, st["iterations"], dbg, L


@pytest.mark.gpu
@pytest.mark.parametrize("t2i", [False, True], ids=["c2i", "t2i"])
@pytest.mark.parametrize("cfg", [1.0, 4.0])
@pytest.mark.parametrize("L", [2, 8, 16])
def test_greedy_sjd_equals_greedy_generate_fp32(t2i, cfg, L):
    from llamagen_b200 import generate
    m = _model(t2i)
    cond, em = _cond(m, 3)
    want = generate(m, cond, 40, emb_masks=em, cfg_scale=cfg, sample_logits=False)
    got, st = generate(m, cond, 40, emb_masks=em, cfg_scale=cfg, sample_logits=False, sjd_window=L, return_stats=True)
    assert torch.equal(got, want)
    assert 1 <= st["iterations"] <= 39 and st["tokens_per_iteration"] == 39 / st["iterations"]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_greedy_sjd_tokens_are_argmax_of_score_16bit(dtype):
    """Every token is the argmax of score()'s logits at its position, or within 4 units in the last place of the model dtype at that
    row's largest logit: the window pass and the scoring pass round bf16 / fp16 activations in different places (4 layers)."""
    from llamagen_b200 import generate, score
    m = _model(False, dtype, dim=512, n_layer=4, n_head=8)
    cond, _ = _cond(m, 4)
    toks = generate(m, cond, 48, cfg_scale=4.0, sample_logits=False, sjd_window=8)
    _, logits = score(m, cond, toks.long(), cfg_scale=4.0, return_logits=True)
    picked = logits.gather(-1, toks.long()[..., None])[..., 0]
    top = logits.max(-1).values
    _, e = torch.frexp(top.abs())
    margin = 4 * torch.ldexp(torch.ones_like(top), e - (8 if dtype == torch.bfloat16 else 11))
    gap = top - picked
    assert (gap <= margin).all(), (gap.max().item(), margin.min().item())


def _replay_check(m, cond, em, S, L, cfg, **sk):
    toks, passes, dbg, L = _sjd_dbg(m, cond, em, S, L, cfg, **sk)
    d = dbg[:passes].cpu().numpy()
    want, n = so.replay(d, toks[:, 0].cpu().numpy(), S, L, m.vocab_size, sk["seed"], not sk.get("sample_logits", True))
    assert n == passes
    assert np.array_equal(toks.cpu().numpy(), want)
    return toks, passes, dbg


@pytest.mark.gpu
@pytest.mark.parametrize("t2i", [False, True], ids=["c2i", "t2i"])
def test_sampled_sjd_replays_exactly_bf16(t2i):
    from llamagen_b200 import generate
    m = _model(t2i, torch.bfloat16)
    cond, em = _cond(m, 4)
    sk = dict(seed=77, top_k=40, top_p=0.9, temperature=1.0, cfg_interval=10)
    toks, passes, dbg = _replay_check(m, cond, em, 48, 8, 4.0, **sk)
    # token 0 is drawn exactly as generate() draws it
    ref = generate(m, cond, 48, emb_masks=em, cfg_scale=4.0, cfg_interval=10, top_k=40, top_p=0.9, seed=77)
    assert torch.equal(ref[:, 0], toks[:, 0])


@pytest.mark.gpu
def test_sjd_is_deterministic_graph_and_eager(monkeypatch):
    from llamagen_b200 import generate
    m = _model(False, torch.bfloat16)
    cond, _ = _cond(m, 5)
    kw = dict(cfg_scale=4.0, top_k=50, seed=5, sjd_window=16)
    a = generate(m, cond, 60, **kw)
    b = generate(m, cond, 60, **kw)
    monkeypatch.setenv("LG_NO_GRAPH", "1")
    m._drop_engine()
    c = generate(m, cond, 60, **kw)
    assert torch.equal(a, b) and torch.equal(a, c)


@pytest.mark.gpu
def test_sjd_fp8_cache_runs_and_replays():
    m = _model(False, torch.bfloat16, kv="fp8")
    cond, _ = _cond(m, 3)
    _replay_check(m, cond, None, 40, 8, 4.0, seed=9, top_k=30)


@pytest.mark.gpu
def test_generate_and_score_unchanged_after_sjd():
    from llamagen_b200 import generate, score
    m = _model(False, torch.bfloat16)
    cond, _ = _cond(m, 4)
    g0 = generate(m, cond, 32, cfg_scale=4.0, seed=3, top_k=20)
    s0 = score(m, cond, g0.long(), cfg_scale=4.0)
    generate(m, cond, 32, cfg_scale=4.0, seed=3, top_k=20, sjd_window=8)
    g1 = generate(m, cond, 32, cfg_scale=4.0, seed=3, top_k=20)
    s1 = score(m, cond, g1.long(), cfg_scale=4.0)
    assert torch.equal(g0, g1) and torch.equal(s0, s1)
