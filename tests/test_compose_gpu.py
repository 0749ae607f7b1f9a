"""GPU: composable guidance, generate(..., cond_weights=) / lg_generate_composed, and the sample kernel's grouped mix.

* Kernel (lg_test_sample_groups): random logits, B in {1, 8, 64} images, K in {1, 2, 3, 8} conditions, round dtype f32 / bf16 / f16,
  the FILTERS of test_serve_guidance_gpu, sampled and greedy: K = 1 with weight w equals lg_sample_rows at cfg_scale = w bit for
  bit; greedy ids equal the float64 K-way mix of the rounded rows followed by sample_oracle; a zero-weight group changes no id
  whatever its logits; every image's token reaches all K of its next_tokens rows.
* K = 1 end to end: generate(cond[:, None], cond_weights=[s]) is generate(cond, cfg_scale=s) token for token, c2i and t2i, in
  bf16, fp16, bf16 with an fp8 KV cache and with fp8 weights, on the plain, prefix, negative, given and logprobs paths (logprobs
  equal too), at B = 64 with two decode chains.
* K > 1, fp32 greedy on the golden models: K = 2 and 3 with mixed-sign per-image weights (t2i also with a negative, c2i also with
  a prefix) give the compose oracle's tokens.
* Independence: other images' conditions and weights do not change image 0's tokens."""
import ctypes

import pytest
import torch

from compose_oracle import compose_oracle
from oracle import GPTOracle
from test_given_gpu import _cond, _model, _run
from test_negative_gpu import _cond as _caption
from test_serve_guidance_gpu import FILTERS
from util import build_gpt, load_golden

pytestmark = pytest.mark.gpu

V = 16384
RD = {"f32": 0, "bf16": 1, "f16": 2}


def _round(x, rd):
    return x if rd == "f32" else x.to(torch.bfloat16 if rd == "bf16" else torch.float16).float()


def _groups(lib, x, B, K, rd, f, w, seeds, steps, stream):
    from llamagen_b200 import _lib
    sc = _lib.SampleCfg(1.0, -1, 1.0, f["top_k"], f["top_p"], f["greedy"], 0)
    got = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    nxt = torch.full((B * K,), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.lg_test_sample_groups(_lib.ptr(x), B, K, V, RD[rd], ctypes.byref(sc), _lib.ptr(w), _lib.ptr(seeds), _lib.ptr(steps),
                                         _lib.ptr(got), _lib.ptr(nxt), stream), "lg_test_sample_groups")
    got, nxt = got.cpu(), nxt.cpu()
    assert torch.equal(nxt, got.repeat_interleave(K)), "an image's token must reach all K of its rows"
    return got


@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("K", [1, 2, 3, 8])
@pytest.mark.parametrize("B", [1, 8, 64])
def test_grouped_mix(B, K, rd):
    from llamagen_b200 import _lib
    from oracle.sampling_oracle import sample_oracle
    lib = _lib.load()
    stream = _lib.current_stream("cuda")
    g = torch.Generator().manual_seed(100 * B + 10 * K + RD[rd])
    R = B * K
    x = (3.0 * torch.randn(2 * R, V, generator=g)).cuda()
    steps = torch.randint(0, 12, (B,), generator=g, dtype=torch.int32).cuda()
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64).cuda()
    w = (4.0 * torch.rand(B, K, generator=g) - 1.5).cuda()                         # mixed signs
    for f in FILTERS:
        if K == 1:   # plain CFG at the same scale: same rows, same keys
            w1 = torch.full((B, 1), 4.0, device="cuda")
            got = _groups(lib, x, B, K, rd, f, w1, seeds, steps, stream)
            sc = _lib.SampleCfg(4.0, -1, 1.0, f["top_k"], f["top_p"], f["greedy"], 0)
            want = torch.full((B,), -1, dtype=torch.int32, device="cuda")
            _lib.check(lib.lg_sample_rows(_lib.ptr(x), B, V, 1, RD[rd], ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), _lib.ptr(want),
                                          None, 0, stream), "lg_sample_rows")
            assert torch.equal(got, want.cpu()), (f, (got != want.cpu()).nonzero().flatten().tolist())
        got = _groups(lib, x, B, K, rd, f, w, seeds, steps, stream)
        if f["greedy"]:
            xr = _round(x.cpu(), rd).double()
            c, u = xr[:R].view(B, K, V), xr[R:].view(B, K, V)[:, 0]
            mixed = u + ((c - u[:, None]) * w.cpu().double()[:, :, None]).sum(1)
            idx, _ = sample_oracle(mixed, top_k=f["top_k"], top_p=f["top_p"], sample_logits=False)
            top2 = mixed.topk(2, dim=-1).values
            clear = (top2[:, 0] - top2[:, 1]) > 1e-3 * top2[:, 0].abs().clamp_min(1.0)   # skip near-ties of fp32 against fp64
            assert torch.equal(got[clear], idx[:, 0].to(torch.int32)[clear]), f
        if K > 1:   # a zero-weight group: its logits are never seen
            z = K // 2
            wz = w.clone()
            wz[:, z] = 0.0
            a = _groups(lib, x, B, K, rd, f, wz, seeds, steps, stream)
            x2 = x.clone()
            x2[:R].view(B, K, V)[:, z] = (3.0 * torch.randn(B, V, generator=g)).cuda()
            b = _groups(lib, x2, B, K, rd, f, wz, seeds, steps, stream)
            assert torch.equal(a, b), f


# ------------------------------------------------------------------------------------------------------------ K = 1 end to end
def _k1_pair(m, cond, em, S, s, **kw):
    """generate(cond, cfg_scale=s, ...) and generate(cond[:, None], cond_weights=[s], ...)."""
    plain = _run_any(m, cond, em, S, cfg_scale=s, **kw)
    em1 = None if em is None else em[:, None]
    comp = _run_any(m, cond[:, None], em1, S, cond_weights=[s], **kw)
    return plain, comp


def _run_any(m, cond, em, S, **kw):
    from llamagen_b200 import generate
    out = generate(m, cond, S, em, **kw)
    torch.cuda.synchronize()
    if isinstance(out, tuple):
        return tuple(o.cpu() if torch.is_tensor(o) else {k: v.cpu() for k, v in o.items()} for o in out)
    return out.cpu()


def _equal(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    return torch.equal(a, b)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("store", ["bf16", "f16", "kv_fp8", "w_fp8"])
def test_k1_equals_cfg(kind, store, monkeypatch):
    from llamagen_b200 import _lib
    monkeypatch.delenv("LG_SPLIT", raising=False)
    dt = torch.float16 if store == "f16" else torch.bfloat16
    m = _model(dt, kv="fp8" if store == "kv_fp8" else "auto", w8="fp8" if store == "w_fp8" else "auto", t2i=kind == "t2i")
    S, P, B = 256, 40, 64
    cond, em = _cond(m, B)
    s = 4.0
    gv = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(9))
    hole = torch.ones(S, dtype=torch.bool)
    hole[100:180] = False
    hole[30] = False
    cases = {"plain": dict(top_k=100, seed=5, cfg_interval=150), "greedy": dict(sample_logits=False),
             "prefix": dict(top_k=100, seed=6, prefix=gv[:, :P]), "given": dict(top_k=100, seed=7, given=gv, given_mask=hole),
             "logprobs": dict(top_k=100, seed=8, return_logprobs=True, top_logprobs=3),
             # top-k only: a top-p draw is not run-to-run deterministic over thousands of draws even on the plain path (the nucleus
             # mass histogram sums in shared-memory float atomics), so two top-p calls cannot be compared bit for bit
             "prefix_logprobs": dict(top_k=50, seed=10, prefix=gv[:, :P], return_logprobs=True)}
    if kind == "t2i":
        T, C = m.cls_token_num, m.config.caption_dim
        neg = (0.5 * torch.randn(1, T, C, generator=torch.Generator().manual_seed(3))).to("cuda", dt)
        nm = torch.ones(1, T, device="cuda")
        nm[:, :5] = 0
        cases["negative"] = dict(top_k=100, seed=11, negative_cond=neg, negative_emb_masks=nm)
        cases["negative_prefix"] = dict(top_k=100, seed=12, negative_cond=neg, prefix=gv[:, :P])
    lib = _lib.load()
    for name, kw in cases.items():
        plain, comp = _k1_pair(m, cond, em, S, s, **kw)
        assert _equal(plain, comp), f"{kind} {store} {name}: K = 1 differs from cfg_scale={s}"
        if name == "prefix" and store in ("bf16", "f16") and kind == "c2i":
            n = ctypes.c_int(0)
            lib.lg_test_prefix_chunks(m.engine(), ctypes.byref(n))
            assert n.value == 2, f"B = {B} was meant to run two decode chains, ran {n.value}"


# ------------------------------------------------------------------------------------------------------------ K > 1 against the oracle
def _golden(name):
    g = load_golden(name)
    return g, build_gpt(g["cfg"], g["state_dict"], torch.float32)


def test_fp32_c2i_against_compose_oracle():
    g, m = _golden("gpt_c2i.pt")
    S, labels = g["S"], g["cond"]
    B, nc = labels.shape[0], g["cfg"]["num_classes"]
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for K in (2, 3):
        cond = torch.stack([labels] + [(labels + 3 * i + 1) % nc for i in range(1, K)], 1)
        w = torch.tensor([[4.0, -1.5, 2.0], [2.5, 1.0, -0.5], [-1.0, 5.0, 0.25], [3.0, 0.0, 1.5]])[:, :K]
        w = w.repeat(B // 4 + 1, 1)[:B]
        for kw in (dict(), dict(prefix=g["tokens_cfg4.0"][:, : S // 2].long())):
            out = _run_any(m, cond.cuda(), None, S, cond_weights=w, sample_logits=False, **kw)
            want, _ = compose_oracle(orc, cond, w, S, sample_logits=False, **kw)
            assert torch.equal(out, want.cpu()), f"K={K} {sorted(kw)}: greedy tokens differ from the compose oracle"


def test_fp32_t2i_against_compose_oracle():
    g, m = _golden("gpt_t2i.pt")
    S, cond0, em0 = g["S"], g["cond"], g["emb_masks"]
    B, T, C = cond0.shape
    orc = GPTOracle(g["state_dict"], g["cfg"])
    extra = [_caption(B, T, C, [(7 * b + 3 * i) % T + 1 for b in range(B)], 20 + i) for i in range(2)]
    neg, nm = _caption(1, T, C, [T // 3], 31)
    for K in (2, 3):
        cond = torch.stack([cond0] + [e[0] for e in extra[: K - 1]], 1)
        em = torch.stack([em0] + [e[1] for e in extra[: K - 1]], 1)
        w = torch.tensor([[6.0, -2.0, 1.0], [1.5, 3.0, -0.75]])[:, :K].repeat(B // 2 + 1, 1)[:B]
        for kw in (dict(), dict(negative_cond=neg, negative_emb_masks=nm)):
            out = _run_any(m, cond.cuda(), em.cuda(), S, cond_weights=w, sample_logits=False,
                           **{k: v.cuda() for k, v in kw.items()})
            want, _ = compose_oracle(orc, cond, w, S, emb_masks=em, negative=kw.get("negative_cond"),
                                     negative_emb_masks=kw.get("negative_emb_masks"), sample_logits=False)
            assert torch.equal(out, want.cpu()), f"K={K} {sorted(kw)}: greedy tokens differ from the compose oracle"


def test_k2_given_keeps_tokens_and_an_empty_mask_is_the_plain_call():
    m = _model(torch.bfloat16, dim=512, n_head=8)
    S, B, K = 256, 8, 2
    cond = torch.randint(0, 1000, (B, K), generator=torch.Generator().manual_seed(2)).cuda()
    w = torch.tensor([3.0, 1.5])
    gv = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(4))
    kw = dict(cond_weights=w, top_k=200, seed=3)
    plain = _run(m, cond, None, S, **kw)
    assert torch.equal(_run(m, cond, None, S, given=gv, given_mask=torch.zeros(S, dtype=torch.bool), **kw), plain)
    hole = torch.ones(S, dtype=torch.bool)
    hole[64:160] = False
    got = _run(m, cond, None, S, given=gv, given_mask=hole, **kw)
    assert torch.equal(got[:, hole], gv[:, hole].to(torch.int32))
    lead = torch.zeros(S, dtype=torch.bool)
    lead[:50] = True
    assert torch.equal(_run(m, cond, None, S, given=gv, given_mask=lead, **kw), _run(m, cond, None, S, prefix=gv[:, :50], **kw))


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_independence_of_other_images(kind):
    m = _model(torch.bfloat16, t2i=kind == "t2i")
    S, B, K = 256, 4, 3
    g = torch.Generator().manual_seed(5)
    w = torch.tensor([[4.0, -1.0, 2.0]]).repeat(B, 1)
    if kind == "c2i":
        cond = torch.randint(0, 1000, (B, K), generator=g).cuda()
        other = cond.clone()
        other[1:] = torch.randint(0, 1000, (B - 1, K), generator=g).cuda()
        em = em2 = None
    else:
        T, C = m.cls_token_num, m.config.caption_dim
        cond = (0.5 * torch.randn(B, K, T, C, generator=g)).to("cuda", torch.bfloat16)
        other = cond.clone()
        other[1:] = (0.5 * torch.randn(B - 1, K, T, C, generator=g)).to("cuda", torch.bfloat16)
        em = torch.ones(B, K, T, device="cuda")
        em2 = em.clone()
        em2[1:, :, :3] = 0
    w2 = w.clone()
    w2[1:] = torch.tensor([-2.0, 0.0, 7.0])
    a = _run(m, cond, em, S, cond_weights=w, top_k=500, seed=1)
    b = _run(m, other, em2, S, cond_weights=w2, top_k=500, seed=1)
    assert torch.equal(a[0], b[0]), "image 0's tokens depend on the other images"
    assert not torch.equal(a[1:], b[1:])
