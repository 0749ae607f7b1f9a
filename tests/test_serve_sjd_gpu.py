"""GPU: speculative Jacobi decoding in serve.LLM (sjd_window=L).

* Kernel: one per-slot verify + refresh (lg_test_sjd_slots) on given p / x rows, slots with their own seeds and pass counters, against
  tests/sjd_oracle.Image (b = 0, the slot's own pass index); a frozen slot's state is left as it was.
* Bit for bit: with one slot and no CFG (c2i and t2i, bf16, L in {4, 16}) every request's tokens and pass count equal
  generate(sjd_window=L, seed=s) at B = 1.
* Schedule independence under CFG, per-request scales, intervals and seeds (negatives on t2i): all-queued, staggered and reversed
  arrivals give the same tokens per request (bf16, fp16, fp8 KV cache, head_dim 128).
* Replay: with every pass's p rows dumped, each request's tokens and pass count are the oracle's replay of its own slot.
* Greedy t2i (temperature 0): fp32 tokens equal the plain LLM's; bf16 tokens are the argmax of score()'s teacher-forced logits.
* Hand-back: generate() and a plain LLM give the same tokens before and after an SJD LLM ran on the model."""
import numpy as np
import pytest
import torch

import sjd_oracle as so
from test_serve_guidance_gpu import _run
from test_serve_prefix_gpu import C2I
from test_serve_t2i_gpu import HD128, XL3, _captions, _model

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("greedy", [0, 1])
def test_slot_verify_refresh_matches_oracle(greedy):
    from llamagen_b200 import _lib
    lib, stream = _lib.load(), _lib.current_stream("cuda")
    B, S, L, V = 5, 40, 6, 96
    rng = np.random.default_rng(7 + greedy)
    seeds = [3, 2 ** 63 - 5, 12345, 99, 7]
    passes = [0, 4, 1, 9, 2]
    frozen = 3                                   # nfin >= S: verify and refresh leave it alone
    imgs = [so.Image(S, L, V, seeds[b], 0, int(rng.integers(V))) for b in range(B)]
    out = np.full((B, S), -1, np.int32)
    for b, im in enumerate(imgs):
        out[b, 0] = im.out[0]
    q = np.zeros((B, L, V), np.float32)
    qflag = np.ones((B, L), np.int32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(q=dev(q), qflag=dev(qflag), win=dev(np.array([im.win for im in imgs], np.int32)),
             nfin=dev(np.array([1, 1, 1, S, 1], np.int32)), start=dev(np.ones(B, np.int32)),
             seeds=dev(np.array(seeds, np.uint64).view(np.int64)), passes=dev(np.array(passes, np.int32)),
             seed_rows=torch.zeros(B * L, dtype=torch.int64, device="cuda"), step_rows=torch.zeros(B * L, dtype=torch.int32, device="cuda"),
             out=dev(out))
    for it in range(S):                                          # every pass makes a token final: every slot finishes
        before = {k: v.clone() for k, v in d.items()}
        p = rng.random((B, L, V), dtype=np.float32) ** 4
        p[:, :, rng.integers(V)] += 2.0                         # a likely token, so that drafts get accepted
        p /= p.sum(-1, keepdims=True)
        x = np.zeros((B, L), np.int32)
        for b, im in enumerate(imgs):
            if b != frozen and not im.done:
                x[b] = so.draws(p[b], seeds[b], 0, passes[b], im.s, greedy)
        p_d, x_d = dev(p), dev(x)                               # kept alive until the call has run
        _lib.check(lib.lg_test_sjd_slots(B, S, L, V, greedy, _lib.ptr(p_d), _lib.ptr(x_d), _lib.ptr(d["q"]), _lib.ptr(d["qflag"]),
                                         _lib.ptr(d["win"]), _lib.ptr(d["nfin"]), _lib.ptr(d["start"]), _lib.ptr(d["seeds"]),
                                         _lib.ptr(d["passes"]), _lib.ptr(d["seed_rows"]), _lib.ptr(d["step_rows"]), _lib.ptr(d["out"]),
                                         stream), "lg_test_sjd_slots")
        torch.cuda.synchronize()
        for b, im in enumerate(imgs):
            if b == frozen or im.done:                          # nothing of the slot changes
                for k in ("q", "qflag", "win", "nfin", "start", "seeds", "passes", "out"):
                    assert torch.equal(d[k][b], before[k][b]), (it, b, k)
                for k in ("seed_rows", "step_rows"):
                    assert torch.equal(d[k][b * L:(b + 1) * L], before[k][b * L:(b + 1) * L]), (it, b, k)
                continue
            im.step(p[b], x[b], greedy)
            passes[b] += 1
            assert d["out"][b, :im.n].tolist() == im.out[:im.n], (it, b)
            assert (int(d["nfin"][b]), int(d["start"][b]), int(d["passes"][b])) == (im.n, im.s, passes[b]), (it, b)
            if im.done:
                continue
            assert d["win"][b].tolist() == im.win, (it, b)
            for t in range(im.n - im.s, L - 1):                 # the q of every draft (other entries are never read)
                assert int(d["qflag"][b, t]) == (im.q[t] is None), (it, b, t)
                if im.q[t] is not None:
                    assert np.array_equal(d["q"][b, t].cpu().numpy(), im.q[t]), (it, b, t)
            want_seed = so.pass_seed(seeds[b], 0, passes[b])
            assert [int(v) & so.M64 for v in d["seed_rows"][b * L:(b + 1) * L].tolist()] == [want_seed] * L, (it, b)
            assert d["step_rows"][b * L:(b + 1) * L].tolist() == [im.s + t for t in range(L)], (it, b)
    assert all(im.done for b, im in enumerate(imgs) if b != frozen)


# ------------------------------------------------------------------------------------------------------------ serving
def _c2i(dt=torch.bfloat16, kv="auto"):
    return _model(dt, kv, **C2I)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("L", [4, 16])
def test_one_slot_equals_generate_sjd_bit_for_bit(kind, L):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    from test_serve_prefix_gpu import _oracle_cond
    if kind == "t2i":
        m, S, conds = _model(torch.bfloat16, **XL3), 32, _captions([5, 120, 64], XL3["caption_dim"], 9)
    else:
        m, S, conds = _c2i(), 48, [207, 360, 387]
    seeds = [123456789, 0, 2 ** 63 - 1]
    reqs = [(c, SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, seed=s), None, None) for c, s in zip(conds, seeds)]
    llm = LLM(m, cfg_scale=1.0, max_num_seqs=1, seed=40, sjd_window=L)
    got = _run(llm, reqs, [(0, [0, 1, 2])])
    for r, (c, s) in enumerate(zip(conds, seeds)):
        cond, em = _oracle_cond(llm, c)
        ref, st = generate(m, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), cfg_scale=1.0, temperature=1.0, top_k=1000,
                           seed=s, sjd_window=L, return_stats=True)
        assert ref[0].cpu().tolist() == got[r], f"request {r} (seed {s})"
        assert llm.sjd_request_passes[str(r)] == st["iterations"], r
    assert llm.sjd_passes >= sum(llm.sjd_request_passes.values()) and llm.sjd_tokens == 3 * (S - 1)


GUIDES = [(4.0, -1, 11), (2.0, 3, 22), (1.0, -1, 33), (7.5, 0, 44), (7.5, 10, 55), (4.0, -1, 66)]


def _mixed(kind, dt, kv, cfg=None):
    from llamagen_b200.serve import SamplingParams
    if kind == "t2i":
        m, S = _model(dt, kv, **(cfg or XL3)), 24
        C = (cfg or XL3)["caption_dim"]
        conds = _captions([5, 37, 64, 120, 17, 90], C, 11)
        negs = [None, _captions([9], C, 3)[0], None, _captions([120], C, 4)[0], None, None]
    else:
        m, S = _c2i(dt, kv), 32
        conds, negs = [207, 360, 387, 974, 88, 979], [None] * 6
    reqs = [(conds[i], SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, cfg_scale=c, cfg_interval=k, seed=s * 1000 + 7), None,
             negs[i] if c > 1.0 else None) for i, (c, k, s) in enumerate(GUIDES)]
    return m, S, reqs


@pytest.mark.parametrize("kind, dt, kv, cfg", [("c2i", torch.bfloat16, "auto", None), ("t2i", torch.bfloat16, "auto", None),
                                               ("c2i", torch.float16, "auto", None), ("t2i", torch.float16, "auto", None),
                                               ("c2i", torch.bfloat16, "fp8", None), ("t2i", torch.bfloat16, "fp8", None),
                                               ("t2i", torch.bfloat16, "auto", HD128)],
                         ids=["c2i_bf16", "t2i_bf16", "c2i_f16", "t2i_f16", "c2i_kv_fp8", "t2i_kv_fp8", "t2i_hd128"])
def test_tokens_do_not_depend_on_the_schedule(kind, dt, kv, cfg):
    from llamagen_b200.serve import LLM
    m, S, reqs = _mixed(kind, dt, kv, cfg)
    n = len(reqs)
    runs = []
    for waves in ([(0, list(range(n)))], [(0, [0, 1]), (2, [2, 3]), (5, [4, 5])], [(0, list(reversed(range(n))))]):
        llm = LLM(m, cfg_scale=4.0, max_num_seqs=4, seed=5, sjd_window=8)
        got = _run(llm, reqs, waves)
        assert sorted(got) == list(range(n)) and all(len(t) == S for t in got.values())
        runs.append(got)
        assert llm.sjd_tokens == n * (S - 1) and llm.sjd_passes < n * (S - 1)
    assert runs[0] == runs[1] == runs[2]
    assert len({tuple(t) for t in runs[0].values()}) == n


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_every_request_replays_from_its_own_slot(kind, monkeypatch):
    from llamagen_b200.serve import LLM
    m, S, reqs = _mixed(kind, torch.bfloat16, "auto")
    L, B = 8, 3
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=B, seed=5, sjd_window=L)
    rec = []
    orig = LLM._device_sjd_pass

    def dump(self, st, params, dbg=None):
        d = torch.full((B, L, m.vocab_size), float("nan"), device="cuda")
        orig(self, st, params, d)
        rec.append((st["passes"], d, [None if r is None else r.request_id for r in self._slots], list(st["first_pass"])))

    monkeypatch.setattr(LLM, "_device_sjd_pass", dump)
    got = _run(llm, reqs, [(0, [0, 1, 2, 3]), (3, [4]), (6, [5])])
    for r, toks in got.items():
        rid, seed = str(r), reqs[r][1].seed
        im = so.Image(S, L, m.vocab_size, seed, 0, toks[0])
        j = 0
        for p, d, slots, first in rec:
            if rid not in slots or im.done:
                continue
            b = slots.index(rid)
            assert p >= first[b]
            rows = d[b].cpu().numpy()
            im.step(rows, so.draws(rows, seed, 0, j, im.s, False), False)
            j += 1
        assert im.done and im.out == toks, r
        assert llm.sjd_request_passes[rid] == j, r


def _small_t2i(dtype, **kw):
    from test_sjd_gpu import _model as sjd_model
    return sjd_model(True, dtype, **kw)


def _small_caps(n, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((int(rng.integers(2, 9)), 64)).astype(np.float32) for _ in range(n)]


def test_greedy_t2i_equals_plain_greedy_fp32():
    from llamagen_b200.serve import LLM, SamplingParams
    m = _small_t2i(torch.float32)
    S, caps = 40, _small_caps(5, 3)
    sp = SamplingParams(temperature=0.0, max_tokens=S)
    reqs = [(c, sp, None, None) for c in caps]
    waves = [(0, [0, 1]), (3, [2, 3]), (7, [4])]
    plain = _run(LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=1), reqs, waves)
    for L in (4, 16):
        assert _run(LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=1, sjd_window=L), reqs, waves) == plain, L


def test_greedy_t2i_tokens_are_argmax_of_score_bf16():
    from llamagen_b200 import score
    from llamagen_b200.serve import LLM, SamplingParams
    m = _small_t2i(torch.bfloat16, dim=512, n_layer=4, n_head=8)
    S, caps = 48, _small_caps(4, 5)
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=2, seed=1, sjd_window=8)
    got = _run(llm, [(c, SamplingParams(temperature=0.0, max_tokens=S), None, None) for c in caps], [(0, [0, 1, 2, 3])])
    conds = [llm._caption(c) for c in caps]
    cond = torch.stack([c for c, _ in conds]).to(device="cuda", dtype=torch.bfloat16)
    em = torch.stack([k for _, k in conds]).cuda()
    toks = torch.tensor([got[i] for i in range(len(caps))], device="cuda")
    _, logits = score(m, cond, toks, emb_masks=em, cfg_scale=4.0, return_logits=True)
    picked = logits.gather(-1, toks[..., None])[..., 0]
    top = logits.max(-1).values
    _, e = torch.frexp(top.abs())
    margin = 4 * torch.ldexp(torch.ones_like(top), e - 8)     # 4 bf16 ulps at the row's largest logit, as for generate(sjd_window=)
    gap = top - picked
    assert (gap <= margin).all(), (gap.max().item(), margin.min().item())


def test_generate_and_plain_serving_unchanged_after_sjd_serving():
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m = _c2i()
    S = 32
    cond = torch.tensor([3, 500, 999], device="cuda")
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S)

    def both():
        g = generate(m, cond, S, cfg_scale=4.0, top_k=1000, seed=9)
        gs = generate(m, cond, S, cfg_scale=4.0, top_k=1000, seed=9, sjd_window=8)
        s = LLM(m, cfg_scale=4.0, max_num_seqs=2, seed=2).generate(prompt_token_ids=[[3], [500], [1000], [1000]], sampling_params=sp)
        return g.cpu(), gs.cpu(), [o.outputs[0].token_ids for o in s]

    before = both()
    sjd = LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=2, sjd_window=8).generate(
        prompt_token_ids=[[3], [500], [7], [1000], [1000], [1000]], sampling_params=sp)
    assert [o.outputs[0].token_ids for o in sjd[:3]] == [o.outputs[0].token_ids for o in sjd[3:]]   # the null-class twins
    after = both()
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1]) and before[2] == after[2]


def test_two_sjd_llms_alternate_on_one_model():
    """Every SJD LLM keeps its own slot state: LLM A (2 slots, L = 8), then B on the same model (6 slots, L = 4, the same max_tokens),
    then A again. A gives the same tokens both times, and B those of a fresh LLM of its configuration."""
    from llamagen_b200.serve import LLM
    m, S, reqs = _mixed("c2i", torch.bfloat16, "auto")
    a = LLM(m, cfg_scale=4.0, max_num_seqs=2, seed=5, sjd_window=8)
    first = _run(a, reqs[:3], [(0, [0, 1, 2])])
    got_b = _run(LLM(m, cfg_scale=4.0, max_num_seqs=6, seed=5, sjd_window=4), reqs, [(0, list(range(6)))])
    again = _run(a, reqs[:3], [(0, [0, 1, 2])])
    assert again == first
    assert got_b == _run(LLM(m, cfg_scale=4.0, max_num_seqs=6, seed=5, sjd_window=4), reqs, [(0, list(range(6)))])
