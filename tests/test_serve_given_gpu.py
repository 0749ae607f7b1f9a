"""GPU: inpainting requests in serve.LLM (add_request(..., given=, given_mask=)), c2i and t2i.

* fp32 exact mode on the golden models, greedy: inpainting, prefix and plain requests arrive in three waves into 3 slots that still hold
  stale K / V; every inpainting request's tokens equal given_oracle's, every prefix request's prefix_oracle's, every plain request's
  GPTOracle.generate's; again with a negative prompt and with per-request cfg_scale / cfg_interval.
* One slot, cfg 1.0, sampled: the tokens equal generate(given=..., given_mask=..., seed=base + r) bit for bit (a run longer than 64).
* Schedule invariance in bf16, fp16, bf16 with an fp8 KV cache and bf16 with fp8 weights; an n = 3 request in a busy batch and alone.
* lg_extend_slot writes positions T + a - 1 .. T + a + K - 1 of its slot's rows and no other workspace byte, the same in slot 0 and
  slot B - 1.
* lg_sample_rows_given: rows with a given token return it, the others draw what lg_sample_rows_keyed / lg_sample_rows_logprobs draw.
* CFG greedy at the GPT-L c2i shape in bf16 agrees with generate(given=) up to a first difference at a top-1 / top-2 gap <= 0.25."""
import ctypes

import pytest
import torch

from given_oracle import given_oracle
from prefix_oracle import prefix_oracle
from test_serve_prefix_gpu import C2I, GPT_L, _oracle_cond, _workspace
from test_serve_t2i_gpu import XL3, _captions, _model
from util import build_gpt, load_golden, top2_gap

pytestmark = pytest.mark.gpu


def _ids(S, V, seed):
    return torch.randint(0, V, (S,), generator=torch.Generator().manual_seed(seed))


def _mask(S, runs):
    m = torch.zeros(S, dtype=torch.bool)
    for a, b in runs:
        m[a:b] = True
    return m


def _run(llm, conds, kws, sp, waves):
    """waves: [(steps before the wave, [request indices])]; request i is conds[i] with add_request keywords kws[i] (given / prefix /
    negative) and sampling params sp (one, or one per request). Request ids follow the indices. Returns {index: [tokens per sample]}."""
    order = [i for _, w in waves for i in w]
    llm.request_counter = iter(order)
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            p = sp[i] if isinstance(sp, list) else sp
            if llm.t2i:
                llm.add_request(prompt_embeds=conds[i], sampling_params=p, **kws[i])
            else:
                llm.add_request([conds[i]], p, **kws[i])
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): [c.token_ids for c in o.outputs] for o in outs}
    assert sorted(got) == sorted(order)
    for i in got:
        kw = kws[i]
        if "given" in kw:
            for t in got[i]:
                assert torch.equal(torch.tensor(t)[kw["given_mask"]], kw["given"][kw["given_mask"]]), f"request {i}: a given token changed"
    return got


def _golden_kws(S, V, n):
    """Inpainting (box holes, runs of one, a trailing run), prefix and plain requests for the golden models' S = 16."""
    masks = [_mask(S, [(0, 3), (5, 9), (12, S)]), _mask(S, [(2, 3), (4, 5), (9, 13)]), _mask(S, [(1, 14)]), _mask(S, [(0, 8)]),
             _mask(S, [(6, S)])]
    kws = [dict(given=_ids(S, V, 10 + i), given_mask=m) for i, m in enumerate(masks)]
    kws += [dict(prefix=_ids(5, V, 30)), dict(), dict(prefix=_ids(S - 1, V, 31))]
    return kws[:n]


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("mode", ["cfg1", "cfg4", "negative_and_guidance"])
def test_fp32_exact_against_the_oracles_in_three_waves(name, mode):
    from llamagen_b200.serve import LLM, SamplingParams
    from oracle import GPTOracle
    if mode == "negative_and_guidance" and name == "gpt_c2i.pt":
        pytest.skip("negative prompts are t2i only; c2i per-request guidance runs in cfg4 below")
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    S, V = g["S"], m.vocab_size
    kws = _golden_kws(S, V, 8)
    n = len(kws)
    t2i = m.model_type == "t2i"
    conds = _captions([5, 37, 64, 120, 9, 88, 17, 120], g["cfg"]["caption_dim"], 7) if t2i else [1, 2, 3, 4, 5, 6, 7, 8]
    cfg = 1.0 if mode == "cfg1" else 4.0
    base = SamplingParams(temperature=1.0, top_k=1, max_tokens=S)
    sp = [base] * n
    negs = [None] * n
    if mode != "cfg1":   # per-request guidance: scales and intervals differ between requests of one batch
        sp = [SamplingParams(temperature=1.0, top_k=1, max_tokens=S, cfg_scale=[4.0, 2.5, 1.0, 7.0][i % 4], cfg_interval=[-1, 6, -1, 3][i % 4])
              for i in range(n)]
    if mode == "negative_and_guidance":
        negs = _captions([7, 50, 3, 12, 9, 1, 30, 90], g["cfg"]["caption_dim"], 8)
        negs = [ng if sp[i].cfg_scale > 1 and i % 2 == 0 and "given" in kws[i] else None for i, ng in enumerate(negs)]
        for i, ng in enumerate(negs):
            if ng is not None:
                kws[i] = dict(kws[i], negative_prompt_embeds=ng)
    llm = LLM(m, cfg_scale=cfg, num_classes=g["cfg"]["num_classes"], max_num_seqs=3, seed=3)
    got = _run(llm, conds, kws, sp, [(0, [0, 1, 5]), (3, [2, 6, 3]), (S + 5, [4, 7])])
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for i, (c, kw) in enumerate(zip(conds, kws)):
        cond, em = _oracle_cond(llm, c)
        scale = cfg if sp[i].cfg_scale is None else sp[i].cfg_scale
        ok = dict(emb_masks=em, cfg_scale=scale, cfg_interval=-1 if sp[i].cfg_interval is None else sp[i].cfg_interval,
                  sample_logits=False)
        if "given" in kw:
            ng = None
            if negs[i] is not None:
                ncond, nmask = llm._caption(negs[i])
                ng, ok["negative_emb_masks"] = ncond[None], nmask[None]
            want, _ = given_oracle(orc, cond, kw["given"][None], kw["given_mask"][None], S, negative=ng, **ok)
        elif "prefix" in kw:
            want, _ = prefix_oracle(orc, cond, kw["prefix"][None], S, **ok)
        else:
            want, _ = orc.generate(cond, S, **ok)
        assert got[i][0] == want[0].tolist(), f"request {i} ({sorted(kw)})"


@pytest.mark.parametrize("case", ["c2i_bf16", "t2i_bf16"])
def test_one_slot_without_cfg_is_generate_bit_for_bit(case):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    if case == "t2i_bf16":
        m, S, conds = _model(torch.bfloat16, **XL3), 100, _captions([5, 120, 64], XL3["caption_dim"], 9)
    else:
        m, S, conds = _model(torch.bfloat16, **C2I), 160, [207, 360, 387]
    masks = [_mask(S, [(5, 10), (20, 100), (S - 7, S)]),            # a run of 80: two window chunks (64 + 17)
             _mask(S, [(0, 12), (30, 31), (40, 44)]),               # a leading run (a prefix join), a run of one
             _mask(S, [(k, k + 1) for k in range(1, S - 1, 3)])]
    kws = [dict(given=_ids(S, m.vocab_size, 40 + i), given_mask=mk) for i, mk in enumerate(masks)]
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S)
    llm = LLM(m, cfg_scale=1.0, max_num_seqs=1, seed=40)
    got = _run(llm, conds, kws, sp, [(0, [0, 1, 2])])
    for r, (c, kw) in enumerate(zip(conds, kws)):
        cond, em = _oracle_cond(llm, c)
        ref = generate(m, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), cfg_scale=1.0, temperature=1.0, top_k=1000,
                       seed=40 + r, given=kw["given"][None], given_mask=kw["given_mask"])
        assert ref[0].cpu().tolist() == got[r][0], f"request {r}"


def _kv(m, ws):
    """K and V of every layer in a tensor laid out as m's workspace: [L, rows, H, max_seq, hd * esz] each (lg_engine::carve_kv)."""
    c = m.config
    rows, max_seq = m._ws_shape
    hd = c.dim // c.n_head
    esz = 1 if m._kv_cache[0] == "fp8" else m.tok_embeddings.weight.element_size()
    kbytes = c.n_layer * rows * c.n_head * max_seq * hd * esz
    return [ws[s:s + kbytes].view(c.n_layer, rows, c.n_head, max_seq, hd * esz) for s in (0, (kbytes + 255) // 256 * 256)]


def _mixed(kind, dt, kv, w8=False):
    m = _model(dt, kv, **(XL3 if kind == "t2i" else C2I))
    if w8:
        m.set_weight_dtype("fp8")
    if kind == "t2i":
        S, cfg, conds = 100, 7.5, _captions([5, 37, 64, 120, 17, 90, 1], XL3["caption_dim"], 11)
    else:
        S, cfg, conds = 140, 4.0, [207, 360, 387, 974, 88, 979, 417]
    V = m.vocab_size
    kws = [dict(given=_ids(S, V, 60), given_mask=_mask(S, [(0, 30), (34, 40), (44, 50), (54, 70), (75, S)])),
           dict(), dict(given=_ids(S, V, 61), given_mask=_mask(S, [(3, 90)])), dict(prefix=_ids(9, V, 62)),
           dict(given=_ids(S, V, 63), given_mask=_mask(S, [(k, k + 1) for k in range(2, S - 1, 2)])),
           dict(given=_ids(S, V, 64), given_mask=_mask(S, [(0, 50)])), dict(given=_ids(S, V, 65), given_mask=_mask(S, [(10, 12), (60, S)]))]
    return m, S, cfg, conds, kws


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("dt, kv, w8", [(torch.bfloat16, "auto", False), (torch.float16, "auto", False), (torch.bfloat16, "fp8", False),
                                        (torch.bfloat16, "auto", True)], ids=["bf16", "f16", "bf16_kv_fp8", "bf16_w_fp8"])
def test_tokens_do_not_depend_on_the_schedule(kind, dt, kv, w8):
    from llamagen_b200.serve import LLM, SamplingParams
    m, S, cfg, conds, kws = _mixed(kind, dt, kv, w8)
    sp = SamplingParams(temperature=1.0, top_k=1000, top_p=1.0, max_tokens=S)
    n = len(conds)
    runs = []
    for waves in ([(0, list(range(n)))], [(0, [0, 1]), (3, [2, 3, 4]), (7, [5, 6])], [(0, list(reversed(range(n))))]):
        runs.append(_run(LLM(m, cfg_scale=cfg, max_num_seqs=5, seed=21), conds, kws, sp, waves))
    assert runs[0] == runs[1] == runs[2]
    assert len({tuple(t[0]) for t in runs[0].values()}) == n
    if dt == torch.bfloat16 and kv == "auto" and not w8:   # an n = 3 inpainting request in a busy batch and alone
        sp3 = [sp] * n
        sp3[2] = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, n=3, seed=5)
        busy = _run(LLM(m, cfg_scale=cfg, max_num_seqs=7, seed=21), conds, kws, sp3, [(0, [0, 1]), (2, [2, 3, 4])])
        alone = _run(LLM(m, cfg_scale=cfg, max_num_seqs=7, seed=21), conds, kws, sp3, [(0, [2])])   # same slot count: same decode shapes
        assert busy[2] == alone[2] and len(busy[2]) == 3 and len({tuple(t) for t in busy[2]}) == 3


@pytest.mark.parametrize("kind, dt, kv", [("c2i", torch.bfloat16, "auto"), ("t2i", torch.bfloat16, "auto"), ("c2i", torch.bfloat16, "fp8"),
                                          ("c2i", torch.float32, "auto")], ids=["c2i_bf16", "t2i_bf16", "c2i_kv_fp8", "c2i_f32"])
def test_extend_writes_only_its_slot_rows(kind, dt, kv):
    from llamagen_b200 import _lib
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(dt, kv, **(XL3 if kind == "t2i" else C2I))
    B, S, a, K, cfg = 3, 128, 20, 70, 4.0     # K + 1 = 71 rows: a chunk of 64 and one of 7
    T = m.cls_token_num
    llm = LLM(m, cfg_scale=cfg, max_num_seqs=B, seed=1)
    sp = SamplingParams(top_k=1000, max_tokens=S)
    conds = _captions([40, 120], XL3["caption_dim"], 5) if kind == "t2i" else [3, 4]
    for c in conds:
        if kind == "t2i":
            llm.add_request(prompt_embeds=c, sampling_params=sp)
        else:
            llm.add_request([c], sp)
    for _ in range(6):
        llm.step()                                                        # slots 0, 1 run; slot 2 is free and holds zeros
    st, lib = llm._state, _lib.load()
    st["out"][B - 1] = _ids(S, m.vocab_size, 3).to(torch.int32).cuda()
    if kind == "t2i":
        st["mask"][B - 1] = 1.0
        st["neg_mask"][B - 1] = 1.0

    def extend(slot):
        ws, nb = m._slot_extend_scratch(1, K)
        em = _lib.ptr(st["mask"][slot]) if kind == "t2i" else None
        nm = _lib.ptr(st["neg_mask"][slot]) if kind == "t2i" else None
        _lib.check(lib.lg_extend_slot(m.engine(), _lib.ptr(st["out"][B - 1]), S, a, K, slot, B, 1, em, nm, ws, nb, _lib.ptr(st["join_logits"]),
                                      _lib.current_stream(st["dev"])), "lg_extend_slot")
        torch.cuda.synchronize()
        return st["join_logits"].clone()

    ws = _workspace(m)
    may = torch.zeros_like(ws, dtype=torch.bool)
    for v in _kv(m, may):
        v[:, [B - 1, 2 * B - 1], :, T + a - 1:T + a + K] = True
    torch.cuda.synchronize()
    before = ws.clone()
    logits_last = extend(B - 1)
    changed = ws != before
    assert not bool((changed & ~may).any()), "lg_extend_slot wrote outside its slot's positions"
    got = [v[:, [B - 1, 2 * B - 1], :, T + a - 1:T + a + K].clone() for v in _kv(m, ws)]
    for gk in got:
        assert bool((gk[:, 0] != 0).any()) and bool((gk[:, 1] != 0).any())
    assert bool(torch.isfinite(logits_last).all())
    # slot 0 with the same history (positions [0, T + a - 1) copied from slot B - 1) writes the same bytes and gives the same logits
    if kind == "t2i":
        st["mask"][0] = 1.0
        st["neg_mask"][0] = 1.0
    llm._device_copy_kv(st, B - 1, [0], T + a - 1)
    logits_first = extend(0)
    for gk, v in zip(got, _kv(m, ws)):
        assert torch.equal(gk, v[:, [0, B], :, T + a - 1:T + a + K]), "slot 0 and slot B - 1 differ"
    assert torch.equal(logits_first, logits_last)


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("logprobs", [False, True])
def test_sample_rows_given_keeps_given_rows_and_draws_the_others(dt, logprobs):
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, V, S = 16, 16384, 32
    gen = torch.Generator().manual_seed(0)
    logits = (torch.randn(2 * B, V, generator=gen) * 3).cuda()
    seeds = torch.randint(0, 2 ** 40, (B,), generator=gen).cuda()
    steps = torch.randint(0, S, (B,), generator=gen).to(torch.int32).cuda()
    cfg = torch.tensor([4.0, 1.0, 2.5, 7.5] * (B // 4)).cuda()
    interval = torch.tensor([-1, 3, 10, -1] * (B // 4), dtype=torch.int32).cuda()
    img = torch.arange(B, dtype=torch.int32).cuda() % 3
    given = torch.full((B, S), -1, dtype=torch.int32)
    rows = list(range(0, B, 3))
    for b in rows:
        given[b, int(steps[b])] = 7 + b
    given = given.cuda()
    sc = _lib.SampleCfg(4.0, -1, 1.0, 100, 0.95, 0, 0)
    dtc = _lib.dtype_code(dt)

    def run(name, *extra):
        out_idx = torch.full((B,), -5, dtype=torch.int32, device="cuda")
        out_seq = torch.full((B, S), -5, dtype=torch.int32, device="cuda")
        lp = torch.zeros(B, S, device="cuda")
        rank = torch.zeros(B, S, dtype=torch.int32, device="cuda")
        spec = _lib.Logprobs(lp.data_ptr(), rank.data_ptr(), 0, 0, 0)
        lpa = (ctypes.byref(spec),) if logprobs else (None,)
        fn = getattr(lib, name)
        head = (_lib.ptr(logits), B, V, 1, dtc, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), _lib.ptr(cfg), _lib.ptr(interval),
                _lib.ptr(img))
        _lib.check(fn(*head, *extra, *(lpa if name != "lg_sample_rows_keyed" else ()), _lib.ptr(out_idx), _lib.ptr(out_seq), S, None), name)
        torch.cuda.synchronize()
        return out_idx.cpu(), out_seq.cpu(), lp.cpu(), rank.cpu()

    ref = run("lg_sample_rows_logprobs" if logprobs else "lg_sample_rows_keyed")
    got = run("lg_sample_rows_given", _lib.ptr(given))
    for b in range(B):
        k = int(steps[b])
        want = 7 + b if b in rows else int(ref[0][b])
        assert int(got[0][b]) == want and int(got[1][b, k]) == want, b
        if logprobs and b not in rows:
            assert float(got[2][b, k]) == float(ref[2][b, k]) and int(got[3][b, k]) == int(ref[3][b, k])
    assert any(int(ref[0][b]) != 7 + b for b in rows)


def test_cfg_greedy_agrees_with_generate_up_to_a_near_tie():
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(torch.bfloat16, **GPT_L)
    S = 256
    conds = [207, 360, 387, 974]
    masks = [_mask(S, [(0, 96), (100, 112), (116, 128), (132, 144), (148, S)]),        # a 4 x 4 hole in a 16 x 16 grid
             _mask(S, [(k * 16, k * 16 + 8) for k in range(16)]),                     # the left half
             _mask(S, [(0, 64), (192, S)]), _mask(S, [(10, 200)])]
    kws = [dict(given=_ids(S, m.vocab_size, 80 + i), given_mask=mk) for i, mk in enumerate(masks)]
    got = _run(LLM(m, cfg_scale=4.0, max_num_seqs=4, seed=0), conds, kws, SamplingParams(temperature=1.0, top_k=1, max_tokens=S),
               [(0, [0, 1]), (5, [2, 3])])
    for r, (c, kw) in enumerate(zip(conds, kws)):
        cond = torch.tensor([c], device="cuda")
        ref = generate(m, cond, S, cfg_scale=4.0, sample_logits=False, given=kw["given"][None], given_mask=kw["given_mask"])[0].cpu().tolist()
        if ref == got[r][0]:
            continue
        k = next(i for i in range(S) if ref[i] != got[r][0][i])
        assert not kw["given_mask"][k]
        _, logits = generate(m, cond, S, cfg_scale=4.0, sample_logits=False, return_logits=True,
                             teacher=torch.tensor([got[r][0]], dtype=torch.int32, device="cuda"))
        gap = top2_gap(logits[k, 0].float().cpu()).item()
        print(f"[request {r}] first difference at token {k}, top-1 / top-2 gap {gap:.4f}")
        assert gap <= 0.25, (r, k, gap)
