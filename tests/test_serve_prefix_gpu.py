"""GPU: image-completion requests in serve.LLM (lg_prefill_slot_prefix joins), c2i and t2i.

* fp32 exact mode on the golden models, greedy (top-k 1), with and without CFG: completion requests (P from 1 to max_tokens - 1)
  and plain requests arrive in three waves, join mid-sequence and into slots that still hold an earlier request's K / V; every
  completion request's tokens equal prefix_oracle's, every plain request's GPTOracle.generate's.
* With one slot and cfg 1.0 (the row counts of generate with B = 1), sampled: the tokens equal generate(prefix=..., seed=base + r)
  bit for bit.
* Schedule invariance, sampling, in bf16, fp16 and bf16 with an fp8 KV cache: the same requests (mixed P, mixed with plain requests)
  all queued at once, in staggered waves and in reversed arrival order (other slots, other co-runners) give the same tokens.
* A join writes positions 0 .. T + P - 1 of its slot's two cache rows and no other byte of the workspace, and those bytes equal
  what generate(prefix=...) writes for the same request.
* CFG greedy at the GPT-L c2i shape in bf16: the tokens agree with generate(prefix=...) up to a first difference at a top-1 / top-2
  gap of at most 0.25 (the rule of tools/bench_prefix.py)."""
import pytest
import torch

from prefix_oracle import prefix_oracle
from test_serve_t2i_gpu import XL3, _captions, _model
from util import build_gpt, load_golden, top2_gap

pytestmark = pytest.mark.gpu

C2I = dict(n_layer=2, n_head=16, dim=1024, vocab_size=16384, block_size=256, num_classes=1000)
GPT_L = dict(C2I, n_layer=4)


def _prefix(P, V, seed):
    return torch.randint(0, V, (P,), generator=torch.Generator().manual_seed(seed)) if P else None


def _run(llm, conds, prefixes, sp, waves):
    """waves: [(steps to run before the wave, [request indices])]; request i is conds[i] (a class id or caption features) with
    prefixes[i] (or None). Request ids follow the indices whatever the arrival order, so that request r keeps its RNG stream (seed
    base + r) in every schedule. Returns {index: tokens}."""
    order = [i for _, w in waves for i in w]
    llm.request_counter = iter(order)
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            if llm.t2i:
                llm.add_request(prompt_embeds=conds[i], sampling_params=sp, prefix=prefixes[i])
            else:
                llm.add_request([conds[i]], sp, prefix=prefixes[i])
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): o.outputs[0].token_ids for o in outs}
    assert sorted(got) == sorted(order) and all(len(t) == sp.max_tokens for t in got.values())
    for i, pf in enumerate(prefixes):
        if pf is not None:
            assert got[i][:len(pf)] == pf.tolist(), f"request {i}: token_ids[:P] != prefix"
    return got


def _oracle_cond(llm, c):
    """The condition and emb-mask a request's join is given, as the oracle takes them (a batch of one)."""
    if not llm.t2i:
        return torch.tensor([c]), None
    cond, mask = llm._caption(c)
    return cond[None], mask[None]


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
def test_fp32_exact_against_prefix_oracle_in_three_waves(name, cfg_scale):
    from llamagen_b200.serve import LLM, SamplingParams
    from oracle import GPTOracle
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    S, V = g["S"], m.vocab_size
    Ps = [3, 0, S - 1, 1, 7, 0, S // 2, 2]
    conds = (_captions([5, 37, 64, 120, 9, 88, 17, 120], g["cfg"]["caption_dim"], 7) if m.model_type == "t2i"
             else [1, 2, 3, 4, 5, 6, 7, 8])
    prefixes = [_prefix(P, V, 100 + i) for i, P in enumerate(Ps)]
    llm = LLM(m, cfg_scale=cfg_scale, num_classes=g["cfg"]["num_classes"], max_num_seqs=3, seed=3)
    sp = SamplingParams(temperature=1.0, top_k=1, max_tokens=S)
    got = _run(llm, conds, prefixes, sp, [(0, [0, 1]), (3, [2, 3, 4]), (S + 5, [5, 6, 7])])
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for i, (c, pf) in enumerate(zip(conds, prefixes)):
        cond, em = _oracle_cond(llm, c)
        if pf is None:
            want, _ = orc.generate(cond, S, emb_masks=em, cfg_scale=cfg_scale, sample_logits=False)
        else:
            want, _ = prefix_oracle(orc, cond, pf[None], S, emb_masks=em, cfg_scale=cfg_scale, sample_logits=False)
        assert got[i] == want[0].tolist(), f"request {i} (P={Ps[i]})"


@pytest.mark.parametrize("case", ["c2i_bf16", "t2i_bf16"])
def test_one_slot_without_cfg_is_generate_bit_for_bit(case):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    if case == "t2i_bf16":
        m, S, conds = _model(torch.bfloat16, **XL3), 32, _captions([5, 120, 64], XL3["caption_dim"], 9)
    else:
        m, S, conds = _model(torch.bfloat16, **C2I), 160, [207, 360, 387]
    Ps = [5, 0, S - 2]
    prefixes = [_prefix(P, m.vocab_size, 30 + i) for i, P in enumerate(Ps)]
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S)
    llm = LLM(m, cfg_scale=1.0, max_num_seqs=1, seed=40)
    got = _run(llm, conds, prefixes, sp, [(0, [0, 1, 2])])
    for r, (c, pf) in enumerate(zip(conds, prefixes)):
        cond, em = _oracle_cond(llm, c)
        kw = dict(emb_masks=None if em is None else em.cuda(), cfg_scale=1.0, temperature=1.0, top_k=1000, seed=40 + r)
        ref = generate(m, cond.cuda(), S, prefix=None if pf is None else pf[None], **kw)
        assert ref[0].cpu().tolist() == got[r], f"request {r} (P={Ps[r]})"


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("dt, kv", [(torch.bfloat16, "auto"), (torch.float16, "auto"), (torch.bfloat16, "fp8")],
                         ids=["bf16", "f16", "bf16_kv_fp8"])
def test_tokens_do_not_depend_on_the_schedule(kind, dt, kv):
    from llamagen_b200.serve import LLM, SamplingParams
    if kind == "t2i":      # T + P reaches past 128 positions (kernel 2 for fp8 caches)
        m, S, cfg = _model(dt, kv, **XL3), 24, 7.5
        conds = _captions([5, 37, 64, 120, 17, 90, 1], XL3["caption_dim"], 11)
        Ps = [0, 23, 10, 0, 1, 16, 4]
    else:                  # P of 130 and 139: Tq > 128 from position 0
        m, S, cfg = _model(dt, kv, **C2I), 140, 4.0
        conds = [207, 360, 387, 974, 88, 979, 417]
        Ps = [0, 139, 64, 0, 1, 130, 9]
    prefixes = [_prefix(P, m.vocab_size, 50 + i) for i, P in enumerate(Ps)]
    sp = SamplingParams(temperature=1.0, top_k=1000, top_p=1.0, max_tokens=S)
    n = len(conds)
    runs = []
    for waves in ([(0, list(range(n)))],                                   # all queued at once
                  [(0, [0, 1]), (3, [2, 3, 4]), (7, [5, 6])],             # staggered waves
                  [(0, list(reversed(range(n))))]):                       # reversed: other slots, other co-runners
        llm = LLM(m, cfg_scale=cfg, max_num_seqs=5, seed=21)
        runs.append(_run(llm, conds, prefixes, sp, waves))
    assert runs[0] == runs[1] == runs[2]
    assert len({tuple(t) for t in runs[0].values()}) == n                 # the requests really differ


def _workspace(m):
    """m's workspace from its 256-byte aligned base, as raw bytes."""
    buf = m._workspace
    return buf[(buf.data_ptr() + 255) // 256 * 256 - buf.data_ptr():]


def _kv(m, ws):
    """K and V of every layer in a tensor laid out as m's workspace: [L, rows, H, max_seq, hd * esz] each (lg_engine::carve_kv)."""
    c = m.config
    rows, max_seq = m._ws_shape
    hd, esz = c.dim // c.n_head, (1 if m._kv_cache[0] == "fp8" else 2)
    kbytes = c.n_layer * rows * c.n_head * max_seq * hd * esz
    return [ws[s:s + kbytes].view(c.n_layer, rows, c.n_head, max_seq, hd * esz) for s in (0, (kbytes + 255) // 256 * 256)]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_join_writes_only_its_slot_rows(kind):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    shape, cfg = (XL3, 7.5) if kind == "t2i" else (C2I, 4.0)
    m = _model(torch.bfloat16, **shape)
    conds = _captions([40, 120, 7], XL3["caption_dim"], 5) if kind == "t2i" else [3, 4, 5]
    B, P, S = 3, 50, 64
    T = m.cls_token_num
    pf = _prefix(P, m.vocab_size, 8)
    llm = LLM(m, cfg_scale=cfg, max_num_seqs=B, seed=1)
    sp = SamplingParams(top_k=1000, max_tokens=S)
    for c in conds[:2]:
        if kind == "t2i":
            llm.add_request(prompt_embeds=c, sampling_params=sp)
        else:
            llm.add_request([c], sp)
    for _ in range(6):
        llm.step()                                                        # slots 0, 1 run; slot 2 is free
    ws = _workspace(m)
    may = torch.zeros_like(ws, dtype=torch.bool)
    for v in _kv(m, may):
        v[:, [2, B + 2], :, :T + P] = True
    torch.cuda.synchronize()
    before = ws.clone()
    if kind == "t2i":
        llm.add_request(prompt_embeds=conds[2], sampling_params=sp, prefix=pf)
    else:
        llm.add_request([conds[2]], sp, prefix=pf)
    st = llm._state
    req = llm._waiting.popleft()                                          # join it by hand: the slot's rows alone, no decode step
    llm._slots[2] = req
    if kind == "t2i":
        st["cond"][2].copy_(req.cond)
        st["mask"][2].copy_(req.mask)
    else:
        st["tok"][2] = conds[2]
    st["seeds"][2] = llm._seed + int(req.request_id)
    st["out"][2, :P] = pf.cuda().to(torch.int32)
    llm._device_join_prefix(st, sp, 2, P)
    torch.cuda.synchronize()
    changed = ws != before
    assert not bool((changed & ~may).any()), "lg_prefill_slot_prefix wrote outside its slot's K / V rows"
    got = [v[:, [2, B + 2], :, :T + P].clone() for v in _kv(m, ws)]
    for g in got:                                                         # and it wrote K and V of both rows
        assert bool((g[:, 0] != 0).any()) and bool((g[:, 1] != 0).any())
    assert bool(torch.isfinite(st["join_logits"]).all())
    # the same request through generate(prefix=...) (B = 1: rows 0 and 1) on a fresh copy of the model writes the same bytes
    m2 = _model(torch.bfloat16, **shape)
    cond, em = _oracle_cond(llm, conds[2])
    generate(m2, cond.cuda(), P + 1, emb_masks=None if em is None else em.cuda(), cfg_scale=cfg, sample_logits=False, prefix=pf[None])
    torch.cuda.synchronize()
    for a, b in zip(got, _kv(m2, _workspace(m2))):
        assert torch.equal(a, b[:, [0, 1], :, :T + P]), "the join's K / V differ from generate(prefix=...)'s"


def test_cfg_greedy_agrees_with_generate_up_to_a_near_tie():
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(torch.bfloat16, **GPT_L)
    S = 256
    conds = [207, 360, 387, 974]
    Ps = [64, 128, 192, 1]
    prefixes = [_prefix(P, m.vocab_size, 70 + i) for i, P in enumerate(Ps)]
    got = _run(LLM(m, cfg_scale=4.0, max_num_seqs=4, seed=0), conds, prefixes, SamplingParams(temperature=1.0, top_k=1, max_tokens=S),
               [(0, [0, 1]), (5, [2, 3])])
    for r, (c, pf) in enumerate(zip(conds, prefixes)):
        cond = torch.tensor([c], device="cuda")
        ref = generate(m, cond, S, cfg_scale=4.0, sample_logits=False, prefix=pf[None])[0].cpu().tolist()
        if ref == got[r]:
            continue
        k = next(i for i in range(S) if ref[i] != got[r][i])
        assert k >= Ps[r]
        _, logits = generate(m, cond, S, cfg_scale=4.0, sample_logits=False, return_logits=True,
                             teacher=torch.tensor([got[r]], dtype=torch.int32, device="cuda"))
        gap = top2_gap(logits[k, 0].float().cpu()).item()
        print(f"[request {r}, P={Ps[r]}] first difference at token {k}, top-1 / top-2 gap {gap:.4f}")
        assert gap <= 0.25, (r, k, gap)
