"""GPU: serve.LLM on text-conditional models (lg_prefill_slot joins, lg_decode_rows_t2i steps).

* fp32 exact mode on the reference-made golden t2i model, cfg 4.0, greedy: requests in three arrival waves, more requests than
  slots, joins mid-sequence and into slots that still hold an earlier request's K / V; every request's tokens equal the oracle's on
  its caption through the reference front end (sample_t2i.py:89-106, restated as in test_t2i_feature_files_to_tokens_match_oracle).
* Schedule invariance, sampling at cfg 7.5 / top-k 1000: GPT-XL t2i cut to 3 layers in bf16, fp16 and bf16 with an fp8 KV cache
  (attn_prefill_tc_kernel for the joins), and an hd-128 shape (attention_kernel for the joins). The same requests all queued at once,
  in staggered waves and in reversed arrival order (other slots, other co-runners) give the same tokens, byte for byte.
* A join writes positions 0 .. T - 1 of its slot's cache rows and no other byte of the workspace.
* Anchor to generate(): with one slot and cfg 1.0 (the row counts of generate with B = 1) the tokens equal generate(seed=base + r)
  bit for bit, sampling included; with cfg 7.5 and greedy decoding they agree up to a first difference at a top-1 / top-2 gap of
  at most 0.5 (the rule of test_chunks_match_one_chunk)."""
import ctypes

import numpy as np
import pytest
import torch

from util import build_gpt, load_golden, top2_gap

pytestmark = pytest.mark.gpu

XL3 = dict(n_layer=3, n_head=20, dim=1280, vocab_size=16384, block_size=256, cls_token_num=120, model_type="t2i", caption_dim=2048)
HD128 = dict(XL3, n_head=10)


def _model(dt, kv="auto", **cfg):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(1234)
    m = Transformer(ModelArgs(**cfg))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dt).eval()
    m.set_kv_cache(kv)
    return m


def _captions(lens, C, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((1, n, C)).astype(np.float32) for n in lens]     # the .npy layout of extract_t5_feature.py


def _run(llm, feats, sp, waves):
    """waves: [(steps to run before the wave, [caption indices])]; returns {caption index: tokens}. Request ids follow the caption
    indices whatever the arrival order, so that request r keeps its RNG stream (seed base + r) in every schedule."""
    order = [i for _, w in waves for i in w]
    llm.request_counter = iter(order)
    outs = []
    for steps, w in waves:
        for _ in range(steps):
            outs += llm.step()
        for i in w:
            llm.add_request(prompt_embeds=feats[i], sampling_params=sp)
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): o.outputs[0].token_ids for o in outs}
    assert sorted(got) == sorted(order) and all(len(t) == sp.max_tokens for t in got.values())
    return got


def test_fp32_exact_against_oracle_in_three_waves():
    from llamagen_b200.serve import LLM, SamplingParams
    from oracle import GPTOracle
    g = load_golden("gpt_t2i.pt")
    T, C, S = g["cfg"]["cls_token_num"], g["cfg"]["caption_dim"], g["S"]
    lens = [5, 37, 64, 120, 9, 88, 17, 120]
    feats = _captions(lens, C, 7)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=3, seed=3)
    sp = SamplingParams(temperature=0.0, max_tokens=S)
    # wave 1 takes two of three slots; in wave 2 one request joins mid-sequence and two wait for wave 1's slots (stale K / V);
    # wave 3 arrives while wave 2 runs
    got = _run(llm, feats, sp, [(0, [0, 1]), (3, [2, 3, 4]), (S + 5, [5, 6, 7])])
    orc = GPTOracle(g["state_dict"], g["cfg"])
    for i, f in enumerate(feats):
        n = f.shape[1]
        emb, mask = torch.zeros(1, T, C), torch.zeros(1, T)          # sample_t2i.py:89-106: right-padded, then the per-prompt loop
        emb[0, :n], mask[0, :n] = torch.from_numpy(f[0]), 1
        new_mask = torch.flip(mask, dims=[-1])
        new_emb = torch.cat([emb[0, n:], emb[0, :n]])[None]
        ref, _ = orc.generate(new_emb * new_mask[:, :, None], S, emb_masks=new_mask, cfg_scale=4.0, sample_logits=False)
        assert got[i] == ref[0].tolist(), f"caption {i} (length {n})"


@pytest.mark.parametrize("shape, dt, kv", [
    (XL3, torch.bfloat16, "auto"), (XL3, torch.float16, "auto"), (XL3, torch.bfloat16, "fp8"), (HD128, torch.bfloat16, "auto"),
], ids=["xl3_bf16", "xl3_f16", "xl3_bf16_kv_fp8", "hd128_bf16"])
def test_tokens_do_not_depend_on_the_schedule(shape, dt, kv):
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(dt, kv, **shape)
    lens = [5, 37, 64, 120, 17, 90, 1]
    feats = _captions(lens, shape["caption_dim"], 11)
    sp = SamplingParams(temperature=1.0, top_k=1000, top_p=1.0, max_tokens=24)
    n = len(lens)
    runs = []
    for waves in ([(0, list(range(n)))],                                   # all queued at once
                  [(0, [0, 1]), (3, [2, 3, 4]), (7, [5, 6])],             # staggered waves
                  [(0, list(reversed(range(n))))]):                       # reversed: other slots, other co-runners
        llm = LLM(m, cfg_scale=7.5, max_num_seqs=5, seed=21)
        runs.append(_run(llm, feats, sp, waves))
    assert runs[0] == runs[1] == runs[2]
    assert len({tuple(t) for t in runs[0].values()}) == n                 # the requests really differ


def test_join_writes_only_its_slot_rows():
    from llamagen_b200 import _lib
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(torch.bfloat16, **XL3)
    feats = _captions([40, 120, 7], XL3["caption_dim"], 5)
    B = 3
    llm = LLM(m, cfg_scale=7.5, max_num_seqs=B, seed=1)
    for f in feats[:2]:
        llm.add_request(prompt_embeds=f, sampling_params=SamplingParams(top_k=1000, max_tokens=32))
    for _ in range(6):
        llm.step()                                                        # slots 0, 1 run; slot 2 is free
    st = llm._state
    st["cond"][2].copy_(llm._caption(feats[2])[0])
    st["mask"][2].copy_(llm._caption(feats[2])[1])
    buf = m._workspace
    off = (buf.data_ptr() + 255) // 256 * 256 - buf.data_ptr()
    rows, max_seq = m._ws_shape
    H, hd, L, T = XL3["n_head"], XL3["dim"] // XL3["n_head"], XL3["n_layer"], XL3["cls_token_num"]
    kbytes = L * rows * H * max_seq * hd * 2
    starts = (0, (kbytes + 255) // 256 * 256)                             # K, then V (lg_engine::carve_kv)
    may = torch.zeros(buf.numel() - off, dtype=torch.bool, device="cuda")
    for start in starts:
        view = may[start:start + kbytes].view(L, rows, H, max_seq, hd * 2)
        view[:, [2, B + 2], :, :T] = True
    torch.cuda.synchronize()
    before = buf[off:].clone()
    ws, ws_bytes = m._slot_scratch(True)
    lib = _lib.load()
    _lib.check(lib.lg_prefill_slot(m.engine(), _lib.ptr(st["cond"][2]), _lib.ptr(st["mask"][2]), T, 2, B, 1, ws, ws_bytes,
                                   _lib.ptr(st["join_logits"]), _lib.current_stream(torch.device("cuda"))), "lg_prefill_slot")
    torch.cuda.synchronize()
    after = buf[off:]
    changed = after != before
    assert not bool((changed & ~may).any()), "lg_prefill_slot wrote outside its slot's K / V rows"
    for start in starts:                                                  # and it did write K and V of both of the slot's rows
        view = changed[start:start + kbytes].view(L, rows, H, max_seq, hd * 2)
        assert bool(view[:, 2, :, :T].any()) and bool(view[:, B + 2, :, :T].any())
    assert bool(torch.isfinite(st["join_logits"]).all())


@pytest.mark.parametrize("case", ["xl3_bf16", "golden_f32"])
def test_one_slot_without_cfg_is_generate_bit_for_bit(case):
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    if case == "golden_f32":
        g = load_golden("gpt_t2i.pt")
        m, C, S, topk = build_gpt(g["cfg"], g["state_dict"], torch.float32), g["cfg"]["caption_dim"], g["S"], 100
    else:
        m, C, S, topk = _model(torch.bfloat16, **XL3), XL3["caption_dim"], 32, 1000
    feats = _captions([5, 120, 64], C, 9)
    sp = SamplingParams(temperature=1.0, top_k=topk, max_tokens=S)
    got = _run(LLM(m, cfg_scale=1.0, max_num_seqs=1, seed=40), feats, sp, [(0, [0, 1, 2])])
    for r, f in enumerate(feats):
        llm = LLM(m, cfg_scale=1.0, max_num_seqs=1)
        c, mk = llm._caption(f)
        ref = generate(m, c[None].cuda(), S, emb_masks=mk[None].cuda(), cfg_scale=1.0, temperature=1.0, top_k=topk, seed=40 + r)
        assert ref[0].cpu().tolist() == got[r], f"caption {r}"


def test_cfg_greedy_agrees_with_generate_up_to_a_near_tie():
    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m = _model(torch.bfloat16, **XL3)
    S = 48
    feats = _captions([5, 37, 120], XL3["caption_dim"], 13)
    got = _run(LLM(m, cfg_scale=7.5, max_num_seqs=1, seed=0), feats, SamplingParams(temperature=0.0, max_tokens=S), [(0, [0, 1, 2])])
    for r, f in enumerate(feats):
        c, mk = LLM(m, cfg_scale=7.5, max_num_seqs=1)._caption(f)
        c, mk = c[None].cuda(), mk[None].cuda()
        ref = generate(m, c, S, emb_masks=mk, cfg_scale=7.5, sample_logits=False)[0].cpu().tolist()
        if ref == got[r]:
            continue
        k = next(i for i in range(S) if ref[i] != got[r][i])
        _, logits = generate(m, c, S, emb_masks=mk, cfg_scale=7.5, sample_logits=False, return_logits=True,
                             teacher=torch.tensor([got[r]], dtype=torch.int32, device="cuda"))
        gap = top2_gap(logits[k, 0].float().cpu()).item()
        print(f"[caption {r}] first difference at token {k}, top-1 / top-2 gap {gap:.4f}")
        assert gap <= 0.5, (r, k, gap)
