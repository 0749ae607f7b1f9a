"""GPU parity of the AR engine (lg_generate / lg_prefill / lg_decode_step) against the oracle and the
reference-produced golden vectors.

Protocol (SURVEY §8c): fp32 "exact" mode must reproduce the fp32 oracle's greedy token ids bit-exactly and
its logits to 1e-4; bf16 mode is checked teacher-forced at every step against the fp32 oracle run on the
same bf16-rounded weights (tolerance 4e-2 at logit scale ~2.7 = the oracle's own bf16-vs-fp32 spread) with
arg-max agreement wherever the oracle's top-1/top-2 gap exceeds twice the tolerance."""
import pytest
import torch

from oracle import GPTOracle
from util import build_gpt, cpu_state, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-4
BF16_TOL = 4e-2


def _gen(model, cond, S, em, **kw):
    from llamagen_b200 import generate
    toks, logits = generate(model, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), sample_logits=False,
                            return_logits=True, **kw)
    torch.cuda.synchronize()
    return toks.cpu(), logits.cpu()


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
def test_fp32_matches_reference_golden(name, cfg_scale):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    toks, logits = _gen(m, g["cond"], g["S"], g["emb_masks"], cfg_scale=cfg_scale)
    ref_l = g[f"logits_cfg{cfg_scale}"]
    assert (logits - ref_l).abs().max().item() <= FP32_TOL
    assert torch.equal(toks, g[f"tokens_cfg{cfg_scale}"]), "greedy token ids must be bit-exact in fp32 mode"


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_fp32_cfg_interval_golden(name):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    toks, _ = _gen(m, g["cond"], g["S"], g["emb_masks"], cfg_scale=4.0, cfg_interval=3)
    assert torch.equal(toks, g["tokens_cfg4.0_int3"])


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_graph_replay_equals_eager(name, monkeypatch):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    t_graph, l_graph = _gen(m, g["cond"], g["S"], g["emb_masks"], cfg_scale=4.0)
    monkeypatch.setenv("LG_NO_GRAPH", "1")
    m2 = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    t_eager, l_eager = _gen(m2, g["cond"], g["S"], g["emb_masks"], cfg_scale=4.0)
    assert torch.equal(t_graph, t_eager) and torch.equal(l_graph, l_eager)


@pytest.mark.parametrize("name,eager", [("gpt_c2i.pt", False), ("gpt_t2i.pt", False), ("gpt_c2i.pt", True), ("gpt_t2i.pt", True)],
                         ids=["gpt_c2i.pt", "gpt_t2i.pt", "gpt_c2i.pt-eager", "gpt_t2i.pt-eager"])
def test_bf16_teacher_forced_vs_oracle(name, eager, monkeypatch):
    """eager: LG_NO_GRAPH=1, every decode step launched eagerly with the fused sampling tail (graph replay otherwise)."""
    if eager:
        monkeypatch.setenv("LG_NO_GRAPH", "1")
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.bfloat16)
    sd = cpu_state(m)                                   # bf16 weights
    cond = g["cond"] if name == "gpt_c2i.pt" else g["cond"].bfloat16()
    orc = GPTOracle(sd, g["cfg"])                       # bf16 oracle: same dtype, same rounding points
    ref_t, ref_l = orc.generate(cond, g["S"], emb_masks=g["emb_masks"], cfg_scale=4.0, sample_logits=False)
    toks, logits = _gen(m, cond, g["S"], g["emb_masks"], cfg_scale=4.0, teacher=ref_t[:, :].clone())
    assert (logits - ref_l).abs().max().item() <= BF16_TOL
    decisive = top2_gap(ref_l) > 2 * BF16_TOL
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    assert torch.equal(toks.t()[decisive], ref_t.t()[decisive])


def _registry_model(name, dtype, seed, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(seed)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)              # SURVEY G1
    return m.to(device="cuda", dtype=dtype).eval()


def test_gpt_b_fp32_greedy_bit_exact_vs_oracle():
    """BASELINE config C1 shape (GPT-B c2i 16x16, cfg 4.0) in the fp32 exact mode, truncated to 24 tokens."""
    m = _registry_model("GPT-B", torch.float32, 0, block_size=256, vocab_size=16384)
    cond = torch.tensor([207, 360])
    S = 24
    orc = GPTOracle(cpu_state(m), oracle_cfg(m))
    ref_t, ref_l = orc.generate(cond, S, cfg_scale=4.0, sample_logits=False)
    toks, logits = _gen(m, cond, S, None, cfg_scale=4.0)
    assert (logits - ref_l).abs().max().item() <= FP32_TOL
    assert torch.equal(toks, ref_t)


def _bf16_parity(m, cond, S):
    """bf16 engine vs the oracle, teacher-forced on the fp32 oracle's greedy stream. The tolerance is calibrated
    on the spot: the engine may deviate from the fp32 oracle (same bf16-rounded weights) by at most 1.5x the
    ORACLE'S OWN bf16-vs-fp32 spread on these CFG-mixed logits (cfg 4.0 amplifies rounding noise ~7x; for GPT-L
    that spread is max 0.22 / mean 0.04 at logit std 3.1, abs-max 13), and from the bf16 oracle (like for like)
    by the same bound; arg-max must agree wherever the fp32 oracle's top-1/top-2 gap exceeds 2x the bound."""
    cfg = oracle_cfg(m)
    ref_t, ref_l = GPTOracle(cpu_state(m, torch.float32), cfg).generate(cond, S, cfg_scale=4.0, sample_logits=False)
    _, b16_l = GPTOracle(cpu_state(m), cfg).generate(cond, S, cfg_scale=4.0, sample_logits=False, teacher=ref_t)
    spread_max = (b16_l - ref_l).abs().max().item()
    spread_mean = (b16_l - ref_l).abs().mean().item()
    tol_max, tol_mean = 1.5 * spread_max + 0.02, 1.5 * spread_mean + 0.005
    toks, logits = _gen(m, cond, S, None, cfg_scale=4.0, teacher=ref_t.clone())
    for other in (ref_l, b16_l):
        err = (logits - other).abs()
        assert err.max().item() <= tol_max, (err.max().item(), tol_max)
        assert err.mean().item() <= tol_mean, (err.mean().item(), tol_mean)
    decisive = top2_gap(ref_l) > 2 * tol_max
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    assert torch.equal(toks.t()[decisive], ref_t.t()[decisive])


@pytest.mark.parametrize("B", [1, 2, 3, 4, 9, 20, 40, 64])
def test_gpt_l_bf16_teacher_forced(B):
    """GPT-L bf16 (BASELINE config C2 model): B=1..4 exercise the small-row GEMV path (R=2..8), B=9 / 20 / 40 / 64 the
    tensor-core path with BM=32 / 64 / 128 / 128 tiles; B=64 is the bench batch."""
    m = _registry_model("GPT-L", torch.bfloat16, 1, block_size=256, vocab_size=16384)
    torch.manual_seed(B)
    _bf16_parity(m, torch.randint(0, 1000, (B,)), 6)


def test_gpt_3b_head_dim_100_bf16():
    """SURVEY G4: GPT-3B has head_dim 100 (not a multiple of 16). 4 layers of the 3B shape keep the CPU oracle fast."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(3)
    m = Transformer(ModelArgs(n_layer=4, n_head=32, dim=3200, block_size=576, vocab_size=16384))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    _bf16_parity(m, torch.tensor([1, 2, 3]), 5)


def test_forward_api_matches_generate_path():
    """Transformer.forward (prefill / decode, gpt.py:348-368 semantics) is usable by the reference's own Python loop."""
    g = load_golden("gpt_c2i.pt")
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    cond = g["cond"].cuda()
    B = cond.shape[0]
    cond2 = torch.cat([cond, torch.full_like(cond, m.num_classes)])
    m.setup_caches(2 * B, 1 + g["S"], torch.float32)
    logits, _ = m(None, cond2, torch.arange(0, 1, device="cuda"))
    mixed = logits[B:, -1] + (logits[:B, -1] - logits[B:, -1]) * 4.0
    ref = g["logits_cfg4.0"][0]
    assert (mixed.cpu() - ref).abs().max().item() <= FP32_TOL
    tok = mixed.argmax(-1, keepdim=True)
    logits, _ = m(torch.cat([tok, tok]), None, torch.tensor([1], device="cuda", dtype=torch.int))
    mixed = logits[B:, -1] + (logits[:B, -1] - logits[B:, -1]) * 4.0
    assert (mixed.cpu() - g["logits_cfg4.0"][1]).abs().max().item() <= FP32_TOL


def test_sampling_run_is_seed_reproducible_and_in_range():
    from llamagen_b200 import generate
    m = _registry_model("GPT-B", torch.bfloat16, 5, block_size=256, vocab_size=16384)
    cond = torch.randint(0, 1000, (4,), device="cuda")
    a = generate(m, cond, 32, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, seed=11)
    b = generate(m, cond, 32, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, seed=11)
    c = generate(m, cond, 32, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True, seed=12)
    assert a.dtype == torch.int32 and tuple(a.shape) == (4, 32)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert int(a.min()) >= 0 and int(a.max()) < 16384


def test_attention_kernels_agree_large_batch_t2i(monkeypatch):
    """The TMA attention kernel, fused with the QKV epilogue (the default) and unfused, must agree with the CUDA-core kernel on a
    masked t2i decode at a large batch (rows * heads = 640)."""
    g = load_golden("gpt_t2i.pt")
    B, S = 160, 6
    torch.manual_seed(0)
    em = torch.zeros(B, 120)
    lens = torch.randint(3, 120, (B,))
    for b in range(B):
        em[b, -int(lens[b]):] = 1
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).bfloat16()
    outs = {}
    for tag, env in (("v1", {"LG_ATTN_TMA": "1", "LG_FUSE_QKV": "1"}),          # default: fused QKV epilogue
                     ("v1_unfused", {"LG_ATTN_TMA": "1", "LG_FUSE_QKV": "0"}),
                     ("cuda_core", {"LG_ATTN_TMA": "0", "LG_FUSE_QKV": "1"})):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        m = build_gpt(g["cfg"], g["state_dict"], torch.bfloat16)
        teacher = torch.randint(0, 512, (B, S), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
        _, logits = _gen(m, cond, S, em, cfg_scale=4.0, teacher=teacher)
        outs[tag] = logits
    for tag in ("v1", "v1_unfused"):
        err = (outs[tag] - outs["cuda_core"]).abs().max().item()
        assert err <= BF16_TOL, (tag, err)


def test_multi_chain_decode_is_bit_identical(monkeypatch):
    """Large batches can be decoded as two independent half-batch chains (LG_SPLIT=2) on their own streams and CUDA graphs.
    Every image's arithmetic is unchanged, so tokens, logits AND sampled streams must equal the single-chain run bit for bit."""
    g = load_golden("gpt_c2i.pt")
    B, S = 48, 10
    cond = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(3))
    outs = {}
    for split in ("1", "2"):
        monkeypatch.setenv("LG_SPLIT", split)
        m = build_gpt(g["cfg"], g["state_dict"], torch.bfloat16)
        toks, logits = _gen(m, cond, S, None, cfg_scale=4.0)
        from llamagen_b200 import generate
        sampled = generate(m, cond.cuda(), S, cfg_scale=4.0, temperature=1.0, top_k=50, top_p=1.0, sample_logits=True, seed=5).cpu()
        outs[split] = (toks, logits, sampled)
    for i in range(3):
        assert torch.equal(outs["2"][i], outs["1"][i]), i


@pytest.mark.parametrize("B", [1, 3, 4])
def test_small_row_decode_path(B, monkeypatch):
    """R = 2B <= 8 rows take the column-owner tensor-core GEMV path (gemv_small.cu: RMSNorm in the prologue, residual /
    SwiGLU in the epilogue, 5 kernels per layer). It must meet the same oracle bound as the batched path and agree with
    the batched path itself (same rounding points; only fp32 summation order differs) on a teacher-forced stream."""
    m = _registry_model("GPT-B", torch.bfloat16, 2, block_size=256, vocab_size=16384)
    torch.manual_seed(10 + B)
    cond = torch.randint(0, 1000, (B,))
    monkeypatch.setenv("LG_SMALL_R", "1")
    _bf16_parity(m, cond, 6)
    teacher = torch.randint(0, 16384, (B, 12), generator=torch.Generator().manual_seed(B), dtype=torch.int32)
    _, small = _gen(m, cond, 12, None, cfg_scale=4.0, teacher=teacher.clone())
    monkeypatch.setenv("LG_SMALL_R", "0")
    _, batched = _gen(m, cond, 12, None, cfg_scale=4.0, teacher=teacher.clone())
    err = (small - batched).abs()
    scale = batched.std().item()
    assert err.max().item() <= 0.08 * scale + 0.02, (err.max().item(), scale)
    assert err.mean().item() <= 0.01 * scale + 0.002, (err.mean().item(), scale)
    # sampled streams are reproducible on the small-row path as well
    monkeypatch.setenv("LG_SMALL_R", "1")
    from llamagen_b200 import generate
    a = generate(m, cond.cuda(), 16, cfg_scale=4.0, top_k=100, seed=3)
    b = generate(m, cond.cuda(), 16, cfg_scale=4.0, top_k=100, seed=3)
    assert torch.equal(a, b)


def test_small_grid_attention_parallel_chunks_long_context(monkeypatch):
    """Few (row, head) items take the 8-stage attention whose warp groups process the chunks of a context concurrently
    (attn_tma.cu, NST = 8). A 400-token context (> 8 x 32 keys) also exercises the per-group stage refill. It must agree
    with the 2-stage kernel (same arithmetic per key, different merge order) and stay greedy-identical where decisive."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(4)
    m = Transformer(ModelArgs(n_layer=2, n_head=4, dim=256, block_size=400, vocab_size=1024))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    cond = torch.tensor([3, 7])
    teacher = torch.randint(0, 1024, (2, 400), generator=torch.Generator().manual_seed(2), dtype=torch.int32)
    outs = {}
    for deep in ("1", "0"):
        monkeypatch.setenv("LG_ATTN_DEEP", deep)
        _, outs[deep] = _gen(m, cond, 400, None, cfg_scale=2.0, teacher=teacher.clone())
    err = (outs["1"] - outs["0"]).abs()
    assert err.max().item() <= BF16_TOL, err.max().item()
    assert err.mean().item() <= BF16_TOL / 10, err.mean().item()


def test_small_row_path_t2i_masked_condition(monkeypatch):
    """t2i decode at R = 6 rows on the small-row path: the 120-token condition prefix is masked per image (emb_masks,
    generate.py:154-163) inside the 8-stage attention; the batched path is the reference point."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(8)
    m = Transformer(ModelArgs(n_layer=3, n_head=4, dim=256, block_size=64, vocab_size=1024, cls_token_num=120, caption_dim=64,
                              model_type="t2i"))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    B, S = 3, 40
    em = torch.zeros(B, 120)
    for b, n in enumerate((5, 61, 120)):
        em[b, -n:] = 1                                           # left-padded: valid tokens at the right end
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).bfloat16()
    teacher = torch.randint(0, 1024, (B, S), generator=torch.Generator().manual_seed(5), dtype=torch.int32)
    outs = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("LG_SMALL_R", flag)
        _, outs[flag] = _gen(m, cond, S, em, cfg_scale=3.0, teacher=teacher.clone())
    # same rounding points on both paths, different fp32 summation order; a wrong mask or row mapping would show up as an
    # error of the order of the logit scale itself
    err = (outs["1"] - outs["0"]).abs()
    scale = outs["0"].std().item()
    assert err.max().item() <= 0.2 * scale + 0.05, (err.max().item(), scale)
    assert err.mean().item() <= 0.03 * scale + 0.005, (err.mean().item(), scale)



@pytest.mark.parametrize("B", [2, 12])
def test_t2i_prefill_tensor_core_attention(B, monkeypatch):
    """The T = 120 condition prefill runs its masked causal attention on the TMA + mma.sync kernel (attn_prefill_tc_kernel, one
    CTA per (row, head)); the CUDA-core kernel (one CTA per query) is the reference point, with ragged left-padded emb_masks
    (generate.py:154-163) and CFG twin rows. The prefill logits feed token 0, the cache feeds every later step."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(11)
    m = Transformer(ModelArgs(n_layer=3, n_head=4, dim=256, block_size=64, vocab_size=1024, cls_token_num=120, caption_dim=64,
                              model_type="t2i"))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    S = 24
    em = torch.zeros(B, 120)
    for b in range(B):
        em[b, -(1 + (37 * b + 5) % 120):] = 1                   # left-padded: valid tokens at the right end, 6..120 of them
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).bfloat16()
    teacher = torch.randint(0, 1024, (B, S), generator=torch.Generator().manual_seed(6), dtype=torch.int32)
    outs = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("LG_ATTN_PREFILL_TC", flag)
        _, outs[flag] = _gen(m, cond, S, em, cfg_scale=3.0, teacher=teacher.clone())
    err = (outs["1"] - outs["0"]).abs()
    scale = outs["0"].std().item()
    assert err.max().item() <= 0.2 * scale + 0.05, (err.max().item(), scale)
    assert err.mean().item() <= 0.03 * scale + 0.005, (err.mean().item(), scale)
    assert err[0].max().item() <= 0.2 * scale + 0.05            # step 0 = the prefill's own logits


@pytest.mark.parametrize("B", [1, 2, 3, 4])
def test_small_row_decode_long_context_and_masks(B, monkeypatch):
    """Small-row path (R = 2B <= 8 rows) on a t2i model: masked 120-token condition prefix + a 300-token image (contexts to 420
    keys, past the 256 keys the 8-stage attention ring holds, so the ring refills). The batched path is the reference point."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(8)
    m = Transformer(ModelArgs(n_layer=3, n_head=4, dim=256, block_size=324, vocab_size=1024, cls_token_num=120, caption_dim=64,
                              model_type="t2i"))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    S = 300
    em = torch.zeros(B, 120)
    for b, n in enumerate((5, 61, 120, 33)[:B]):
        em[b, -n:] = 1
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).bfloat16()
    teacher = torch.randint(0, 1024, (B, S), generator=torch.Generator().manual_seed(5), dtype=torch.int32)
    outs = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("LG_SMALL_R", flag)
        _, outs[flag] = _gen(m, cond, S, em, cfg_scale=3.0, teacher=teacher.clone())
    err = (outs["1"] - outs["0"]).abs()
    scale = outs["0"].std().item()
    assert err.max().item() <= 0.2 * scale + 0.05, (err.max().item(), scale)
    assert err.mean().item() <= 0.03 * scale + 0.005, (err.mean().item(), scale)
