"""GPU: fp16 models (the samplers' --precision fp16) through the same wgmma / mma.sync / TMA-attention / GEMV kernels as bf16.

Rounding points are the reference's with fp16 in place of bf16 (weights, activations and the KV cache fp16, RMSNorm normalised in
fp32 and rounded, RoPE in fp32, the head's logits rounded to fp16 once). The GEMM test bounds the error by the operands' own
magnitude, so an operand silently converted to bf16 fails it; the model tests calibrate their bounds on the fp16 oracle's own
spread from the fp32 oracle, like the bf16 tests do."""
import ctypes

import pytest
import torch

from oracle import GPTOracle, cfg_mix_oracle, sample_oracle
from test_gemm_gpu import SHAPES
from util import build_gpt, cpu_state, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

# N % 128 != 0: the wgmma kernel needs 128-feature tiles, so these run on the mma.sync fallback even with LG_GEMM_TC=1
FALLBACK_SHAPES = [(16, 1000, 1024), (40, 2000, 768), (130, 712, 2048)]


def run_gemm_f16(x, w):
    from llamagen_b200 import _lib
    lib = _lib.load()
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=torch.float32, device=x.device)
    scratch = torch.empty(16 * M * N + 1024, dtype=torch.float32, device=x.device)
    _lib.check(lib.lg_test_gemm(_lib.ptr(x), _lib.ptr(w), M, N, K, _lib.LG_DTYPE_F16, _lib.ptr(y), _lib.ptr(scratch),
                                ctypes.c_size_t(scratch.numel() * 4), _lib.current_stream(x.device)), "lg_test_gemm")
    return y


@pytest.mark.parametrize("M,N,K", SHAPES + FALLBACK_SHAPES)
@pytest.mark.parametrize("tc", ["1", "0"])
def test_gemm_f16(M, N, K, tc, monkeypatch):
    """skinny, wgmma and mma.sync in fp16 against float64 of the same fp16 operands, element by element:
    |y - ref| <= 2^-16 * (|x| |w|^T). An operand rounded to bf16 misses that by ~2^-9 / sqrt(K) of the same sum."""
    monkeypatch.setenv("LG_GEMM_TC", tc)
    torch.manual_seed(M * 7 + N + K)
    x = (torch.randn(M, K, device="cuda") * 0.5).half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    y = run_gemm_f16(x, w).double()
    ref = x.double() @ w.double().t()
    bound = 2.0 ** -16 * (x.double().abs() @ w.double().abs().t())
    excess = ((y - ref).abs() - bound).max().item()
    assert excess <= 0.0, excess


def _gen(model, cond, S, em, **kw):
    from llamagen_b200 import generate
    toks, logits = generate(model, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), sample_logits=False,
                            return_logits=True, **kw)
    torch.cuda.synchronize()
    return toks.cpu(), logits.cpu()


def _f16_parity(m, cond, S, em=None):
    """fp16 engine vs the fp32 oracle (same fp16-rounded weights) and the fp16 oracle, teacher-forced on the fp32 oracle's greedy
    stream: at most 1.5x the fp16 oracle's own spread from the fp32 oracle, plus floors one eighth of the bf16 ones (fp16 has
    3 more mantissa bits). arg-max must agree where the fp32 oracle's top-1 / top-2 gap exceeds twice the bound.
    Returns the engine's logits and the max bound."""
    cfg = oracle_cfg(m)
    cond32 = cond if cond.dtype == torch.long else cond.float()
    ref_t, ref_l = GPTOracle(cpu_state(m, torch.float32), cfg).generate(cond32, S, emb_masks=em, cfg_scale=4.0, sample_logits=False)
    _, h_l = GPTOracle(cpu_state(m), cfg).generate(cond, S, emb_masks=em, cfg_scale=4.0, sample_logits=False, teacher=ref_t)
    tol_max = 1.5 * (h_l - ref_l).abs().max().item() + 0.0025
    tol_mean = 1.5 * (h_l - ref_l).abs().mean().item() + 0.000625
    toks, logits = _gen(m, cond, S, em, cfg_scale=4.0, teacher=ref_t.clone())
    for other in (ref_l, h_l):
        err = (logits - other).abs()
        assert err.max().item() <= tol_max, (err.max().item(), tol_max)
        assert err.mean().item() <= tol_mean, (err.mean().item(), tol_mean)
    decisive = top2_gap(ref_l) > 2 * tol_max
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    assert torch.equal(toks.t()[decisive], ref_t.t()[decisive])
    return logits, tol_max


def _golden_f16(name):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float16)
    cond = g["cond"] if name == "gpt_c2i.pt" else g["cond"].half()
    return g, m, cond


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_f16_tiny_goldens_teacher_forced(name):
    g, m, cond = _golden_f16(name)
    _f16_parity(m, cond, g["S"], g["emb_masks"])


def _registry_model(name, dtype, seed, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(seed)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dtype).eval()


@pytest.mark.parametrize("B", [1, 9, 40])
def test_gpt_l_f16_teacher_forced(B):
    """B = 1: the R <= 8 column-owner GEMV path (gemv_small.cu); B = 9 / 40: the wgmma split-K GEMM."""
    m = _registry_model("GPT-L", torch.float16, 1, block_size=256, vocab_size=16384)
    torch.manual_seed(B)
    _f16_parity(m, torch.randint(0, 1000, (B,)), 6)


def test_gpt_3b_head_dim_100_f16():
    """GPT-3B's head_dim 100: 112-wide KV rows on the TMA attention."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(3)
    m = Transformer(ModelArgs(n_layer=4, n_head=32, dim=3200, block_size=576, vocab_size=16384))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.float16).eval()
    _f16_parity(m, torch.tensor([1, 2, 3]), 5)


def test_t2i_f16_masked_prefill_tensor_core_attention():
    """t2i with a 120-token condition and emb_masks at B = 8: the condition prefill runs on attn_prefill_tc_kernel."""
    g = load_golden("gpt_t2i.pt")
    m = build_gpt(g["cfg"], g["state_dict"], torch.float16)
    B = 8
    torch.manual_seed(4)
    em = torch.zeros(B, 120)
    for b, n in enumerate((5, 61, 120, 17, 90, 1, 33, 100)):
        em[b, -n:] = 1
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).half()
    _f16_parity(m, cond, 5, em)


def test_f16_is_closer_to_fp32_than_bf16():
    """The same GPT-L weights in fp16 and in bf16: fp16's mean logit error against the fp32 oracle must be at most half of bf16's
    (one eighth is expected from the 3 extra mantissa bits)."""
    torch.manual_seed(1)
    from llamagen_b200 import GPT_models
    base = GPT_models["GPT-L"](block_size=256, vocab_size=16384)
    base.output.weight.data.normal_(std=0.02)
    cond = torch.randint(0, 1000, (9,), generator=torch.Generator().manual_seed(9))
    ref_t, ref_l = GPTOracle(cpu_state(base, torch.float32), oracle_cfg(base)).generate(cond, 6, cfg_scale=4.0, sample_logits=False)
    err = {}
    for dt in (torch.float16, torch.bfloat16):
        m = GPT_models["GPT-L"](block_size=256, vocab_size=16384)
        m.load_state_dict(base.state_dict())
        m = m.to(device="cuda", dtype=dt).eval()
        _, logits = _gen(m, cond, 6, None, cfg_scale=4.0, teacher=ref_t.clone())
        err[dt] = (logits - ref_l).abs().mean().item()
        del m
    assert err[torch.float16] <= 0.5 * err[torch.bfloat16], err


def test_f16_paths_agree(monkeypatch):
    """CUDA-core attention and the mma.sync GEMM stay within the calibrated bound of the default path; the default path (CUDA-graph
    replay, fused sampling tail) is bit-identical to two-chain decode, to the unfused tail and to eager launches with the tail off
    and on (with it, the sample kernel advances the position counter that the next step's fused attention reads)."""
    g = load_golden("gpt_c2i.pt")
    B, S = 48, 8
    cond = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(3))
    m = build_gpt(g["cfg"], g["state_dict"], torch.float16)
    _, tol = _f16_parity(m, cond, S)
    teacher = torch.randint(0, g["cfg"]["vocab_size"], (B, S), generator=torch.Generator().manual_seed(1), dtype=torch.int32)

    def run(env):
        for k in ("LG_ATTN_TMA", "LG_GEMM_TC", "LG_NO_GRAPH", "LG_SPLIT", "LG_FUSE_TAIL"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        mm = build_gpt(g["cfg"], g["state_dict"], torch.float16)
        forced = _gen(mm, cond, S, None, cfg_scale=4.0, teacher=teacher)
        from llamagen_b200 import generate
        sampled = generate(mm, cond.cuda(), S, cfg_scale=4.0, temperature=1.0, top_k=50, top_p=1.0, sample_logits=True, seed=5).cpu()
        return forced[0], forced[1], sampled

    base = run({"LG_SPLIT": "1"})
    for env in ({"LG_ATTN_TMA": "0", "LG_SPLIT": "1"}, {"LG_GEMM_TC": "0", "LG_SPLIT": "1"}):
        _, logits, _ = run(env)
        assert (logits - base[1]).abs().max().item() <= tol, env
    for env in ({"LG_SPLIT": "2"}, {"LG_FUSE_TAIL": "0", "LG_SPLIT": "1"}, {"LG_NO_GRAPH": "1", "LG_FUSE_TAIL": "0", "LG_SPLIT": "1"},
                {"LG_NO_GRAPH": "1", "LG_SPLIT": "1"}):
        other = run(env)
        for i in range(3):
            assert torch.equal(other[i], base[i]), (env, i)


@pytest.mark.parametrize("k,p,cfg", [(0, 1.0, 4.0), (2000, 1.0, 4.0), (1000, 0.9, 1.0), (1, 1.0, 7.5)])
def test_sample_round_f16(k, p, cfg):
    """lg_sample with round dtype F16: the oracle filter of the fp16-rounded logits (CFG mix and softmax in fp32)."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(k + 1)
    B, V = 4, 16384
    mix = cfg > 1.0
    logits = torch.randn(2 * B if mix else B, V) * 2.7
    rounded = logits.half().float()
    ridx, rprobs = sample_oracle(cfg_mix_oracle(rounded, cfg) if mix else rounded, temperature=1.0, top_k=k, top_p=p,
                                 sample_logits=False)
    idx = torch.empty(B, dtype=torch.int32, device="cuda")
    probs = torch.empty(B, V, dtype=torch.float32, device="cuda")
    sc = _lib.SampleCfg(cfg, -1, 1.0, k, p, 1, 1)
    x = logits.cuda().contiguous()
    _lib.check(lib.lg_sample(_lib.ptr(x), B, V, 1 if mix else 0, _lib.LG_DTYPE_F16, ctypes.byref(sc), 0, _lib.ptr(idx),
                             _lib.ptr(probs), _lib.current_stream(x.device)), "lg_sample")
    probs = probs.cpu()
    if p >= 1.0:
        assert torch.equal(probs == 0, rprobs == 0)
    else:   # the nucleus boundary depends on fp32 cumsum order
        assert ((probs == 0) != (rprobs == 0)).sum().item() <= 2 * B
    assert (probs - rprobs).abs().max().item() <= (1e-6 if p >= 1.0 else 1e-3)
    assert torch.equal(idx.cpu().long(), ridx.view(-1))


def test_f16_forward_logits_are_f16_values():
    """lg_prefill / lg_decode_step round the head's logits to fp16 (gpt.py:368 `.float()` of an fp16 tensor)."""
    g, m, cond = _golden_f16("gpt_c2i.pt")
    cond = cond.cuda()
    B = cond.shape[0]
    m.setup_caches(2 * B, 1 + g["S"], torch.float16)
    logits, _ = m(None, torch.cat([cond, torch.full_like(cond, m.num_classes)]), torch.arange(0, 1, device="cuda"))
    assert torch.equal(logits, logits.half().float())
    tok = logits[:, -1].argmax(-1, keepdim=True)
    logits, _ = m(tok, None, torch.tensor([1], device="cuda", dtype=torch.int))
    assert torch.equal(logits, logits.half().float())


def test_serve_llm_f16_matches_generate():
    from llamagen_b200 import GPT_models, generate
    from llamagen_b200.serve import LLM, SamplingParams
    torch.manual_seed(0)
    gpt = GPT_models["GPT-B"](vocab_size=16384, block_size=64, num_classes=1000, cls_token_num=1, model_type="c2i")
    gpt = gpt.to("cuda", torch.float16).eval()
    gpt.output.weight.data.normal_(std=0.02)
    S, slots = 64, 4
    sp = SamplingParams(temperature=1.0, top_p=1.0, top_k=2000, max_tokens=S)
    llm = LLM(gpt, cfg_scale=4.0, num_classes=1000, max_num_seqs=slots, seed=11)
    labels = [207, 360, 387, 974, 88]
    outs = []
    for c in labels:
        llm.add_request([c], sp)
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): o.outputs[0].token_ids for o in outs}
    for rid, c in enumerate(labels):
        ref = generate(gpt, torch.full((slots,), c, device="cuda"), S, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, seed=11 + rid)
        assert ref[0].cpu().tolist() == got[rid], rid


def test_sample_c2i_cli_fp16(tmp_path, monkeypatch):
    from llamagen_b200.sample import sample_c2i
    monkeypatch.chdir(tmp_path)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--image-size", "256", "--cfg-scale", "4.0",
                                                 "--top-k", "2000", "--seed", "1", "--precision", "fp16"])
    sample_c2i.main(args)
    from PIL import Image
    img = Image.open(tmp_path / "sample_c2i.png")
    assert img.size == (4 * 256 + 5 * 2, 2 * 256 + 3 * 2)
