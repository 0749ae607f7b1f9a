"""GPU parity AT the configurations bench.py measures and BASELINE.json names (VERDICT r1, item 2).

Every test runs the bf16 engine teacher-forced on the fp32 oracle's greedy stream and compares the CFG-mixed logits of
EVERY step with (a) the fp32 oracle on the same bf16-rounded weights and (b) the bf16 oracle (like for like). The oracle
(oracle/gpt_oracle.py, pinned to the live reference) takes device tensors, so it runs on the same GPU in plain torch
(fp32 matmuls with TF32 off) — a CPU run of GPT-L at R=128 for 256 steps would take minutes per case.

Bound (same protocol as tests/test_gpt_gpu.py::_bf16_parity): the engine may deviate from either oracle by at most
1.5x the ORACLE'S OWN bf16-vs-fp32 spread on these logits (+0.02 max / +0.005 mean); arg-max and the sampled greedy token
must agree wherever the fp32 oracle's top-1/top-2 gap exceeds twice that bound. The MEASURED errors are printed next to
the bounds (pytest -s) and appended to gpurun_out/parity_report.jsonl so a regression inside the slack stays visible.

    C2  GPT-L  c2i 16x16, B=64 (R=128, one decode chain), all 256 tokens       <- the benchmarked configuration
    C2' GPT-L  c2i 16x16, B=32 (R=64), all 256 tokens                          <- north_star's per-GPU point (B=256 / 8 GPUs)
    C3  GPT-XL c2i 24x24, contexts to 577 keys, R=4 (small-row path) and R=16 (wgmma path)
    C5  GPT-XL t2i 32x32, T=120 prefill with ragged emb_masks + 1024 tokens (context 1144), R=4 and R=16
    C4  GPT-3B (head_dim 100) full depth, R=32, 40 tokens
"""
import json
import os

import pytest
import torch

from oracle import GPTOracle
from util import oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _registry(name, seed, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(seed)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)              # SURVEY G1: the stock init zeroes the head
    return m.to(device="cuda", dtype=torch.bfloat16).eval()


def _dev_state(model, dtype=None):
    return {k: (v.detach().to(dtype) if dtype is not None else v.detach()) for k, v in model.state_dict().items()}


def _report(tag, **vals):
    line = {"test": tag, **{k: (round(v, 6) if isinstance(v, float) else v) for k, v in vals.items()}}
    print("\n[parity] " + json.dumps(line))
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", "parity_report.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")
    except OSError:
        pass


def parity_on_device(tag, m, cond, S, emb_masks=None, cfg_scale=4.0):
    """Teacher-forced bf16 engine vs fp32 + bf16 oracle, everything resident on the GPU. Returns the measured errors."""
    from llamagen_b200 import generate
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = oracle_cfg(m)
    cond = cond.cuda()
    em = None if emb_masks is None else emb_masks.cuda()
    with torch.no_grad():
        cond32 = cond.float() if cond.is_floating_point() else cond
        ref_t, ref_l = GPTOracle(_dev_state(m, torch.float32), cfg).generate(cond32, S, emb_masks=em, cfg_scale=cfg_scale,
                                                                            sample_logits=False)
        _, b16_l = GPTOracle(_dev_state(m), cfg).generate(cond, S, emb_masks=em, cfg_scale=cfg_scale, sample_logits=False,
                                                         teacher=ref_t)
    spread_max = (b16_l - ref_l).abs().max().item()
    spread_mean = (b16_l - ref_l).abs().mean().item()
    tol_max, tol_mean = 1.5 * spread_max + 0.02, 1.5 * spread_mean + 0.005
    toks, logits = generate(m, cond, S, emb_masks=em, cfg_scale=cfg_scale, sample_logits=False, return_logits=True,
                            teacher=ref_t.clone())
    torch.cuda.synchronize()
    errs = {}
    for name, other in (("fp32_oracle", ref_l), ("bf16_oracle", b16_l)):
        e = (logits - other).abs()
        errs[name] = (e.max().item(), e.mean().item())
    del b16_l
    decisive = top2_gap(ref_l) > 2 * tol_max
    agree_argmax = bool(torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive]))
    agree_tokens = bool(torch.equal(toks.t()[decisive], ref_t.t()[decisive]))
    _report(tag, rows=int((2 if cfg_scale > 1 else 1) * cond.shape[0]), steps=int(S), logit_std=ref_l.std().item(),
            oracle_bf16_vs_fp32_max=spread_max, oracle_bf16_vs_fp32_mean=spread_mean, bound_max=tol_max, bound_mean=tol_mean,
            err_vs_fp32_oracle_max=errs["fp32_oracle"][0], err_vs_fp32_oracle_mean=errs["fp32_oracle"][1],
            err_vs_bf16_oracle_max=errs["bf16_oracle"][0], err_vs_bf16_oracle_mean=errs["bf16_oracle"][1],
            decisive_frac=decisive.float().mean().item(), argmax_agree=agree_argmax, tokens_agree=agree_tokens)
    for name, (emax, emean) in errs.items():
        assert emax <= tol_max, (tag, name, emax, tol_max)
        assert emean <= tol_mean, (tag, name, emean, tol_mean)
    assert agree_argmax and agree_tokens, tag
    return errs


@pytest.mark.parametrize("B", [64, 32])
def test_c2_gpt_l_bench_config_full_sequence(B):
    """BASELINE configs[1]: GPT-L c2i 16x16, cfg 4.0. B=64 is the benchmarked batch (R=128 rows in one decode chain: a
    27 MB GPT-L layer is more than a third of the H100's 50 MB L2; contexts to 257 keys on attn_tma_kernel); B=32 is the
    per-GPU batch of north_star's B=256-over-8-GPUs point."""
    m = _registry("GPT-L", 1, block_size=256, vocab_size=16384)
    torch.manual_seed(B)
    parity_on_device(f"C2 GPT-L c2i S=256 B={B}", m, torch.randint(0, 1000, (B,)), 256)


@pytest.mark.parametrize("B", [2, 8])
def test_c3_gpt_xl_c2i_24x24(B):
    """BASELINE configs[2] shape: GPT-XL c2i 24x24 = 576 tokens (contexts to 577 keys). B=2 -> R=4 (small-row path),
    B=8 -> R=16 (wgmma GEMMs + TMA attention)."""
    m = _registry("GPT-XL", 2, block_size=576, vocab_size=16384)
    torch.manual_seed(10 + B)
    parity_on_device(f"C3 GPT-XL c2i S=576 B={B}", m, torch.randint(0, 1000, (B,)), 576)


@pytest.mark.parametrize("B", [2, 8])
def test_c5_gpt_xl_t2i_32x32_ragged_masks(B):
    """BASELINE configs[4] shape: GPT-XL t2i, T=120 caption prefill with ragged left-padded emb_masks, then 1024 tokens
    (context 1144). B=8 is C5's per-GPU batch (R=16)."""
    m = _registry("GPT-XL", 3, block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i")
    torch.manual_seed(20 + B)
    T = 120
    em = torch.zeros(B, T)
    lens = torch.randint(8, T + 1, (B,))
    lens[0] = T                                              # one full-length caption, the rest ragged
    for b in range(B):
        em[b, T - int(lens[b]):] = 1                         # left padding: valid features sit at the right end
    cond = (torch.randn(B, T, 2048) * em[:, :, None]).bfloat16()
    parity_on_device(f"C5 GPT-XL t2i T=120 S=1024 B={B}", m, cond, 1024, emb_masks=em, cfg_scale=7.5)


def test_c4_gpt_3b_full_depth():
    """BASELINE configs[3] model: GPT-3B (24 layers, dim 3200, head_dim 100) at C4's per-GPU batch (B=16, R=32), 40 tokens."""
    m = _registry("GPT-3B", 4, block_size=576, vocab_size=16384)
    torch.manual_seed(4)
    parity_on_device("C4 GPT-3B c2i B=16 S=40", m, torch.randint(0, 1000, (16,)), 40)
