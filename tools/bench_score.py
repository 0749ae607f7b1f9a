"""Teacher-forced scoring throughput (llamagen_b200.score) on two workloads a likelihood user runs:
  * GPT-L c2i 256 px (16x16 tokens), B = 64, cfg off and cfg 4.0: the validation loss of a c2i checkpoint;
  * GPT-XL t2i 512 px (32x32 tokens, 120 caption positions), B = 8, cfg 7.5: guided likelihoods of text-to-image samples.
Each is timed with CUDA events after a warm-up, alternating with two baselines on the same GPU: the torch bf16 forward of the oracle
(the reference's ops: one condition forward + one multi-token forward through its KV cache) and, for c2i, the engine's
generate(teacher=tokens) (S sequential decode steps). Random weights with a N(0, 0.02) head; the work does not depend on them.
Prints one JSON line per workload (tokens/s, ms per pass, TFLOP/s from shape-computed FLOPs) with the card's name and power limit.

    python tools/bench_score.py [--iters 5] [--out bench_score.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def flops(m, B, T, S, nh):
    """Multiply-adds x 2 of one scoring pass: the layers' GEMMs over rows * seq positions, causal attention (QK^T and PV over
    the visible half of the seq x seq scores), the caption MLP (t2i) and the head over rows * S scored positions."""
    c = m.config
    D, F, L, V = c.dim, c.ffn_dim, c.n_layer, c.vocab_size
    rows, seq = nh * B, T + S - 1
    gemm = 2.0 * rows * seq * (4 * D * D + 3 * D * F) * L
    attn = 2.0 * 2 * rows * D * seq * (seq + 1) / 2 * L
    cap = 2.0 * rows * T * (c.caption_dim * D + D * D) if c.model_type == "t2i" else 0.0
    head = 2.0 * rows * S * D * V
    return gemm + attn + cap + head


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    from llamagen_b200 import GPT_models, generate, score
    from oracle import GPTOracle
    from score_oracle import score_oracle
    from util import oracle_cfg
    dev = "cuda"
    info = card()
    rows_out = []
    workloads = [("GPT-L", "c2i", 256, 64, 1.0), ("GPT-L", "c2i", 256, 64, 4.0), ("GPT-XL", "t2i", 512, 8, 7.5)]
    models = {}
    for name, kind, px, B, cfg in workloads:
        grid = px // 16
        key = (name, kind, px)
        if key not in models:
            torch.manual_seed(0)
            kw = dict(block_size=grid * grid, vocab_size=16384)
            if kind == "t2i":
                kw.update(cls_token_num=120, model_type="t2i")
            m = GPT_models[name](**kw)
            m.output.weight.data.normal_(std=0.02)
            models[key] = m.to(device=dev, dtype=torch.bfloat16).eval()
        m = models[key]
        T, S = m.cls_token_num, grid * grid
        g = torch.Generator(device=dev).manual_seed(1)
        toks = torch.randint(0, 16384, (B, S), device=dev, generator=g)
        if kind == "c2i":
            cond = torch.randint(0, 1000, (B,), device=dev, generator=g)
            em = None
        else:
            cond = (torch.randn(B, T, 2048, device=dev, generator=g) * 0.1).bfloat16()
            em = (torch.arange(T, device=dev)[None] >= torch.randint(0, T // 2, (B, 1), device=dev, generator=g)).float()
        nh = 2 if cfg > 1.0 else 1
        orc = GPTOracle({k: v.detach() for k, v in m.state_dict().items()}, oracle_cfg(m))
        ours = lambda: score(m, cond, toks, emb_masks=em, cfg_scale=cfg)
        base = lambda: score_oracle(orc, cond, toks, em, cfg)
        dec = (lambda: generate(m, cond, S, cfg_scale=cfg, sample_logits=False, teacher=toks)) if kind == "c2i" else None
        with torch.no_grad():
            for f in (ours, base, dec):
                if f is not None:
                    f()
            torch.cuda.synchronize()
            t_ours, t_base, t_dec = [], [], []
            for _ in range(2):                              # alternate the arms twice
                t_ours.append(timed(ours, args.iters))
                t_base.append(timed(base, max(1, args.iters // 2)))
                if dec is not None:
                    t_dec.append(timed(dec, 1))
        fl = flops(m, B, T, S, nh)
        tok = B * S
        ms = min(t_ours)
        row = {"workload": f"{name} {kind} {px}px B={B} cfg={cfg}", "scored_tokens": tok, "score_ms": round(ms, 3),
               "score_tokens_per_s": round(tok / ms * 1e3), "score_tflops": round(fl / ms / 1e9, 1),
               "torch_bf16_forward_ms": round(min(t_base), 3), "speedup_vs_torch": round(min(t_base) / ms, 2),
               "model_tflop_per_pass": round(fl / 1e12, 3), "score_ms_runs": [round(x, 3) for x in t_ours],
               "card": info}
        if t_dec:
            row.update({"generate_teacher_ms": round(min(t_dec), 3), "speedup_vs_generate_teacher": round(min(t_dec) / ms, 2)})
        print(json.dumps(row), flush=True)
        rows_out.append(row)
        del orc
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows_out, f, indent=1)


if __name__ == "__main__":
    main()
