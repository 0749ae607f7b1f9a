"""Timing of generate() calls whose decode steps all run eagerly: S - P - 1 = 3 decode steps, fewer than graph replay needs, so
every step is launched from the host and its first kernel waits for the previous step's sample kernel to complete.

    python tools/bench_eager_steps.py [--reps 20] [--out eager_steps.json]

The benchmark's model (GPT-L c2i, bf16, V = 16384, cfg 4.0, top-k 2000) at batch 64 (R = 128, batched decode path) and batch 1
(R = 2, small-row path), plain (P = 0, S = 4) and as a completion (P = 252, S = 256). Every number is a median [min, max] over
--reps CUDA-event timings of one call, after two warm-up calls. Random-init weights (output head N(0, 0.02)); what is timed does
not depend on their values."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--out", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eager_steps needs a CUDA device")
    from llamagen_b200 import GPT_models, generate
    torch.manual_seed(0)
    m = GPT_models["GPT-L"](block_size=256, vocab_size=16384)
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    res = {"card": card(), "workload": "GPT-L c2i bf16, cfg 4.0, top-k 2000; 3 decode steps after the first draw, all eager",
           "reps": args.reps}
    for B in (64, 1):
        cond = torch.randint(0, 1000, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
        pf = torch.randint(0, 16384, (B, 252), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        m.setup_caches(max_batch_size=2 * B, max_seq_length=1 + 256, dtype=torch.bfloat16)
        calls = {"plain_S4": lambda: generate(m, cond, 4, cfg_scale=4.0, top_k=2000, seed=3),
                 "prefix_P252_S256": lambda: generate(m, cond, 256, cfg_scale=4.0, top_k=2000, seed=3, prefix=pf)}
        for name, fn in calls.items():
            for _ in range(2):
                timed(fn)
            xs = [timed(fn) for _ in range(args.reps)]
            res[f"B{B}_{name}"] = {"median_ms": round(statistics.median(xs), 4), "min_ms": round(min(xs), 4),
                                   "max_ms": round(max(xs), 4)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
