"""Composable guidance: generate() with cond_weights at K = 1, 2, 3 conditions against plain CFG, alternated in one process.

GPT-L c2i at 256 px (256 tokens), B = 32 images, top-k 2000, bf16 with random weights (the cost does not depend on the weights) and
random per-image weights. Arms:
  plain      generate(cond, cfg_scale=4) at B = 32 (64 rows);
  k1, k2, k3 generate(cond [B, K], cond_weights [B, K]) at B = 32 (2 K B rows);
  plain_b64  plain CFG at B = 64: the same 128 rows as k2, so k2 / plain_b64 is the cost of the mix alone.
Per arm: ms per step (the call's wall time over its 256 tokens; the c2i prefill is one position) and images/s, as the median of
--rounds runs with the min / max beside it. Then the sample kernel alone (CUDA events over --kernel-iters launches, median of
--rounds): the grouped mix at K = 1, 2, 3 against lg_sample_rows (plain CFG) on [2 K B, 16384] logits. Prints one JSON line with the
card name and power limit; --out also writes it.

    python tools/bench_compose.py --rounds 5 --out /tmp/bench_compose.json
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def spread(ts):
    return {"median": round(statistics.median(ts), 4), "min": round(min(ts), 4), "max": round(max(ts), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_compose needs a CUDA device")
    from llamagen_b200 import GPT_models, _lib, generate
    torch.manual_seed(0)
    S, B, V = 256, a.batch, 16384
    m = GPT_models["GPT-L"](block_size=S, vocab_size=V, num_classes=1000, cls_token_num=1, model_type="c2i")
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    g = torch.Generator().manual_seed(1)
    labels = torch.randint(0, 1000, (2 * B, 3), generator=g).cuda()
    weights = (4.0 * torch.rand(B, 3, generator=g) - 1.0)
    weights[:, 0] += 3.0
    arms = {"plain": (labels[:B, 0], dict(cfg_scale=4.0)), "plain_b64": (labels[:, 0], dict(cfg_scale=4.0))}
    for K in (1, 2, 3):
        arms[f"k{K}"] = (labels[:B, :K].contiguous(), dict(cond_weights=weights[:, :K].contiguous()))

    def run(cond, kw):
        torch.cuda.synchronize()
        t = time.perf_counter()
        generate(m, cond, S, top_k=2000, seed=3, **kw)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    for cond, kw in arms.values():   # warm-up: module load, graph capture, workspace of every row count
        run(cond, kw)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, (cond, kw) in arms.items():
            times[k].append(run(cond, kw))
    res = {"gpu": gpu_info(), "model": "GPT-L c2i", "image_size": 256, "tokens": S, "batch": B, "top_k": 2000, "rounds": a.rounds}
    for k, ts in times.items():
        n = arms[k][0].shape[0]
        res[f"{k}_ms_per_step"] = spread([1000.0 * t / S for t in ts])
        res[f"{k}_images_per_s"] = spread([n / t for t in ts])
    med = {k: statistics.median(ts) for k, ts in times.items()}
    for K in (1, 2, 3):
        res[f"k{K}_over_plain"] = round(med[f"k{K}"] / med["plain"], 4)
    res["k2_over_plain_b64"] = round(med["k2"] / med["plain_b64"], 4)

    # the sample kernel alone
    lib = _lib.load()
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g, dtype=torch.int64).cuda()
    steps = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    out = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = _lib.SampleCfg(4.0, -1, 1.0, 2000, 1.0, 0, 0)
    x = (3.0 * torch.randn(6 * B, V, generator=g)).cuda()
    wk = torch.full((B, 3), 4.0, device="cuda")

    wks = {K: wk[:, :K].contiguous() for K in (1, 2, 3)}

    def launch(K, st):
        if K == 0:
            return lib.lg_sample_rows(_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                      _lib.ptr(out), None, 0, st)
        return lib.lg_test_sample_groups(_lib.ptr(x), B, K, V, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(wks[K]), _lib.ptr(seeds),
                                         _lib.ptr(steps), _lib.ptr(out), None, st)

    kt = {K: [] for K in (0, 1, 2, 3)}
    graphs = {}
    for K in kt:   # one graph of kernel_iters launches per variant, so host launch cost stays out of the numbers
        _lib.check(launch(K, _lib.current_stream("cuda")), "sample kernel")
        torch.cuda.synchronize()
        graphs[K] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[K]):
            cs = _lib.current_stream("cuda")
            for _ in range(a.kernel_iters):
                _lib.check(launch(K, cs), "sample kernel")
    for _ in range(a.rounds):
        for K in kt:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graphs[K].replay()
            e1.record()
            torch.cuda.synchronize()
            kt[K].append(1000.0 * e0.elapsed_time(e1) / a.kernel_iters)
    names = {0: "sample_rows_cfg", 1: "sample_groups_k1", 2: "sample_groups_k2", 3: "sample_groups_k3"}
    for K, ts in kt.items():
        res[f"{names[K]}_us"] = spread(ts)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
