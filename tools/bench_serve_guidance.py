"""Per-request guidance in serve.LLM on one GPU: GPT-L c2i 256 px (256 tokens, top-k 2000, random-init weights, output head
N(0, 0.02)), max_num_seqs 64, 192 requests (seeded labels) whose cfg_scale cycles through 2.0, 4.0, 7.5.

    python tools/bench_serve_guidance.py [--reps 3] [--out guidance.json]

(a) mixed: one LLM (cfg_scale 4.0) serves all 192 requests, each with its own SamplingParams(cfg_scale=...).
(b) per-scale: what a caller without per-request scales does, one LLM per scale (cfg_scale 2.0, 4.0, 7.5), each serving its 64
    requests, back to back.
(c) uniform: the LLM of (a) with every request at 4.0.
(d) sample kernel at B = 64, V = 16384 (top-k 2000, bf16 rounding, CFG, identical inputs): lg_sample_rows against
    lg_sample_rows_guided with every row at the scalar config's scale and interval, CUDA events over 200 launches per sample.
Wall times end in a device synchronise. (a), (b) and (c) report seconds for all 192 requests, images / s and ms per serve step
(wall / steps_run). Every number is a median [min, max] over --reps repetitions, the variants alternated in one process."""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_serve import card, model, stats, wall  # noqa: E402

SCALES = (2.0, 4.0, 7.5)
S, SLOTS, N, TOPK = 256, 64, 192, 2000


def serve_all(m, labels, groups):
    """groups: [(LLM cfg_scale, [(request index, per-request cfg_scale or None)])], served one LLM after another. Returns (seconds,
    serve steps)."""
    from llamagen_b200.serve import LLM, SamplingParams
    steps = 0

    def run():
        nonlocal steps
        for base, reqs in groups:
            llm = LLM(m, cfg_scale=base, max_num_seqs=SLOTS, seed=0)
            for i, c in reqs:
                llm.add_request([labels[i]], SamplingParams(temperature=1.0, top_k=TOPK, max_tokens=S, cfg_scale=c))
            while llm.has_unfinished_requests():
                llm.step()
            steps += llm.steps_run
    t = wall(run)
    return t, steps


def sample_kernel(reps, iters=200):
    """(d): us per launch of lg_sample_rows and lg_sample_rows_guided on the same [2B, V] logits."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, V = 64, 16384
    g = torch.Generator().manual_seed(0)
    x = (3.0 * torch.randn(2 * B, V, generator=g)).cuda()
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 5, dtype=torch.int32, device="cuda")
    cfg = torch.full((B,), 4.0, dtype=torch.float32, device="cuda")
    interval = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    sc = _lib.SampleCfg(4.0, -1, 1.0, TOPK, 1.0, 0, 0)
    out = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(2)]
    stream = _lib.current_stream("cuda")

    def plain():
        lib.lg_sample_rows(_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), _lib.ptr(out[0]),
                           None, 0, stream)

    def guided():
        lib.lg_sample_rows_guided(_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                  _lib.ptr(cfg), _lib.ptr(interval), _lib.ptr(out[1]), None, 0, stream)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        return 1e3 * e0.elapsed_time(e1) / iters

    for fn in (plain, guided):
        timed(fn)                                                    # warm-up
    res = {"plain": [], "guided": []}
    for _ in range(reps):
        res["plain"].append(timed(plain))
        res["guided"].append(timed(guided))
    torch.cuda.synchronize()
    assert torch.equal(out[0], out[1]), "lg_sample_rows_guided drew other tokens than lg_sample_rows on the same inputs"
    return {k: stats(v, "us") for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workload": f"GPT-L c2i 256px, {N} requests, max_num_seqs {SLOTS}, top-k {TOPK}, scales {list(SCALES)}"}
    print(res["card"], flush=True)
    m = model("GPT-L", block_size=256, vocab_size=16384)
    labels = torch.randint(0, 1000, (N,), generator=torch.Generator().manual_seed(1)).tolist()
    scale_of = [SCALES[i % len(SCALES)] for i in range(N)]
    variants = {
        "a_mixed": [(4.0, [(i, scale_of[i]) for i in range(N)])],
        "b_per_scale": [(s, [(i, None) for i in range(N) if scale_of[i] == s]) for s in SCALES],
        "c_uniform": [(4.0, [(i, 4.0) for i in range(N)])],
    }
    serve_all(m, labels, [(4.0, [(i, scale_of[i]) for i in range(8)])])   # warm-up: every variant runs this LLM shape and path
    secs = {k: [] for k in variants}
    nsteps = {}
    for _ in range(a.reps):
        for k, g in variants.items():
            t, n = serve_all(m, labels, g)
            secs[k].append(t)
            nsteps[k] = n
    for k in variants:
        res[k] = {"s": stats(secs[k], "s"), "img_per_s": stats([N / t for t in secs[k]], "img_per_s"),
                  "ms_per_step": stats([1e3 * t / nsteps[k] for t in secs[k]]), "steps": nsteps[k]}
        print(json.dumps({k: res[k]}), flush=True)
    res["d_sample_kernel_B64_V16384"] = sample_kernel(max(a.reps, 5))
    print(json.dumps({"d_sample_kernel_B64_V16384": res["d_sample_kernel_B64_V16384"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
