"""Composable-guidance requests in serve.LLM on one GPU: GPT-L c2i 256 px (256 tokens, top-k 2000, random-init weights, output head
N(0, 0.02)), max_num_seqs 64, seeded labels.

    python tools/bench_serve_compose.py [--reps 3] [--out compose.json]

(a) composed: one LLM (cfg_scale 4.0) serves 96 requests with SamplingParams(cond_weights=(3.0, 1.5)) and two class ids each (2 slots
    per request).
(b) plain: the same LLM shape serves 192 plain requests (the same 192 slot-requests as (a)).
(c) static: generate(cond_weights=(3.0, 1.5)) on the 96 images of (a), in batches of 32 images (64 + 64 rows, as 64 slots).
(d) sample kernel at 64 slots, V = 16384 (top-k 2000, bf16 rounding): lg_sample_rows_guided against lg_sample_rows_composed with 32
    lead rows (K = 2, scattered rows) and 32 condition rows, CUDA events over 200 launches per sample.
Wall times end in a device synchronise. (a), (b) and (c) report seconds, images / s and, for (a) and (b), ms per serve step (wall /
steps_run). Every number is a median [min, max] over --reps repetitions, the variants alternated in one process."""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_serve import card, model, stats, wall  # noqa: E402

S, SLOTS, N, TOPK, W = 256, 64, 96, 2000, (3.0, 1.5)


def serve(m, labels, composed, n=N):
    """(a) composed (n requests, K = 2) or (b) plain (2n requests). Returns (seconds, serve steps, images)."""
    from llamagen_b200.serve import LLM, SamplingParams
    llm = LLM(m, cfg_scale=4.0, max_num_seqs=SLOTS, seed=0)

    def run():
        if composed:
            for i in range(n):
                llm.add_request([labels[2 * i], labels[2 * i + 1]], SamplingParams(temperature=1.0, top_k=TOPK, max_tokens=S, cond_weights=W))
        else:
            for i in range(2 * n):
                llm.add_request([labels[i]], SamplingParams(temperature=1.0, top_k=TOPK, max_tokens=S))
        while llm.has_unfinished_requests():
            llm.step()
    t = wall(run)
    return t, llm.steps_run, n if composed else 2 * n


def static(m, labels):
    """(c): generate(cond_weights=) over the images of (a), 32 at a time."""
    from llamagen_b200 import generate
    cond = torch.tensor(labels[:2 * N]).view(N, 2)

    def run():
        for b in range(0, N, 32):
            generate(m, cond[b:b + 32].cuda(), S, cond_weights=torch.tensor(W), temperature=1.0, top_k=TOPK, seed=b)
    return wall(run)


def sample_kernel(reps, iters=200):
    """(d): us per launch of lg_sample_rows_guided and lg_sample_rows_composed on the same [2B, V] logits."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, V = SLOTS, 16384
    g = torch.Generator().manual_seed(0)
    x = (3.0 * torch.randn(2 * B, V, generator=g)).cuda()
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 5, dtype=torch.int32, device="cuda")
    cfg = torch.full((B,), 4.0, dtype=torch.float32, device="cuda")
    interval = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    img = torch.zeros(B, dtype=torch.int32, device="cuda")
    rows = torch.full((B, 9), -1, dtype=torch.int32)
    w = torch.zeros(B, 8)
    perm = torch.randperm(B, generator=g).tolist()
    for j in range(B // 2):                      # lead perm[2j] with condition slot perm[2j + 1]
        lead, other = perm[2 * j], perm[2 * j + 1]
        rows[lead, :3] = torch.tensor([B + lead, lead, other])
        rows[other, 0] = -2
        w[lead, :2] = torch.tensor(W)
    rows, w = rows.cuda(), w.cuda()
    sc = _lib.SampleCfg(4.0, -1, 1.0, TOPK, 1.0, 0, 0)
    out = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(2)]
    stream = _lib.current_stream("cuda")

    def plain():
        lib.lg_sample_rows_guided(_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                  _lib.ptr(cfg), _lib.ptr(interval), _lib.ptr(out[0]), None, 0, stream)

    def composed():
        lib.lg_sample_rows_composed(_lib.ptr(x), 2 * B, B, V, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                    _lib.ptr(cfg), _lib.ptr(interval), _lib.ptr(img), None, _lib.ptr(rows), _lib.ptr(w), None,
                                    _lib.ptr(out[1]), None, 0, stream)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        return 1e3 * e0.elapsed_time(e1) / iters

    for fn in (plain, composed):
        timed(fn)                                                    # warm-up
    res = {"plain_guided": [], "composed_K2": []}
    for _ in range(reps):
        res["plain_guided"].append(timed(plain))
        res["composed_K2"].append(timed(composed))
    torch.cuda.synchronize()
    return {k: stats(v, "us") for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workload": f"GPT-L c2i 256px, max_num_seqs {SLOTS}, top-k {TOPK}: {N} composed requests (K = 2, weights "
                                       f"{list(W)}) against {2 * N} plain requests; static generate(cond_weights=) at B = 32"}
    print(res["card"], flush=True)
    m = model("GPT-L", block_size=256, vocab_size=16384)
    labels = torch.randint(0, 1000, (2 * N,), generator=torch.Generator().manual_seed(1)).tolist()
    serve(m, labels, True, 8)                                         # warm-up of both serving paths and the static path
    serve(m, labels, False, 8)
    static(m, labels)
    secs = {"a_composed": [], "b_plain": [], "c_static": []}
    nsteps = {}
    for _ in range(a.reps):
        t, n, _ = serve(m, labels, True)
        secs["a_composed"].append(t)
        nsteps["a_composed"] = n
        t, n, _ = serve(m, labels, False)
        secs["b_plain"].append(t)
        nsteps["b_plain"] = n
        secs["c_static"].append(static(m, labels))
    imgs = {"a_composed": N, "b_plain": 2 * N, "c_static": N}
    for k in secs:
        res[k] = {"s": stats(secs[k], "s"), "img_per_s": stats([imgs[k] / t for t in secs[k]], "img_per_s"), "images": imgs[k]}
        if k in nsteps:
            res[k].update(ms_per_step=stats([1e3 * t / nsteps[k] for t in secs[k]]), steps=nsteps[k])
        print(json.dumps({k: res[k]}), flush=True)
    res["d_sample_kernel_64_slots"] = sample_kernel(max(a.reps, 5))
    print(json.dumps({"d_sample_kernel_64_slots": res["d_sample_kernel_64_slots"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
