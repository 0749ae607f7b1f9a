"""Per-request sampling filters in serve.LLM on one GPU: GPT-L c2i 256 px (256 tokens, random-init weights, output head N(0, 0.02)),
cfg_scale 4.0, max_num_seqs 64, 192 requests (seeded labels) whose (temperature, top_k, top_p) cycle through four settings a demo's
sliders produce: (1.0, 4000, 1.0), (1.0, 1000, 1.0), (0.9, 2000, 0.95), (1.0, 16384, 0.9).

    python tools/bench_serve_sampling.py [--reps 3] [--drain-reps 2] [--out sampling.json]

(a) drain: the default LLM serves the stream; every change of filters waits for the running set to drain.
(b) per-request: LLM(per_request_sampling=True) serves the same stream in one running batch.
(c) uniform: the LLM of (b) with every request at the first setting.
(d) sample kernel at B = 64, V = 16384 (bf16 rounding, CFG, top-k 2000, identical inputs): lg_sample_rows with the scalar config against
    the same call with row arrays holding the same values, CUDA events over 200 launches per sample, alternated.
Wall times end in a device synchronise. (a), (b) and (c) report seconds for all 192 requests, images / s and ms per serve step
(wall / steps_run). Every number is a median [min, max] over the repetitions ((a): --drain-reps, it serves one request at a time)."""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_serve import card, model, stats, wall  # noqa: E402

SETTINGS = ((1.0, 4000, 1.0), (1.0, 1000, 1.0), (0.9, 2000, 0.95), (1.0, 16384, 0.9))
S, SLOTS, N, CFG = 256, 64, 192, 4.0


def serve_all(m, labels, filters, per_request):
    """One LLM serving request i with filters[i]. Returns (seconds, serve steps)."""
    from llamagen_b200.serve import LLM, SamplingParams
    steps = 0

    def run():
        nonlocal steps
        llm = LLM(m, cfg_scale=CFG, max_num_seqs=SLOTS, seed=0, per_request_sampling=per_request)
        for i, (t, k, p) in enumerate(filters):
            llm.add_request([labels[i]], SamplingParams(temperature=t, top_k=k, top_p=p, max_tokens=S))
        while llm.has_unfinished_requests():
            llm.step()
        steps = llm.steps_run
    t = wall(run)
    return t, steps


def sample_kernel(reps, iters=200):
    """(d): us per launch of lg_sample_rows with the scalar config and with row arrays of the same values, on the same logits."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    B, V = 64, 16384
    g = torch.Generator().manual_seed(0)
    x = (3.0 * torch.randn(2 * B, V, generator=g)).cuda()
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 5, dtype=torch.int32, device="cuda")
    scalar = _lib.SampleCfg(CFG, -1, 1.0, 2000, 1.0, 0, 0)
    arr = (torch.full((B,), 1.0, device="cuda"), torch.full((B,), 2000, dtype=torch.int32, device="cuda"), torch.full((B,), 1.0, device="cuda"),
           torch.zeros(B, dtype=torch.int32, device="cuda"))
    rows = _lib.SampleCfg(CFG, -1, 1.0, 2000, 1.0, 0, 0, *(t.data_ptr() for t in arr))
    out = [torch.empty(B, dtype=torch.int32, device="cuda") for _ in range(2)]
    stream = _lib.current_stream("cuda")

    def call(sc, o):
        return lambda: lib.lg_sample_rows(_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                          _lib.ptr(o), None, 0, stream)
    fns = {"scalar": call(scalar, out[0]), "rows": call(rows, out[1])}

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        return 1e3 * e0.elapsed_time(e1) / iters

    for fn in fns.values():
        timed(fn)                                                    # warm-up
    res = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            res[k].append(timed(fn))
    torch.cuda.synchronize()
    assert torch.equal(out[0], out[1]), "the row arrays drew other tokens than the scalar config on the same inputs"
    return {k: stats(v, "us") for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--drain-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workload": f"GPT-L c2i 256px, cfg {CFG}, {N} requests, max_num_seqs {SLOTS}, filters cycling {list(SETTINGS)}"}
    print(res["card"], flush=True)
    m = model("GPT-L", block_size=256, vocab_size=16384)
    labels = torch.randint(0, 1000, (N,), generator=torch.Generator().manual_seed(1)).tolist()
    mixed = [SETTINGS[i % len(SETTINGS)] for i in range(N)]
    variants = {"b_per_request": (mixed, True), "c_uniform": ([SETTINGS[0]] * N, True), "a_drain": (mixed, False)}
    serve_all(m, labels[:8], mixed[:8], True)                     # warm-up: the LLM shape and every filter setting
    secs = {k: [] for k in variants}
    nsteps = {}
    for r in range(max(a.reps, a.drain_reps)):
        for k, (f, per) in variants.items():
            if r >= (a.drain_reps if k == "a_drain" else a.reps):
                continue
            t, n = serve_all(m, labels, f, per)
            secs[k].append(t)
            nsteps[k] = n
    for k in sorted(variants):
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
