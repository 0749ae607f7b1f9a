"""Parallel sampling in serve.LLM on one GPU: 16 captions x SamplingParams(n=4) against the same 64 samples sent as 64 requests.

    python tools/bench_serve_n.py [--captions 16] [--n 4] [--tokens 1024] [--reps 3] [--out serve_n.json]

Workload: the bench_serve.py serving shape, GPT-XL t2i 512 px (bf16, random-init weights with an output head N(0, 0.02), 1024 tokens,
cfg 7.5, top-k 1000, T5-shaped random captions), max_num_seqs = captions x n, every request queued at once and served to the end.
Reported for both variants: wall time and ms per serve step (wall / steps_run), median [min, max] over --reps alternated repetitions
(wall times end in a device synchronise), and, from one more run with a device synchronise around every join, the time spent in joins
(prefill, fan-out and the token-0 draws). Then the sample kernel alone at B = 64 with CFG (logits [128, 16384]): lg_sample_rows_guided
against lg_sample_rows_keyed with image indices, CUDA events over 200 launches each, alternated."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_serve import card, model, stats, wall  # noqa: E402


def serve_once(m, feats, n, S, parallel, timed_joins=False):
    """Every caption as one request with n samples (parallel) or as n requests. Returns (seconds, steps, seconds in joins or None)."""
    from llamagen_b200.serve import LLM, SamplingParams
    llm = LLM(m, cfg_scale=7.5, max_num_seqs=len(feats) * n, seed=0)
    joins = [0.0]
    if timed_joins:
        for name in ("_device_join_t2i", "_device_copy_kv", "_device_join_draws"):
            orig = getattr(llm, name)

            def timed(*a, orig=orig):
                torch.cuda.synchronize()
                t = time.perf_counter()
                orig(*a)
                torch.cuda.synchronize()
                joins[0] += time.perf_counter() - t
            setattr(llm, name, timed)

    def run():
        for f in feats:
            if parallel:
                llm.add_request(prompt_embeds=f, sampling_params=SamplingParams(temperature=1.0, top_k=1000, max_tokens=S, n=n))
            else:
                for _ in range(n):
                    llm.add_request(prompt_embeds=f, sampling_params=SamplingParams(temperature=1.0, top_k=1000, max_tokens=S))
        while llm.has_unfinished_requests():
            llm.step()

    t = wall(run)
    return t, llm.steps_run, joins[0] if timed_joins else None


def sample_kernel_us(B=64, V=16384, launches=200, reps=5):
    """Median us per launch of the sample kernel at B images with CFG: lg_sample_rows_guided and lg_sample_rows_keyed (img_rows set)."""
    from llamagen_b200 import _lib
    lib, stream = _lib.load(), _lib.current_stream("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    x = 3.0 * torch.randn(2 * B, V, device="cuda", generator=g)
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    cfg = torch.full((B,), 7.5, device="cuda")
    interval = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    img = (torch.arange(B, dtype=torch.int32, device="cuda") % 4)
    out = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = _lib.SampleCfg(7.5, -1, 1.0, 1000, 1.0, 0, 0)
    head = (_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), _lib.ptr(cfg), _lib.ptr(interval))
    calls = {"guided": lambda: lib.lg_sample_rows_guided(*head, _lib.ptr(out), None, 0, stream),
             "keyed": lambda: lib.lg_sample_rows_keyed(*head, _lib.ptr(img), _lib.ptr(out), None, 0, stream)}
    res = {k: [] for k in calls}
    for _ in range(reps):
        for k, call in calls.items():
            for _ in range(20):
                call()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(launches):
                call()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) * 1000.0 / launches)
    return {k: stats(v, "us") for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--captions", type=int, default=16)
    ap.add_argument("--n", type=int, default=4)
    ap.add_argument("--tokens", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "captions": a.captions, "n": a.n, "tokens": a.tokens, "reps": a.reps}
    print(res["card"], flush=True)
    m = model("GPT-XL", block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    rng = np.random.default_rng(1)
    feats = [rng.standard_normal((int(rng.integers(8, 121)), 2048)).astype(np.float32) for _ in range(a.captions)]
    variants = {"n": True, "requests": False}
    for par in variants.values():                # warm-up of both paths
        serve_once(m, feats, a.n, 16, par)
    secs, steps = {v: [] for v in variants}, {}
    for _ in range(a.reps):
        for v, par in variants.items():
            t, steps[v], _ = serve_once(m, feats, a.n, a.tokens, par)
            secs[v].append(t)
    for v, par in variants.items():
        row = {"variant": v, "samples": a.captions * a.n, "steps": steps[v], "wall": stats(secs[v], "s"),
               "ms_per_step": stats([1000.0 * t / steps[v] for t in secs[v]]),
               "joins_s": round(serve_once(m, feats, a.n, a.tokens, par, timed_joins=True)[2], 4)}
        print(json.dumps(row), flush=True)
        res.setdefault("rows", []).append(row)
    res["sample_kernel_b64"] = sample_kernel_us()
    print(json.dumps({"sample_kernel_b64": res["sample_kernel_b64"]}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
