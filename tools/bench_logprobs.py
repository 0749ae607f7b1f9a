"""Cost of token log-probabilities on one GPU, three measurements in one command.

    python tools/bench_logprobs.py [--reps 5] [--tokens 256] [--out logprobs.json]

1. The sample kernel alone at B = 64 with CFG (logits [128, 16384], bf16 rounding, top-k 2000): lg_sample_rows_keyed (logprobs off)
   against lg_sample_rows_logprobs with logprob + rank (logprobs=0) and with 20 alternatives too (logprobs=20). CUDA events over 200
   launches each, --reps alternated repetitions, median.
2. generate(): GPT-L c2i 256 px (bf16, random-init weights with an output head N(0, 0.02), 256 tokens), B = 64, cfg 4, top-k 2000, with and
   without return_logprobs, alternated; wall time ending in a device synchronise.
3. serve.LLM on the same model: 64 requests at max_num_seqs 64, every request at logprobs=5 against none, alternated."""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_serve import card, model, stats, wall  # noqa: E402


def sample_kernel_us(reps, B=64, V=16384, launches=200):
    from llamagen_b200 import _lib
    lib, stream = _lib.load(), _lib.current_stream("cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    x = 3.0 * torch.randn(2 * B, V, device="cuda", generator=g)
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    steps = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    out = torch.empty(B, 8, dtype=torch.int32, device="cuda")
    lp = torch.empty(B, 8, device="cuda")
    rank = torch.empty(B, 8, dtype=torch.int32, device="cuda")
    tid = torch.empty(B, 8, 20, dtype=torch.int32, device="cuda")
    tlp = torch.empty(B, 8, 20, device="cuda")
    sc = _lib.SampleCfg(4.0, -1, 1.0, 2000, 1.0, 0, 0)
    head = (_lib.ptr(x), B, V, 1, _lib.LG_DTYPE_BF16, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), None, None, None)
    lp0 = _lib.Logprobs(lp.data_ptr(), rank.data_ptr(), 0, 0, 0)
    lp20 = _lib.Logprobs(lp.data_ptr(), rank.data_ptr(), tid.data_ptr(), tlp.data_ptr(), 20)
    calls = {"off": lambda: lib.lg_sample_rows_keyed(*head, None, _lib.ptr(out), 8, stream),
             "logprobs0": lambda: lib.lg_sample_rows_logprobs(*head, ctypes.byref(lp0), None, _lib.ptr(out), 8, stream),
             "logprobs20": lambda: lib.lg_sample_rows_logprobs(*head, ctypes.byref(lp20), None, _lib.ptr(out), 8, stream)}
    res = {k: [] for k in calls}
    for _ in range(reps):
        for k, call in calls.items():
            for _ in range(20):
                assert call() == 0, _lib.load().lg_last_error()
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps, "tokens": a.tokens}
    print(res["card"], flush=True)
    res["sample_kernel_b64"] = sample_kernel_us(a.reps)
    print(json.dumps({"sample_kernel_b64": res["sample_kernel_b64"]}), flush=True)

    from llamagen_b200 import generate
    from llamagen_b200.serve import LLM, SamplingParams
    m = model("GPT-L", block_size=256, vocab_size=16384, num_classes=1000)
    cond = torch.randint(0, 1000, (64,), generator=torch.Generator().manual_seed(0)).cuda()
    kw = dict(cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, seed=1)
    gen = {"off": lambda: generate(m, cond, a.tokens, **kw), "logprobs": lambda: generate(m, cond, a.tokens, return_logprobs=True, **kw)}
    for f in gen.values():
        f()
    secs = {k: [] for k in gen}
    for _ in range(a.reps):
        for k, f in gen.items():
            secs[k].append(wall(f))
    res["generate_gpt_l_b64"] = {k: stats(v, "s") for k, v in secs.items()}
    print(json.dumps({"generate_gpt_l_b64": res["generate_gpt_l_b64"]}), flush=True)

    def serve_once(lp, S):
        llm = LLM(m, cfg_scale=4.0, max_num_seqs=64, seed=0)
        sp = SamplingParams(temperature=1.0, top_k=2000, max_tokens=S, logprobs=5 if lp else None)

        def run():
            for c in cond.tolist():
                llm.add_request([c], sp)
            while llm.has_unfinished_requests():
                llm.step()
        return wall(run)
    for lp in (False, True):
        serve_once(lp, 16)
    secs = {"off": [], "logprobs5": []}
    for _ in range(a.reps):
        secs["off"].append(serve_once(False, a.tokens))
        secs["logprobs5"].append(serve_once(True, a.tokens))
    res["serve_gpt_l_64"] = {k: stats(v, "s") for k, v in secs.items()}
    print(json.dumps({"serve_gpt_l_64": res["serve_gpt_l_64"]}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
