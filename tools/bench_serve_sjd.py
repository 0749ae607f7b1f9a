"""Speculative Jacobi decoding in serve.LLM on one GPU: the same LLM with and without sjd_window, alternated in one process.

    python tools/bench_serve_sjd.py [--workloads c2i,t2i] [--slots 1,4,8,16] [--windows 4,8,16] [--reps 5] [--out sjd.json]

Workloads (bf16, random-init weights with an output head N(0, 0.02), as tools/bench_sjd.py): GPT-L c2i 256 px (256 tokens, cfg 4.0,
top-k 2000) and GPT-XL t2i 512 px (1024 tokens, cfg 7.5, top-k 1000, T5-shaped random captions). For every max_num_seqs, 2 x
max_num_seqs requests are queued at once and served to the end. Reported per (max_num_seqs, L): images / s, ms per serve step (wall /
steps_run), and with SJD ms per pass (= per step) and tokens per pass per request (max_tokens - 1 over the request's passes, mean over
requests). Wall times end in a device synchronise; every number is a median [min, max] over --reps repetitions. Acceptance on random
weights says nothing about trained checkpoints."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_serve import card, model, stats, wall  # noqa: E402

WORKLOADS = {
    "c2i": dict(name="GPT-L", kw=dict(block_size=256, vocab_size=16384), S=256, cfg=4.0, topk=2000),
    "t2i": dict(name="GPT-XL", kw=dict(block_size=1024, vocab_size=16384, model_type="t2i", cls_token_num=120, caption_dim=2048),
                S=1024, cfg=7.5, topk=1000),
}


def serve_once(m, w, slots, L):
    """2 * slots requests queued at once and served to the end. Returns (seconds, steps, mean tokens per pass per request)."""
    from llamagen_b200.serve import LLM, SamplingParams
    n = 2 * slots
    sp = SamplingParams(temperature=1.0, top_k=w["topk"], max_tokens=w["S"])
    rng = np.random.default_rng(1)
    llm = LLM(m, cfg_scale=w["cfg"], max_num_seqs=slots, seed=0, sjd_window=L)
    if m.model_type == "t2i":
        feats = [rng.standard_normal((int(rng.integers(8, 121)), 2048)).astype(np.float32) for _ in range(n)]
        add = [lambda f=f: llm.add_request(prompt_embeds=f, sampling_params=sp) for f in feats]
    else:
        add = [lambda c=int(c): llm.add_request([c], sp) for c in rng.integers(0, 1000, n)]

    def run():
        for a in add:
            a()
        while llm.has_unfinished_requests():
            llm.step()

    t = wall(run)
    tpp = float(np.mean([(w["S"] - 1) / p for p in llm.sjd_request_passes.values()])) if L else 1.0
    return t, llm.steps_run, tpp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="c2i,t2i")
    ap.add_argument("--slots", default="1,4,8,16")
    ap.add_argument("--windows", default="4,8,16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps}
    print(res["card"], flush=True)
    for wk in a.workloads.split(","):
        w = WORKLOADS[wk]
        m = model(w["name"], **w["kw"])
        for slots in [int(s) for s in a.slots.split(",")]:
            variants = [None] + [int(L) for L in a.windows.split(",")]
            for L in variants:
                serve_once(m, dict(w, S=min(w["S"], 24)), slots, L)      # warm-up of this LLM shape and path
            secs = {L: [] for L in variants}
            meta = {}
            for _ in range(a.reps):
                for L in variants:
                    t, steps, tpp = serve_once(m, w, slots, L)
                    secs[L].append(t)
                    meta[L] = (steps, tpp)
            for L in variants:
                n = 2 * slots
                row = {"workload": wk, "max_num_seqs": slots, "sjd_window": L, "steps": meta[L][0],
                       "img_per_s": stats([n / t for t in secs[L]], "img_per_s"),
                       "ms_per_step": stats([1e3 * t / meta[L][0] for t in secs[L]]), "tokens_per_pass": round(meta[L][1], 3)}
                res[f"{wk}_B{slots}_L{L or 0}"] = row
                print(json.dumps(row), flush=True)
        del m
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
