"""Negative prompts: generate() with and without a negative, alternated in one process, and one serve.LLM run of each.

GPT-XL t2i at 512 px (1024 tokens), B = 8, cfg 7.5, bf16 with random weights and synthetic captions (the cost does not depend on
the weights). A negative only changes the rows the unconditional half is built from and the mask it attends with, so the two arms
run the same kernels on the same shapes. Prints one JSON line; --out also writes it to a file.

    python tools/bench_negative.py --rounds 3 --out /tmp/bench_negative.json
"""
import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--image-size", type=int, default=512)
    ap.add_argument("--serve-requests", type=int, default=8)
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_negative needs a CUDA device")
    from llamagen_b200 import GPT_models, generate
    from llamagen_b200.cond import synthetic_features, prepare_condition
    from llamagen_b200.serve import LLM, SamplingParams
    torch.manual_seed(0)
    S = (a.image_size // 16) ** 2
    m = GPT_models["GPT-XL"](block_size=S, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    B = a.batch
    cond, em = prepare_condition(*synthetic_features(B, 120, 2048, 1, "cuda", torch.bfloat16))
    neg, nm = prepare_condition(*synthetic_features(1, 120, 2048, 2, "cuda", torch.bfloat16))
    arms = {"no_negative": dict(), "negative": dict(negative_cond=neg, negative_emb_masks=nm)}

    def run(kw):
        torch.cuda.synchronize()
        t = time.perf_counter()
        generate(m, cond, S, em, cfg_scale=7.5, top_k=1000, seed=3, **kw)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    for kw in arms.values():   # warm-up: module load, graph capture, workspace
        run(kw)
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, kw in arms.items():
            times[k].append(run(kw))
    res = {"gpu": gpu_info(), "model": "GPT-XL t2i", "image_size": a.image_size, "batch": B, "cfg_scale": 7.5, "rounds": a.rounds}
    for k, ts in times.items():
        res[f"generate_{k}_s"] = [round(t, 4) for t in ts]
        res[f"generate_{k}_median_s"] = round(statistics.median(ts), 4)
    res["generate_negative_over_plain"] = round(res["generate_negative_median_s"] / res["generate_no_negative_median_s"], 4)

    # serve.LLM: the same requests with and without a negative each, 8 slots
    rng = torch.Generator().manual_seed(4)
    n = a.serve_requests
    feats = [torch.randn(int(torch.randint(8, 120, (1,), generator=rng)), 2048, generator=rng) for _ in range(n)]
    negf = torch.randn(20, 2048, generator=rng)
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=S)
    for k, negs in (("no_negative", None), ("negative", [negf] * n)):
        llm = LLM(m, cfg_scale=7.5, max_num_seqs=8, seed=1)
        torch.cuda.synchronize()
        t = time.perf_counter()
        llm.generate(prompt_embeds=feats, sampling_params=sp, negative_prompt_embeds=negs)
        torch.cuda.synchronize()
        res[f"serve_{k}_s"] = round(time.perf_counter() - t, 3)
        res[f"serve_{k}_images_per_s"] = round(n / res[f"serve_{k}_s"], 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
