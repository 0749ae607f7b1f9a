"""fp16 vs bf16 on bench.py's workload, both dtypes measured alternately in one process.

Workload (as bench.py): GPT-L c2i 256 px (256 tokens), cfg 4.0, top-k 2000, batch 64; one step = generate() + VQ-16 decode_code().
The same seeded weights are cast to bf16 and to fp16; after a warm-up the two models take turns, each step timed with a host clock
around work that ends in a device synchronise. Also reports batch-1 generate() latency per token for both dtypes. Prints one JSON
line with the GPU name and power limit.

    python tools/bench_fp16.py [--steps 4] [--warmup 1] [--batch 64] [--out results/bench_fp16.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the timing is still valid; say why the card description is missing
        import torch
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4, help="timed steps per dtype (>= 3)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--b1-tokens", type=int, default=256, help="tokens of the batch-1 latency run")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.steps >= 3

    import torch
    from llamagen_b200 import GPT_models, VQ_models, generate
    assert torch.cuda.is_available(), "bench_fp16.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    g, S, B = 16, 256, args.batch
    torch.manual_seed(0)
    base = GPT_models["GPT-L"](block_size=S, vocab_size=16384)
    base.output.weight.data.normal_(std=0.02)
    models = {}
    for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
        m = GPT_models["GPT-L"](block_size=S, vocab_size=16384)
        m.load_state_dict(base.state_dict())
        models[name] = m.to(device=dev, dtype=dt).eval()
    del base
    vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
    kw = dict(cfg_scale=4.0, cfg_interval=-1, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True)
    labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(1)).to(dev)

    def step(m, seed):
        toks = generate(m, labels, S, seed=seed, **kw)
        img = vq.decode_code(toks, [B, 8, g, g])
        torch.cuda.synchronize()
        return img

    times = {k: [] for k in models}
    with torch.no_grad():
        for i in range(args.warmup):
            for m in models.values():
                step(m, 100 + i)
        for i in range(args.steps):
            for name, m in models.items():
                t0 = time.perf_counter()
                step(m, i)
                times[name].append(time.perf_counter() - t0)
        # batch-1 latency (the column-owner GEMV path): generate() of one image incl. prefill and sampling, per token
        lat = {k: [] for k in models}
        one = labels[:1]
        n = args.b1_tokens
        for name, m in models.items():
            generate(m, one, n, seed=0, **kw)
            torch.cuda.synchronize()
        for i in range(3):
            for name, m in models.items():
                t0 = time.perf_counter()
                generate(m, one, n, seed=i, **kw)
                torch.cuda.synchronize()
                lat[name].append((time.perf_counter() - t0) / n * 1e6)

    res = dict(gpu_info())
    res["workload"] = f"GPT-L c2i 256 px, cfg 4.0, top-k 2000, batch {B}, generate() + VQ-16 decode per step"
    for name in models:
        res[f"{name}_ms_per_step"] = [round(t * 1e3, 2) for t in times[name]]
        res[f"{name}_median_ms"] = round(statistics.median(times[name]) * 1e3, 2)
        res[f"{name}_batch1_us_per_token"] = round(statistics.median(lat[name]), 1)
    res["fp16_over_bf16_step"] = round(res["fp16_median_ms"] / res["bf16_median_ms"], 4)
    res["fp16_over_bf16_batch1"] = round(res["fp16_batch1_us_per_token"] / res["bf16_batch1_us_per_token"], 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
