"""fp8 (e4m3) vs model-dtype ("auto") KV cache on bench.py's workload, both measured alternately in one process.

Workload (as bench.py): GPT-L c2i 256 px (256 tokens), cfg 4.0, top-k 2000, batch 64; one step = generate() + VQ-16 decode_code().
One set of seeded GPT-L weights in bf16, loaded into two models: one keeps the default cache, one calls set_kv_cache("fp8"). After
a warm-up the two take turns, each step timed with a host clock around work that ends in a device synchronise. Also reports:
  - batch-1 generate() latency per token for both;
  - the attention-class device time per step (one prefill + S - 1 decode steps of one generate() per model, lg_profile_read with
    programmatic dependent launch off, so kernel times are additive; the profiler bypasses CUDA graphs and multi-chain decode, so
    this is a per-kernel-class figure, not a step time). With the fused QKV epilogue the cache write is inside the attention class;
    qkv_rope_kvwrite is the unfused epilogue;
  - the algorithmic K/V and weight bytes of a mean decode step, computed from the shapes.
Prints one JSON line with the GPU name, power limit and max SM clock.

    python tools/bench_kv_fp8.py [--steps 4] [--warmup 1] [--batch 64] [--out results/bench_kv_fp8.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_fp16 import gpu_info  # noqa: E402


def step_bytes(c, R, S, kv_bytes):
    """Mean decode step of an S-token generate() with R rows: weights streamed once, K/V of the valid prefix read once."""
    D, F, L, V, H = c.dim, c.ffn_dim, c.n_layer, c.vocab_size, c.n_head
    hd = D // H
    hdp = 112 if hd == 100 else hd
    weights = ((4 * D * D + 3 * D * F) * L + V * D) * 2
    mean_keys = sum(c.cls_token_num + t for t in range(1, S)) / (S - 1)      # decode steps see cls_token_num + 1 .. + S - 1 keys
    kv = 2 * L * R * H * mean_keys * hdp * kv_bytes
    return weights, kv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4, help="timed steps per cache dtype (>= 3)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--b1-tokens", type=int, default=256, help="tokens of the batch-1 latency run")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.steps >= 3

    import torch
    from llamagen_b200 import GPT_models, VQ_models, _lib, generate
    assert torch.cuda.is_available(), "bench_kv_fp8.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    g, S, B = 16, 256, args.batch
    torch.manual_seed(0)
    base = GPT_models["GPT-L"](block_size=S, vocab_size=16384)
    base.output.weight.data.normal_(std=0.02)
    models = {}
    for name in ("auto", "fp8"):
        m = GPT_models["GPT-L"](block_size=S, vocab_size=16384)
        m.load_state_dict(base.state_dict())
        m = m.to(device=dev, dtype=torch.bfloat16).eval()
        m.set_kv_cache(name)
        models[name] = m
    cfg = base.config
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
    lib = _lib.load()
    with torch.no_grad():
        for i in range(args.warmup):
            for m in models.values():
                step(m, 100 + i)
        for i in range(args.steps):
            for name, m in models.items():
                t0 = time.perf_counter()
                step(m, i)
                times[name].append(time.perf_counter() - t0)
        # batch-1 latency (the column-owner GEMV path and the deep-ring fused attention), per token
        lat = {k: [] for k in models}
        one = labels[:1]
        n = args.b1_tokens
        for m in models.values():
            generate(m, one, n, seed=0, **kw)
            torch.cuda.synchronize()
        for i in range(3):
            for name, m in models.items():
                t0 = time.perf_counter()
                generate(m, one, n, seed=i, **kw)
                torch.cuda.synchronize()
                lat[name].append((time.perf_counter() - t0) / n * 1e6)
        # attention-class device time, PDL off (additive kernel times)
        names = {}
        i = 0
        while lib.lg_profile_class_name(i) is not None:
            names[lib.lg_profile_class_name(i).decode()] = i
            i += 1
        prof = {}
        _lib.check(lib.lg_set_pdl(0), "lg_set_pdl")
        for name, m in models.items():
            generate(m, labels, S, seed=7, **kw)
            torch.cuda.synchronize()
            _lib.check(lib.lg_profile_reset(), "lg_profile_reset")
            _lib.check(lib.lg_profile_enable(1), "lg_profile_enable")
            generate(m, labels, S, seed=7, **kw)
            torch.cuda.synchronize()
            _lib.check(lib.lg_profile_enable(0), "lg_profile_enable")
            for cls in ("attention", "qkv_rope_kvwrite"):
                ms, cnt = ctypes.c_double(), ctypes.c_uint64()
                _lib.check(lib.lg_profile_read(names[cls], ctypes.byref(ms), ctypes.byref(cnt)), "lg_profile_read")
                # one launch per layer per forward (the condition prefill and S - 1 decode steps)
                steps = cnt.value / cfg.n_layer
                prof[f"{name}_{cls}_us_per_step"] = round(ms.value * 1e3 / steps, 2) if cnt.value else 0.0
                prof[f"{name}_{cls}_ms_per_generate"] = round(ms.value, 3)
                prof[f"{name}_{cls}_launches"] = cnt.value
        _lib.check(lib.lg_set_pdl(1), "lg_set_pdl")

    res = dict(gpu_info())
    res["workload"] = f"GPT-L c2i 256 px bf16, cfg 4.0, top-k 2000, batch {B}, generate() + VQ-16 decode per step"
    R = 2 * B
    for name, kvb in (("auto", 2), ("fp8", 1)):
        res[f"{name}_ms_per_step"] = [round(t * 1e3, 2) for t in times[name]]
        res[f"{name}_median_ms"] = round(statistics.median(times[name]) * 1e3, 2)
        res[f"{name}_batch1_us_per_token"] = round(statistics.median(lat[name]), 1)
        wb, kv = step_bytes(cfg, R, S, kvb)
        res[f"{name}_mean_decode_step_weight_GB"] = round(wb / 1e9, 3)
        res[f"{name}_mean_decode_step_kv_GB"] = round(kv / 1e9, 3)
    res.update(prof)
    res["fp8_over_auto_step"] = round(res["fp8_median_ms"] / res["auto_median_ms"], 4)
    res["fp8_over_auto_batch1"] = round(res["fp8_batch1_us_per_token"] / res["auto_batch1_us_per_token"], 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
