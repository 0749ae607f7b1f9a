"""fp8 (e4m3) vs 16-bit GEMM weights (`set_weight_dtype`), the variants measured alternately in one process with CUDA events.

Legs (bf16 models with seeded weights; every variant is warmed up before any timing):
  a  batch 1 (R = 2 rows under CFG): GPT-L c2i 256 px, cfg 4.0, generate() of 256 tokens -> us / token; 16-bit vs fp8 weights.
  b  bench.py's workload: GPT-L c2i 256 px, cfg 4.0, top-k 2000, batch 64, one step = generate() + VQ-16 decode_code() -> ms / step and
     images / s for {16-bit, fp8} weights x {16-bit, fp8} KV cache, and for fp8 weights with one and with two decode chains
     (LG_SPLIT=1 / 2; unset, the engine chooses by the bound weight bytes of a layer against the L2 size).
  c  GPT-3B shape (dim 3200, 24 layers, head_dim 100), B = 16 under CFG (R = 32), generate() of 64 tokens -> ms / decode step.
  d  one score() pass (lg_score) of 64 sequences of 256 tokens on GPT-L: compute-bound, the register-A GEMM does extra work there.
For a-c the algorithmic bytes of a mean decode step (weights streamed once, K/V of the valid prefix read once; computed from the
shapes below, not measured) and the rate bytes / measured time are printed, and every timing comes as the median with the min and
max of its repetitions (a difference inside that spread is not resolved): an end-to-end rate of the whole step, not a kernel's
bandwidth. Prints one JSON line with the GPU name, power limit and max SM clock. Fails without a CUDA device; --bytes-only prints the
byte arithmetic alone and times nothing.

    python tools/bench_weight_fp8.py [--steps 5] [--warmup 1] [--legs abcd] [--out results/bench_weight_fp8.json]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def step_bytes(c, R, S, w_fp8, kv_fp8, head_fp8=True):
    """(weight bytes, K/V bytes) of a mean decode step of an S-token generate() with R rows. fp8 weights add their fp32 row scales."""
    D, F, L, V, H = c.dim, c.ffn_dim, c.n_layer, c.vocab_size, c.n_head
    hd = D // H
    hdp = 112 if hd == 100 else hd
    layer = (4 * D * D + 3 * D * F) * (1 if w_fp8 else 2) + ((3 * D + D + 2 * F + D) * 4 if w_fp8 else 0)
    head = V * D * (1 if w_fp8 and head_fp8 else 2) + (V * 4 if w_fp8 and head_fp8 else 0)
    mean_keys = sum(c.cls_token_num + t for t in range(1, S)) / (S - 1)
    return layer * L + head, 2 * L * R * H * mean_keys * hdp * (1 if kv_fp8 else 2)


def shapes():
    from llamagen_b200.gpt import _SHAPES, ModelArgs
    mk = lambda name, S: ModelArgs(n_layer=_SHAPES[name][0], n_head=_SHAPES[name][1], dim=_SHAPES[name][2], block_size=S, vocab_size=16384)
    return {"GPT-L": mk("GPT-L", 256), "GPT-3B": mk("GPT-3B", 256)}


def byte_table():
    cfgs = shapes()
    out = {}
    for leg, name, R, S in (("a", "GPT-L", 2, 256), ("b", "GPT-L", 128, 256), ("c", "GPT-3B", 32, 64)):
        for w8 in (False, True):
            for kv8 in ((False, True) if leg == "b" else (False,)):
                wb, kv = step_bytes(cfgs[name], R, S, w8, kv8)
                out[f"{leg}_{'fp8' if w8 else '16'}w_{'fp8' if kv8 else '16'}kv_step_MB"] = {"weights": round(wb / 1e6, 1), "kv": round(kv / 1e6, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed repetitions per variant")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--legs", default="abcd")
    ap.add_argument("--bytes-only", action="store_true", help="print the algorithmic bytes per decode step and exit (no GPU, no timing)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.steps >= 1 and set(args.legs) <= set("abcd")
    res = {"algorithmic_bytes": byte_table()}
    if args.bytes_only:
        print(json.dumps(res))
        return

    import torch
    from llamagen_b200 import GPT_models, VQ_models, generate, score
    from tools.bench_fp16 import gpu_info
    assert torch.cuda.is_available(), "bench_weight_fp8.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    res.update(gpu_info())
    kw = dict(cfg_scale=4.0, cfg_interval=-1, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True)

    def timed(fn):
        """ms of fn() between two CUDA events on the current stream (fn's work ends on that stream)."""
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def alternate(variants, run):
        """{name: [ms, ...]}: every variant warmed up, then the variants take turns."""
        for _ in range(args.warmup):
            for name, v in variants.items():
                run(name, v, 100)
        torch.cuda.synchronize()
        out = {k: [] for k in variants}
        for i in range(args.steps):
            for name, v in variants.items():
                out[name].append(timed(lambda: run(name, v, i)))
        return out

    def make(name, base_sd, w, kv, S):
        m = GPT_models[name](block_size=S, vocab_size=16384)
        m.load_state_dict(base_sd)
        m = m.to(device=dev, dtype=torch.bfloat16).eval()
        m.set_weight_dtype(w)
        m.set_kv_cache(kv)
        return m

    def with_split(split, fn):
        old = os.environ.pop("LG_SPLIT", None)
        if split is not None:
            os.environ["LG_SPLIT"] = split
        try:
            return fn()
        finally:
            os.environ.pop("LG_SPLIT", None)
            if old is not None:
                os.environ["LG_SPLIT"] = old

    med = statistics.median
    with torch.no_grad():
        if set(args.legs) & set("abd"):
            torch.manual_seed(0)
            base = GPT_models["GPT-L"](block_size=256, vocab_size=16384)
            base.output.weight.data.normal_(std=0.02)
            sd, cfg = base.state_dict(), base.config
            S = 256
        if "a" in args.legs:
            ms = {n: make("GPT-L", sd, n, "auto", S) for n in ("auto", "fp8")}
            one = torch.tensor([207], device=dev)
            t = alternate(ms, lambda n, m, seed: generate(m, one, S, seed=seed, **kw))
            for n in ms:
                us = med(t[n]) / S * 1e3
                wb, kv = step_bytes(cfg, 2, S, n == "fp8", False)
                res[f"a_batch1_{n}_weights_us_per_token"] = round(us, 1)
                res[f"a_batch1_{n}_weights_us_per_token_min_max"] = [round(min(t[n]) / S * 1e3, 1), round(max(t[n]) / S * 1e3, 1)]
                res[f"a_batch1_{n}_weights_algorithmic_GBps"] = round((wb + kv) / (us * 1e-6) / 1e9, 1)
            res["a_fp8_over_auto"] = round(res["a_batch1_fp8_weights_us_per_token"] / res["a_batch1_auto_weights_us_per_token"], 4)
            del ms
        if "b" in args.legs:
            B, g = 64, 16
            vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
            labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(1)).to(dev)
            variants = {f"{w}w_{kv}kv": (make("GPT-L", sd, w, kv, S), None) for w in ("auto", "fp8") for kv in ("auto", "fp8")}
            variants["fp8w_autokv_split1"] = (make("GPT-L", sd, "fp8", "auto", S), "1")
            variants["fp8w_autokv_split2"] = (make("GPT-L", sd, "fp8", "auto", S), "2")

            def step(name, v, seed):
                m, split = v
                with_split(split, lambda: vq.decode_code(generate(m, labels, S, seed=seed, **kw), [B, 8, g, g]))

            t = alternate(variants, step)
            for n in variants:
                w8, kv8 = n.startswith("fp8w"), "_fp8kv" in n
                wb, kv = step_bytes(cfg, 2 * B, S, w8, kv8)
                res[f"b_{n}_ms_per_step"] = [round(x, 1) for x in t[n]]
                res[f"b_{n}_median_ms"] = round(med(t[n]), 1)
                res[f"b_{n}_images_per_s"] = round(B / (med(t[n]) * 1e-3), 1)
                # S - 1 decode steps stream the weights and the cache; generate() + VQ time over them: an end-to-end rate
                res[f"b_{n}_algorithmic_GBps"] = round((wb + kv) * (S - 1) / (med(t[n]) * 1e-3) / 1e9, 1)
            del variants, vq
        if "d" in args.legs:
            ms = {n: make("GPT-L", sd, n, "auto", S) for n in ("auto", "fp8")}
            B = 64
            labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(2)).to(dev)
            toks = torch.randint(0, 16384, (B, S), generator=torch.Generator().manual_seed(3)).to(dev)
            t = alternate(ms, lambda n, m, seed: score(m, labels, toks, cfg_scale=1.0))
            for n in ms:
                res[f"d_score_b64_{n}_weights_ms"] = round(med(t[n]), 2)
                res[f"d_score_b64_{n}_weights_ms_min_max"] = [round(min(t[n]), 2), round(max(t[n]), 2)]
            res["d_fp8_over_auto"] = round(res["d_score_b64_fp8_weights_ms"] / res["d_score_b64_auto_weights_ms"], 4)
            del ms
        if "c" in args.legs:
            torch.manual_seed(1)
            base = GPT_models["GPT-3B"](block_size=256, vocab_size=16384)
            base.output.weight.data.normal_(std=0.02)
            sd3, cfg3 = base.state_dict(), base.config
            del base
            B, S3 = 16, 64
            ms = {n: make("GPT-3B", sd3, n, "auto", 256) for n in ("auto", "fp8")}
            labels = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(4)).to(dev)
            t = alternate(ms, lambda n, m, seed: generate(m, labels, S3, seed=seed, **kw))
            for n in ms:
                per = med(t[n]) / S3
                wb, kv = step_bytes(cfg3, 2 * B, S3, n == "fp8", False)
                res[f"c_gpt3b_r32_{n}_weights_ms_per_step"] = round(per, 3)
                res[f"c_gpt3b_r32_{n}_weights_ms_per_step_min_max"] = [round(min(t[n]) / S3, 3), round(max(t[n]) / S3, 3)]
                res[f"c_gpt3b_r32_{n}_weights_algorithmic_GBps"] = round((wb + kv) / (per * 1e-3) / 1e9, 1)
            res["c_fp8_over_auto"] = round(res["c_gpt3b_r32_fp8_weights_ms_per_step"] / res["c_gpt3b_r32_auto_weights_ms_per_step"], 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
