"""Speculative Jacobi decoding cost: ms per verify pass of generate(..., sjd_window=L) against generate()'s ms per token at the same
batch, the break-even tokens per pass (pass time / step time), the tokens per pass observed, and the attention time per pass on the
window kernel against attention_kernel (LG_ATTN_TMA=0, event-timed through the engine's per-class profiler, graphs off).

Random weights: the acceptance they show says nothing about trained LlamaGen; the break-even figure is what carries over.

    python tools/bench_sjd.py [--quick]
"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from llamagen_b200 import GPT_models, _lib, generate  # noqa: E402

PC_ATTENTION = 2


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps * 1e3, out


def attention_ms(fn):
    lib = _lib.load()
    lib.lg_profile_reset()
    lib.lg_profile_enable(1)
    fn()
    ms, n = ctypes.c_double(), ctypes.c_uint64()
    lib.lg_profile_read(PC_ATTENTION, ctypes.byref(ms), ctypes.byref(n))
    lib.lg_profile_enable(0)
    return ms.value


def model(name, t2i, image_size):
    kw = dict(block_size=(image_size // 16) ** 2, vocab_size=16384)
    if t2i:
        kw.update(model_type="t2i", cls_token_num=120, caption_dim=2048)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=torch.bfloat16).eval()


def run(m, B, Ls, cfg, top_k, t2i, reps):
    S = m.block_size
    if t2i:
        cond = torch.randn(B, 120, 2048, device="cuda", dtype=torch.bfloat16)
        em = torch.ones(B, 120, device="cuda")
    else:
        cond, em = torch.randint(0, 1000, (B,), device="cuda"), None
    kw = dict(emb_masks=em, cfg_scale=cfg, top_k=top_k, seed=0)
    t_gen, _ = timed(lambda: generate(m, cond, S, **kw), reps)
    step = t_gen / S
    rows = []
    for L in Ls:
        t_sjd, (_, st) = timed(lambda: generate(m, cond, S, sjd_window=L, return_stats=True, **kw), reps)
        it = st["iterations"]
        pass_ms = t_sjd / it
        f = lambda: generate(m, cond, S, sjd_window=L, **kw)
        a_win = attention_ms(f)
        os.environ["LG_ATTN_TMA"] = "0"
        try:
            a_cc = attention_ms(f)
        finally:
            del os.environ["LG_ATTN_TMA"]
        rows.append((B, L, step, pass_ms, pass_ms / step, st["tokens_per_iteration"], t_gen, t_sjd, a_win / it, a_cc / it))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="B = 1 and 8, L = 8 only")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"card: {smi}")
    hdr = ("B", "L", "step ms", "pass ms", "break-even tok/pass", "tok/pass seen", "generate ms", "sjd ms", "attn ms/pass window",
           "attn ms/pass attention_kernel")
    print("| " + " | ".join(hdr) + " |")
    print("|" + "---|" * len(hdr))
    fmt = lambda r: "| " + " | ".join(str(x) if isinstance(x, int) else f"{x:.3f}" for x in r) + " |"
    torch.manual_seed(0)
    m = model("GPT-L", False, 256)
    for B in ((1, 8) if args.quick else (1, 8, 64)):
        for r in run(m, B, (8,) if args.quick else (4, 8, 16, 32), 4.0, 2000, False, 1 if B == 64 else 2):
            print("GPT-L c2i 256 px " + fmt(r), flush=True)
    del m
    torch.cuda.empty_cache()
    m = model("GPT-XL", True, 512)
    for r in run(m, 1, (8,) if args.quick else (8, 16), 7.5, 1000, True, 1):
        print("GPT-XL t2i 512 px " + fmt(r), flush=True)


if __name__ == "__main__":
    main()
