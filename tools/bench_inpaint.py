"""Inpainting timing on one GPU: generate(given=, given_mask=) against plain generate() and generate(prefix=).

    python tools/bench_inpaint.py [--reps 3] [--out inpaint.json]

Cases: GPT-L c2i 256 px (B = 64, cfg 4.0, top-k 2000) and GPT-XL t2i 512 px (B = 8, cfg 7.5), random-init weights (output head
N(0, 0.02)); what is timed does not depend on the weights' values. Masks: a centre hole of a quarter of the grid, the right half of
the grid, and an all-False mask (against plain generate()). Every time is a median [min, max] over --reps repetitions of CUDA-event
timings of whole calls, the calls of a case alternated.

Per mask the plan's decode steps and window passes are counted (lg_test_given_plan). One decode step's time is derived from two plain
runs, (t(S) - t(S / 2)) / (S / 2); one window pass's from the mask's run against generate(prefix=) with the mask's leading run P
(plain generate() when P = 0), which runs the same prefill: (t(mask) - t(prefix P) + (S - P - 1 - decode steps) * t(step)) / window
passes. Both are differences of medians, so they carry the spread of the end-to-end times."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def stats(xs):
    return {"median_ms": round(statistics.median(xs), 2), "min_ms": round(min(xs), 2), "max_ms": round(max(xs), 2), "n": len(xs)}


def alternate(reps, fns):
    out = {k: [] for k in fns}
    for f in fns.values():
        f()                                  # warm-up: module loads, graph capture, scratch allocation
    for _ in range(reps):
        for k, f in fns.items():
            out[k].append(timed(f))
    return {k: stats(v) for k, v in out.items()}


def plan(given):
    from llamagen_b200 import _lib
    lib = _lib.load()
    g = given.to(torch.int32).contiguous()
    B, S = g.shape
    buf = (ctypes.c_int32 * (3 * S + 3))()
    n = lib.lg_test_given_plan(_lib.ptr(g), B, S, buf, S + 1)
    assert n > 0, lib.lg_last_error().decode()
    segs = [tuple(buf[3 * i:3 * i + 3]) for i in range(n)]
    return {"lead": segs[0][2], "decode_steps": sum(s[2] for s in segs if s[0] == 1),
            "window_passes": sum(1 for s in segs if s[0] == 2), "window_rows": sum(s[2] + 1 for s in segs if s[0] == 2)}


def masks(grid):
    hole = torch.ones(grid, grid, dtype=torch.bool)
    q = grid // 4
    hole[q:grid - q, q:grid - q] = False                 # the centre quarter of the grid
    right = torch.ones(grid, grid, dtype=torch.bool)
    right[:, grid // 2:] = False                         # the right half is redrawn
    return {"centre_hole": hole.reshape(-1), "right_half": right.reshape(-1), "all_false": torch.zeros(grid * grid, dtype=torch.bool)}


def model(name, dt, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(0)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dt).eval()


def case(label, m, cond, em, S, grid, reps, **kw):
    from llamagen_b200 import generate
    B = cond.shape[0]
    ref = generate(m, cond, S, em, seed=1, **kw)
    fns = {"plain": lambda: generate(m, cond, S, em, seed=1, **kw),
           "plain_half": lambda: generate(m, cond, S // 2, em, seed=1, **kw)}
    info = {}
    for name, mk in masks(grid).items():
        g = torch.where(mk, ref.cpu(), torch.full_like(ref.cpu(), -1))
        info[name] = plan(g)
        fns[name] = (lambda mk=mk: generate(m, cond, S, em, seed=1, given=ref, given_mask=mk, **kw))
        P = info[name]["lead"]
        if P > 0:
            fns[f"prefix_{P}"] = (lambda P=P: generate(m, cond, S, em, seed=1, prefix=ref[:, :P], **kw))
    assert torch.equal(generate(m, cond, S, em, seed=1, given=ref, given_mask=masks(grid)["all_false"], **kw), ref)
    t = alternate(reps, fns)
    step = (t["plain"]["median_ms"] - t["plain_half"]["median_ms"]) / (S // 2)
    rows = {}
    for name in masks(grid):
        p = info[name]
        base = t[f"prefix_{p['lead']}"] if p["lead"] > 0 else t["plain"]
        row = {"call": t[name], "vs_plain": round(t[name]["median_ms"] / t["plain"]["median_ms"], 3), **p}
        if p["window_passes"]:
            win = (t[name]["median_ms"] - base["median_ms"] + (S - p["lead"] - 1 - p["decode_steps"]) * step) / p["window_passes"]
            row.update(window_pass_ms=round(win, 3), decode_step_ms=round(step, 3), window_over_step=round(win / step, 2))
        rows[name] = row
    res = {"case": label, "B": B, "S": S, "decode_step_ms": round(step, 3), "plain": t["plain"], "masks": rows}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    print(res["card"], flush=True)
    m = model("GPT-L", torch.bfloat16, block_size=256, vocab_size=16384)
    cond = torch.randint(0, 1000, (64,), device="cuda")
    res["c2i"] = case("GPT-L c2i 256 px", m, cond, None, 256, 16, a.reps, cfg_scale=4.0, top_k=2000)
    del m
    m = model("GPT-XL", torch.bfloat16, block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    cond = (0.5 * torch.randn(8, 120, 2048, device="cuda")).to(torch.bfloat16)
    em = torch.ones(8, 120, device="cuda")
    res["t2i"] = case("GPT-XL t2i 512 px", m, cond, em, 1024, 32, a.reps, cfg_scale=7.5)
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
