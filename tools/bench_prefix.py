"""Image completion timing on one GPU: generate(prefix=...) against the teacher-forced workaround, the prefill pass against P decode
steps, the fp8-cache prefill attention (kernel 2 against attention_kernel) and a t2i completion.

    python tools/bench_prefix.py [--reps 5] [--out prefix.json]

Every number is a median [min, max] over --reps repetitions of CUDA-event timings, the variants of a row alternated. Random-init
weights (output head N(0, 0.02)); what is timed does not depend on the weights' values."""
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
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def stats(xs):
    return {"median_ms": round(statistics.median(xs), 3), "min_ms": round(min(xs), 3), "max_ms": round(max(xs), 3), "n": len(xs)}


def alternate(reps, **fns):
    out = {k: [] for k in fns}
    for k, f in fns.items():
        f()                                  # warm-up: module loads, graph capture, scratch allocation
    for _ in range(reps):
        for k, f in fns.items():
            out[k].append(timed(f)[0])
    return {k: stats(v) for k, v in out.items()}


def model(name, dt, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(0)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dt).eval()


def c2i_rows(reps):
    from llamagen_b200 import generate
    from llamagen_b200 import _lib
    m = model("GPT-L", torch.bfloat16, block_size=256, vocab_size=16384)
    rows = []
    for B in (1, 64):
        cond = torch.randint(0, 1000, (B,), device="cuda")
        ref = generate(m, cond, 256, cfg_scale=4.0, sample_logits=False)
        for P in (64, 128, 192):
            pf = ref[:, :P].contiguous()
            teacher = ref.clone()
            r = alternate(reps,
                          prefix=lambda: generate(m, cond, 256, cfg_scale=4.0, sample_logits=False, prefix=pf),
                          teacher=lambda: generate(m, cond, 256, cfg_scale=4.0, sample_logits=False, teacher=teacher),
                          prefill_only=lambda: generate(m, cond, P + 1, cfg_scale=4.0, sample_logits=False, prefix=pf),
                          decode_only=lambda: generate(m, cond, 256, cfg_scale=4.0, sample_logits=False))
            # greedy: the prefix run reproduces the plain run's tokens after P up to each image's first disagreement, which must
            # sit where the teacher-forced run's top-2 gap is a near tie (both runs fed the same tokens up to there)
            a = generate(m, cond, 256, cfg_scale=4.0, sample_logits=False, prefix=pf)
            _, lb = generate(m, cond, 256, cfg_scale=4.0, sample_logits=False, teacher=teacher, return_logits=True)
            top = torch.topk(lb, 2, -1).values
            agree = 0
            for i in range(B):
                d = (a[i, P:] != ref[i, P:]).nonzero()
                k = P + int(d[0]) if len(d) else 256
                agree += k - P
                if k < 256:
                    gap = float(top[k, i, 0] - top[k, i, 1])
                    assert gap <= 0.25, f"B={B} P={P} image {i}: token {k} differs at a top-2 gap of {gap:.3f}"
            agree /= B * (256 - P)
            step_ms = r["decode_only"]["median_ms"] / 255
            rows.append({"B": B, "P": P, **r, "decode_step_ms": round(step_ms, 4), "P_decode_steps_ms": round(P * step_ms, 2),
                         "agreement_after_P": round(agree, 4)})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def attention_fp8(reps):
    """One layer's prefill attention of GPT-L c2i at B = 64 under CFG, P = 192 (Tq = 193) on an fp8 cache: kernel 2 against
    attention_kernel (LG_ATTN_TMA=0), through lg_test_attention with graphs off."""
    from llamagen_b200 import _lib
    lib = _lib.load()
    R, Tq, H, hd, S = 128, 193, 16, 64, 264
    kb = torch.randint(0, 0x70, (1, R, H, S, hd), dtype=torch.uint8, device="cuda")
    vb = torch.randint(0, 0x70, (1, R, H, S, hd), dtype=torch.uint8, device="cuda")
    q = (0.1 * torch.randn(R * Tq, H * hd, device="cuda")).to(torch.bfloat16)
    out = torch.empty_like(q)
    path = (ctypes.c_int * 3)()

    def call():
        _lib.check(lib.lg_test_attention(1, 3, 1.0, 1.0, R, Tq, H, hd, hd, S, _lib.ptr(kb), _lib.ptr(vb), 1, 0, 0, None, None, None, 1, 0,
                                         _lib.ptr(q), None, 2, None, 0, None, _lib.ptr(out), path, _lib.current_stream("cuda")))

    def many(env):
        def f():
            if env:
                os.environ["LG_ATTN_TMA"] = "0"
            else:
                os.environ.pop("LG_ATTN_TMA", None)
            for _ in range(20):
                call()
        return f
    r = alternate(reps, kernel2=many(False), attention_kernel=many(True))
    os.environ.pop("LG_ATTN_TMA", None)
    res = {k: {kk: (vv / 20 if kk.endswith("_ms") else vv) for kk, vv in v.items()} for k, v in r.items()}
    res["shape"] = dict(R=R, Tq=Tq, H=H, hd=hd)
    print(json.dumps(res), flush=True)
    return res


def t2i_row(reps):
    from llamagen_b200 import generate
    m = model("GPT-XL", torch.bfloat16, block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    B, P = 8, 512
    cond = (0.5 * torch.randn(B, 120, 2048, device="cuda")).to(torch.bfloat16)
    em = torch.ones(B, 120, device="cuda")
    ref = generate(m, cond, 1024, em, cfg_scale=7.5, sample_logits=False)
    pf, teacher = ref[:, :P].contiguous(), ref.clone()
    r = alternate(reps, prefix=lambda: generate(m, cond, 1024, em, cfg_scale=7.5, sample_logits=False, prefix=pf),
                  teacher=lambda: generate(m, cond, 1024, em, cfg_scale=7.5, sample_logits=False, teacher=teacher))
    r.update(B=B, P=P)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    print(res["card"], flush=True)
    res["c2i"] = c2i_rows(a.reps)
    res["attention_fp8_p192"] = attention_fp8(a.reps)
    res["t2i"] = t2i_row(a.reps)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
