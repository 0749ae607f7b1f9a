"""Inpainting serving timing on one GPU: serve.LLM requests that bring given tokens and a mask (add_request(given=, given_mask=)),
for GPT-L c2i 256 px (256 tokens, cfg 4.0, top-k 2000, 64 slots) and GPT-XL t2i 512 px (1024 tokens, cfg 7.5, top-k 1000, 8 slots),
with the centre-hole and right-half masks of tools/bench_inpaint.py.

    python tools/bench_serve_inpaint.py [--reps 3] [--out serve_inpaint.json]

(a) throughput with a full queue: 2 x max_num_seqs inpainting requests, all queued, against the same requests as plain serving
    requests and as generate(given=) in static batches of max_num_seqs; images per second. The three are alternated in one process.
(b) one slot extend (lg_extend_slot + its draw, the run length K of the mask's first interior given run) into slot 0 of a full
    running set, against one serve step of that set (eager lg_decode_rows / lg_decode_rows_t2i + the draw over every slot); and how many
    extends a request of the mask runs.
Every number is a median [min, max] over --reps repetitions. Random-init weights (output head N(0, 0.02)); synthetic captions of 8 to
120 valid tokens and given tokens, seeded."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_inpaint import masks  # noqa: E402
from bench_serve import Workload, card, model, stats, wall  # noqa: E402


class InpaintWorkload(Workload):
    """Workload whose requests keep given tokens where `mask` is True (one random image's tokens per request)."""

    def __init__(self, name, m, S, cfg, topk, n, seed, mask):
        super().__init__(name, m, S, cfg, topk, n, seed)
        g = torch.Generator().manual_seed(seed + 2)
        self.given_mask = mask
        self.given = [torch.randint(0, m.vocab_size, (S,), generator=g) for _ in range(n)]

    def add_given(self, llm, i):
        kw = dict(given=self.given[i], given_mask=self.given_mask)
        if self.t2i:
            return llm.add_request(prompt_embeds=self.prompts[i], sampling_params=self.sp, **kw)
        return llm.add_request([self.prompts[i]], self.sp, **kw)

    def static_given(self, idx):
        from llamagen_b200 import generate
        i = torch.tensor(idx, device="cuda")
        return generate(self.m, self.cond[i], self.S, emb_masks=None if self.mask is None else self.mask[i], cfg_scale=self.cfg,
                        temperature=1.0, top_k=self.sp.top_k, seed=1, given=torch.stack([self.given[j] for j in idx]),
                        given_mask=self.given_mask)


def throughput(w, slots, reps):
    n = 2 * slots

    def serve(add):
        llm = w.llm(slots)
        for i in range(n):
            add(llm, i)
        while llm.has_unfinished_requests():
            llm.step()

    def static():
        for b0 in range(0, n, slots):
            w.static_given(list(range(b0, b0 + slots)))
    cases = {"serve_inpaint": lambda: serve(w.add_given), "serve_plain": lambda: serve(w.add), "static_generate_given": static}
    for fn in cases.values():                                 # warm-up
        fn()
    res = {k: [] for k in cases}
    for _ in range(reps):
        for k, fn in cases.items():
            res[k].append(n / wall(fn))
    return {k: stats(v, "img_per_s") for k, v in res.items()}


def extend_cost(w, slots, reps, n_steps=16, n_ext=16):
    from llamagen_b200.serve import _given_plan
    gv = torch.where(w.given_mask, w.given[0], torch.full_like(w.given[0], -1)).to(torch.int32)
    _, extends, _ = _given_plan(gv)
    a, K = next(iter(sorted(extends.items())))
    llm = w.llm(slots)
    for i in range(slots):
        w.add(llm, i)
    llm.step()
    st, params = llm._state, llm._params
    st["out"][0] = w.given[0].to(device="cuda", dtype=torch.int32)   # timing only: slot 0's request is abandoned to the extends

    def steps():
        for _ in range(n_steps):
            llm.step()

    def extends_():
        for _ in range(n_ext):
            llm._device_extend(st, params, 0, a, K)
    steps(), extends_()
    step_ms, ext_ms = [], []
    for _ in range(reps):
        step_ms.append(1e3 * wall(steps) / n_steps)
        ext_ms.append(1e3 * wall(extends_) / n_ext)
    return {"extends_per_request": len(extends), "K_timed": K, "serve_step": stats(step_ms), "slot_extend": stats(ext_ms),
            "extend_over_step": round(sorted(ext_ms)[len(ext_ms) // 2] / sorted(step_ms)[len(step_ms) // 2], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    print(res["card"], flush=True)

    def save():
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            json.dump(res, open(a.out, "w"), indent=1)

    for name, slots, make in [
        ("GPT-L c2i 256px", 64, lambda: (model("GPT-L", block_size=256, vocab_size=16384), 256, 4.0, 2000, 16)),
        ("GPT-XL t2i 512px", 8, lambda: (model("GPT-XL", block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i",
                                               caption_dim=2048), 1024, 7.5, 1000, 32)),
    ]:
        m, S, cfg, topk, grid = make()
        for mname in ("centre_hole", "right_half"):
            w = InpaintWorkload(name, m, S, cfg, topk, 2 * slots, slots, masks(grid)[mname])
            row = {"workload": name, "mask": mname, "max_num_seqs": slots, "given_fraction": round(float(w.given_mask.float().mean()), 4)}
            row["extend"] = extend_cost(w, slots, a.reps)
            print(json.dumps(row), flush=True)
            row["throughput"] = throughput(w, slots, a.reps)
            print(json.dumps(row["throughput"]), flush=True)
            res["rows"].append(row)
            save()
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
