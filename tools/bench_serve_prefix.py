"""Image-completion serving timing on one GPU: serve.LLM requests that bring their first P image tokens, for GPT-L c2i 256 px (256
tokens, cfg 4.0, top-k 2000, 16 slots, P in {64, 128, 192}) and GPT-XL t2i 512 px (1024 tokens, cfg 7.5, top-k 1000, 8 slots, P in
{256, 512}).

    python tools/bench_serve_prefix.py [--reps 5] [--out serve_prefix.json]

(a) join: one lg_prefill_slot_prefix + its token-P draw into slot 0 of a full running set, against the P eager serve steps
    (lg_decode_rows / lg_decode_rows_t2i + lg_sample_rows over every slot) a request that decoded its prefix would run.
(b) throughput with a full queue: 2 x max_num_seqs completion requests, P cycling through the workload's values, all queued, against
    generate(prefix=...) in static batches. A static batch needs one P, so the requests are grouped by P and each group runs in
    batches of at most max_num_seqs.
Every number is a median [min, max] over --reps repetitions, the variants of a row alternated in one process. Random-init weights
(output head N(0, 0.02)); synthetic captions of 8 to 120 valid tokens and prefixes, seeded."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_serve import Workload, card, model, stats, wall  # noqa: E402


class PrefixWorkload(Workload):
    """Workload whose request i completes prefixes[i] (P cycling through Ps)."""

    def __init__(self, name, m, S, cfg, topk, n, seed, Ps):
        super().__init__(name, m, S, cfg, topk, n, seed)
        g = torch.Generator().manual_seed(seed + 1)
        self.Ps = Ps
        self.prefixes = [torch.randint(0, m.vocab_size, (Ps[i % len(Ps)],), generator=g) for i in range(n)]

    def add(self, llm, i):
        if self.t2i:
            return llm.add_request(prompt_embeds=self.prompts[i], sampling_params=self.sp, prefix=self.prefixes[i])
        return llm.add_request([self.prompts[i]], self.sp, prefix=self.prefixes[i])

    def static_prefix(self, idx):
        from llamagen_b200 import generate
        i = torch.tensor(idx, device="cuda")
        pf = torch.stack([self.prefixes[j] for j in idx])
        return generate(self.m, self.cond[i], self.S, emb_masks=None if self.mask is None else self.mask[i], cfg_scale=self.cfg,
                        temperature=1.0, top_k=self.sp.top_k, seed=1, prefix=pf)


def join_cost(w, slots, reps, n_steps=32, n_joins=8):
    """(a): slot 0's request is abandoned to the timed joins; the other slots keep decoding between them."""
    plain = Workload(w.name, w.m, w.S, w.cfg, w.sp.top_k, slots, 7)
    llm = plain.llm(slots)
    for i in range(slots):
        plain.add(llm, i)
    llm.step()
    st, params = llm._state, llm._params
    cls = plain.prompts[0] if not w.t2i else None

    def serve_steps():
        for _ in range(n_steps):
            llm.step()

    def joins(P):
        st["out"][0, :P] = w.prefixes[w.Ps.index(P)].to("cuda", torch.int32)
        for _ in range(n_joins):
            if cls is not None:
                st["tok"][0] = cls                            # c2i: the join reads the class id from the slot's input
            llm._device_join_prefix(st, params, 0, P)

    serve_steps()
    for P in w.Ps:
        joins(P)                                              # warm-up (and the scratch of the longest prefix)
    step, join = [], {P: [] for P in w.Ps}
    for _ in range(reps):
        step.append(1e3 * wall(serve_steps) / n_steps)
        for P in w.Ps:
            join[P].append(1e3 * wall(lambda: joins(P)) / n_joins)
    step_med = stats(step)["median_ms"]
    rows = {f"P={P}": dict(join=stats(join[P]), decode_steps_replaced_ms=round(P * step_med, 2),
                           join_over_steps=round(stats(join[P])["median_ms"] / (P * step_med), 4)) for P in w.Ps}
    return {"serve_step": stats(step), **rows}


def throughput(w, slots, reps):
    """(b): 2 x slots completion requests, all queued; images per second."""
    n = 2 * slots
    groups = {P: [i for i in range(n) if w.Ps[i % len(w.Ps)] == P] for P in w.Ps}
    batches = [g[b0:b0 + slots] for g in groups.values() for b0 in range(0, len(g), slots)]

    def serve():
        llm = w.llm(slots)
        for i in range(n):
            w.add(llm, i)
        while llm.has_unfinished_requests():
            llm.step()

    def static():
        for b in batches:
            w.static_prefix(b)
    serve(), static()                                         # warm-up
    s, t = [], []
    for _ in range(reps):
        s.append(n / wall(serve))
        t.append(n / wall(static))
    return {"requests": n, "static_batches": [dict(P=w.Ps[b[0] % len(w.Ps)], images=len(b)) for b in batches],
            "serve": stats(s, "img_per_s"), "static": stats(t, "img_per_s")}


def run(w, slots, reps):
    row = {"workload": w.name, "max_num_seqs": slots, "P": w.Ps}
    row["join"] = join_cost(w, slots, reps)
    print(json.dumps(row), flush=True)
    row["throughput"] = throughput(w, slots, reps)
    print(json.dumps(row["throughput"]), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "rows": []}
    print(res["card"], flush=True)

    def save():
        if a.out:
            os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
            json.dump(res, open(a.out, "w"), indent=1)

    gl = model("GPT-L", block_size=256, vocab_size=16384)
    res["rows"].append(run(PrefixWorkload("GPT-L c2i 256px", gl, 256, 4.0, 2000, 32, 16, [64, 128, 192]), 16, a.reps))
    save()
    del gl
    torch.cuda.empty_cache()
    xl = model("GPT-XL", block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    res["rows"].append(run(PrefixWorkload("GPT-XL t2i 512px", xl, 1024, 7.5, 1000, 16, 8, [256, 512]), 8, a.reps))
    save()


if __name__ == "__main__":
    main()
