"""Continuous-batching timing on one GPU: serve.LLM against generate() in static batches, for GPT-XL t2i 512 px (1024 tokens, cfg 7.5,
top-k 1000) at max_num_seqs 8 and 16, and GPT-L c2i 256 px (256 tokens, cfg 4.0, top-k 2000) on the class-conditional path.

    python tools/bench_serve.py [--reps 5] [--out serve.json]

(a) step: one serve step (eager lg_decode_rows_t2i / lg_decode_rows + lg_sample_rows over every slot) against one graph-replayed
    decode step of generate() at the same row count ((time of S = 65 tokens - time of S = 33 tokens) / 32).
(b) join: one lg_prefill_slot + its token-0 draw (t2i).
(c) throughput with a full queue: 2 x max_num_seqs requests, serve against generate() in static batches of max_num_seqs.
(d) latency for a seeded Poisson arrival trace of 2 x max_num_seqs requests at 70 % of the lower throughput of (c): mean, p50 and p90
    from arrival to completion; static batching starts a batch when max_num_seqs requests wait or the oldest has waited half a
    batch's time.
Every number is a median [min, max] over --reps repetitions, the variants of a row alternated in one process. Random-init weights
(output head N(0, 0.02)); synthetic captions of 8 to 120 valid tokens, seeded."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def stats(xs, unit="ms"):
    return {f"median_{unit}": round(statistics.median(xs), 4), f"min_{unit}": round(min(xs), 4), f"max_{unit}": round(max(xs), 4),
            "n": len(xs)}


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def model(name, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(0)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=torch.bfloat16).eval()


class Workload:
    """One model and its requests: t2i captions (T5-shaped features) or c2i labels."""

    def __init__(self, name, m, S, cfg, topk, n, seed):
        from llamagen_b200.cond import pack_t5_features, prepare_condition
        from llamagen_b200.serve import SamplingParams
        self.name, self.m, self.S, self.cfg = name, m, S, cfg
        self.sp = SamplingParams(temperature=1.0, top_k=topk, max_tokens=S)
        self.t2i = m.model_type == "t2i"
        g = torch.Generator().manual_seed(seed)
        if self.t2i:
            lens = torch.randint(8, 121, (n,), generator=g).tolist()
            self.prompts = [torch.randn(k, m.config.caption_dim, generator=g) for k in lens]
            c, mk = prepare_condition(*pack_t5_features(self.prompts, m.cls_token_num, m.config.caption_dim), left_padding=True)
            self.cond, self.mask = c.to("cuda", torch.bfloat16), mk.cuda()
        else:
            self.prompts = torch.randint(0, 1000, (n,), generator=g).tolist()
            self.cond, self.mask = torch.tensor(self.prompts, device="cuda"), None

    def llm(self, slots, seed=0):
        from llamagen_b200.serve import LLM
        return LLM(self.m, cfg_scale=self.cfg, max_num_seqs=slots, seed=seed)

    def add(self, llm, i):
        if self.t2i:
            return llm.add_request(prompt_embeds=self.prompts[i], sampling_params=self.sp)
        return llm.add_request([self.prompts[i]], self.sp)

    def static(self, idx, S=None):
        from llamagen_b200 import generate
        i = torch.tensor(idx, device="cuda")
        return generate(self.m, self.cond[i], S or self.S, emb_masks=None if self.mask is None else self.mask[i], cfg_scale=self.cfg,
                        temperature=1.0, top_k=self.sp.top_k, seed=1)


def step_rows(w, slots, reps, n_steps=32):
    """(a) and (b)."""
    llm = w.llm(slots)
    for i in range(slots):
        w.add(llm, i)
    llm.step()                                              # every request joins (c2i: and decodes its first token)

    def serve_steps():
        for _ in range(n_steps):
            llm.step()
    idx = list(range(slots))
    serve, graph = [], []
    serve_steps()
    w.static(idx, n_steps + 1), w.static(idx, 2 * n_steps + 1)           # warm-up
    for _ in range(reps):
        serve.append(1e3 * wall(serve_steps) / n_steps)
        a = wall(lambda: w.static(idx, 2 * n_steps + 1))
        b = wall(lambda: w.static(idx, n_steps + 1))
        graph.append(1e3 * (a - b) / n_steps)
    row = {"serve_step": stats(serve), "generate_graph_step": stats(graph)}
    if w.t2i:                                               # (b): joins into slot 0 (timing only: the slot's request is abandoned)
        st, joins = llm._state, []
        for r in range(reps + 1):
            t = wall(lambda: [llm._device_join_t2i(st, llm._params, 0) for _ in range(16)])
            if r:
                joins.append(1e3 * t / 16)
        row["join"] = stats(joins)
    return row


def throughput(w, slots, reps):
    """(c): 2 x slots requests, all queued; images per second."""
    n = 2 * slots

    def serve():
        llm = w.llm(slots)
        for i in range(n):
            w.add(llm, i)
        while llm.has_unfinished_requests():
            llm.step()

    def static():
        for b0 in range(0, n, slots):
            w.static(list(range(b0, b0 + slots)))
    serve(), static()                                         # warm-up
    s, t = [], []
    for _ in range(reps):
        s.append(n / wall(serve))
        t.append(n / wall(static))
    return {"serve": stats(s, "img_per_s"), "static": stats(t, "img_per_s")}


def latency(w, slots, reps, rate, batch_s, seed):
    """(d): one seeded Poisson trace of 2 x slots arrivals at `rate` requests / s, replayed in real time by both variants."""
    n = 2 * slots
    arrive = np.cumsum(np.random.default_rng(seed).exponential(1.0 / rate, n)).tolist()
    timeout = 0.5 * batch_s

    def serve():
        llm, done, t0, nxt = w.llm(slots), {}, time.perf_counter(), 0
        rid = {}
        while len(done) < n:
            now = time.perf_counter() - t0
            while nxt < n and arrive[nxt] <= now:
                rid[w.add(llm, nxt)] = nxt
                nxt += 1
            if llm.has_unfinished_requests():
                for o in llm.step():
                    done[rid[o.request_id]] = time.perf_counter() - t0     # a finished request's tokens were copied to the host
            else:
                time.sleep(max(0.0, arrive[nxt] - now))
        return [done[i] - arrive[i] for i in range(n)]

    def static():
        done, t0, nxt, queue = {}, time.perf_counter(), 0, []
        while len(done) < n:
            now = time.perf_counter() - t0
            while nxt < n and arrive[nxt] <= now:
                queue.append(nxt)
                nxt += 1
            if queue and (len(queue) >= slots or now - arrive[queue[0]] >= timeout or nxt == n):
                batch, queue = queue[:slots], queue[slots:]
                w.static(batch)
                torch.cuda.synchronize()
                for i in batch:
                    done[i] = time.perf_counter() - t0
            else:
                wake = [arrive[nxt]] if nxt < n else []
                wake += [arrive[queue[0]] + timeout] if queue else []
                time.sleep(max(0.0, min(wake) - now))
        return [done[i] - arrive[i] for i in range(n)]

    out = {"serve": {"mean": [], "p50": [], "p90": []}, "static": {"mean": [], "p50": [], "p90": []}}
    for _ in range(reps):
        for k, f in (("serve", serve), ("static", static)):
            lat = f()
            out[k]["mean"].append(float(np.mean(lat)))
            out[k]["p50"].append(float(np.percentile(lat, 50)))
            out[k]["p90"].append(float(np.percentile(lat, 90)))
    res = {k: {q: stats(v, "s") for q, v in d.items()} for k, d in out.items()}
    res.update(rate_per_s=round(rate, 4), requests=n, static_timeout_s=round(timeout, 3))
    return res


def run(w, slots, reps, seed):
    row = {"workload": w.name, "max_num_seqs": slots}
    row.update(step_rows(w, slots, reps))
    print(json.dumps(row), flush=True)
    row["throughput"] = throughput(w, slots, reps)
    print(json.dumps(row["throughput"]), flush=True)
    if w.t2i:
        tp = min(row["throughput"]["serve"]["median_img_per_s"], row["throughput"]["static"]["median_img_per_s"])
        batch_s = slots / row["throughput"]["static"]["median_img_per_s"]
        row["latency"] = latency(w, slots, reps, 0.7 * tp, batch_s, seed)
        print(json.dumps(row["latency"]), flush=True)
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

    xl = model("GPT-XL", block_size=1024, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    for slots in (8, 16):
        res["rows"].append(run(Workload("GPT-XL t2i 512px", xl, 1024, 7.5, 1000, 2 * slots, slots), slots, a.reps, slots))
        save()
    del xl
    torch.cuda.empty_cache()
    gl = model("GPT-L", block_size=256, vocab_size=16384)
    res["rows"].append(run(Workload("GPT-L c2i 256px", gl, 256, 4.0, 2000, 32, 16), 16, a.reps, 16))
    save()


if __name__ == "__main__":
    main()
