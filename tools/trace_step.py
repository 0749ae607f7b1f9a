"""Kernel timeline of one bench step via torch.profiler (CUPTI): per-kernel totals and the idle gaps between
kernels inside the CUDA-graph replay.  Usage: python tools/trace_step.py [--batch 64] [--out trace.json]"""
import argparse, collections, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile
from llamagen_b200 import GPT_models, VQ_models, generate

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--gpt-model", default="GPT-L")
ap.add_argument("--out", default=None)
ap.add_argument("--no-vq", action="store_true")
args = ap.parse_args()
torch.manual_seed(0)
dev = "cuda"
gpt = GPT_models[args.gpt_model](block_size=256, vocab_size=16384)
gpt.output.weight.data.normal_(std=0.02)
gpt = gpt.to(dev, torch.bfloat16).eval()
vq = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).to(dev).eval()
labels = torch.randint(0, 1000, (args.batch,), device=dev)
kw = dict(cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, sample_logits=True)

def step():
    t = generate(gpt, labels, 256, **kw)
    if not args.no_vq:
        vq.decode_code(t, [args.batch, 8, 16, 16])

for _ in range(2):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
evs.sort(key=lambda e: e.time_range.start)
agg = collections.defaultdict(lambda: [0, 0.0])
for e in evs:
    name = e.name.replace("(anonymous namespace)::", "").replace("void ", "")
    name = name.split("(")[0][:70]
    agg[name][0] += 1
    agg[name][1] += e.time_range.end - e.time_range.start
# critical-path view (meaningful with PDL on, where kernels start early and wait): time between consecutive kernel ENDS
ends = sorted(evs, key=lambda e: e.time_range.end)
cp = collections.defaultdict(lambda: [0, 0.0])
for prev, cur in zip(ends[:-1], ends[1:]):
    nm = cur.name.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0][:70]
    cp[nm][0] += 1
    cp[nm][1] += cur.time_range.end - prev.time_range.end
busy = sum(v[1] for v in agg.values())
span = evs[-1].time_range.end - evs[0].time_range.start
gaps = [max(0, b.time_range.start - a.time_range.end) for a, b in zip(evs[:-1], evs[1:])]
gaps_sorted = sorted(gaps)
res = {"kernels": len(evs), "span_us": span, "busy_us": busy, "idle_us": span - busy,
       "median_gap_us": gaps_sorted[len(gaps) // 2], "p90_gap_us": gaps_sorted[int(len(gaps) * 0.9)],
       "end_to_end_delta": {k: {"n": v[0], "total_us": round(v[1], 1), "avg_us": round(v[1] / v[0], 2)} for k, v in sorted(cp.items(), key=lambda kv: -kv[1][1])},
       "per_kernel": {k: {"n": v[0], "total_us": round(v[1], 1), "avg_us": round(v[1] / v[0], 2), "share_of_span": round(v[1] / span, 4)}
                      for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])}}
print(json.dumps(res, indent=1))
if args.out:
    json.dump(res, open(args.out, "w"), indent=1)
