"""Time lg_t5_encode at flan-t5-xl shape (24 layers, d_model 2048, 32 heads, d_ff 5120; random bf16 weights) for B captions of
T = 120 tokens, against the bf16 torch oracle (and transformers' T5EncoderModel when it imports) on the same weights. Prints one
JSON line per B: ms per call (CUDA events over a window of at least --window seconds, after warm-up), TFLOP/s from shape-derived
FLOPs, the card name and its power limit. Then one line for serve.LLM on GPT-XL t2i (random weights, 256 image tokens, cfg 7.5):
the same caption requests sent as prompts= (encoded by the encoder inside the run) and as prompt_embeds= (features encoded before
it), wall time of each run to the last token, and the encoder's share of the prompts= run.
    python tools/bench_t5.py [--batches 1 16 64] [--window 1.0] [--requests 32]"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from llamagen_b200.t5 import T5Config, T5Encoder  # noqa: E402
from oracle.t5_oracle import t5_encoder_oracle  # noqa: E402

CFG = dict(num_layers=24, d_model=2048, d_kv=64, num_heads=32, d_ff=5120, vocab_size=32128)


def flops(B, T, c):
    """Multiply-adds x 2 of the GEMMs and of q.K^T / P.V (norms, softmax and epilogues left out)."""
    D, I, F, L = c["d_model"], c["num_heads"] * c["d_kv"], c["d_ff"], c["num_layers"]
    gemm = 2 * B * T * (3 * I * D + I * D + 2 * F * D + F * D)
    attn = 2 * 2 * B * c["num_heads"] * T * T * c["d_kv"]
    return L * (gemm + attn)


def timed(fn, window_s):
    """ms per call over at least window_s seconds (the count is sized from a probe call), after two warm-up calls."""
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    iters = max(3, int(window_s * 1e3 / max(a.elapsed_time(b), 1e-3)))
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class _Words:
    """Tokenizer stand-in with the HuggingFace call signature: one id per word, eos 1, padded / truncated to max_length."""

    def __call__(self, prompts, max_length, padding, truncation, return_attention_mask, add_special_tokens, return_tensors):
        ids = torch.zeros(len(prompts), max_length, dtype=torch.long)
        for i, p in enumerate(prompts):
            t = ([2 + sum(map(ord, w)) % 32000 for w in p.split()] + [1])[:max_length]
            ids[i, : len(t)] = torch.tensor(t)
        return {"input_ids": ids, "attention_mask": (ids != 0).long()}


def serve_share(enc, n_requests):
    """serve.LLM on GPT-XL t2i 256 px, cfg 7.5: ms of a prompts= run and of a prompt_embeds= run of the same requests."""
    import random
    import time
    from llamagen_b200 import GPT_models
    from llamagen_b200.serve import LLM, SamplingParams
    torch.manual_seed(0)
    gpt = GPT_models["GPT-XL"](block_size=256, vocab_size=16384, cls_token_num=120, model_type="t2i", caption_dim=2048)
    gpt.output.weight.data.normal_(std=0.02)
    gpt = gpt.to("cuda", torch.bfloat16).eval()
    rng = random.Random(0)
    words = "a red blue small large cat dog house tree sea sky night city car old new green bird flower river".split()
    prompts = [" ".join(rng.choice(words) for _ in range(rng.randint(5, 60))) for _ in range(n_requests)]
    sp = SamplingParams(temperature=1.0, top_k=1000, max_tokens=256)

    def run(**kw):
        llm = LLM(gpt, cfg_scale=7.5, max_num_seqs=16, seed=1, text_encoder=enc if "prompts" in kw else None)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = llm.generate(sampling_params=sp, **kw)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, [o.outputs[0].token_ids for o in out]

    run(prompts=prompts[:2])   # warm-up: engines, workspaces, graphs
    ms_p, tok_p = run(prompts=prompts)
    embs, mask = enc(prompts)
    feats = [embs[i][mask[i] != 0] for i in range(len(prompts))]
    ms_e, tok_e = run(prompt_embeds=feats)
    return dict(serve_gpt="GPT-XL t2i 256px cfg 7.5", requests=n_requests, max_num_seqs=16, prompts_ms=round(ms_p, 1),
                prompt_embeds_ms=round(ms_e, 1), encoder_share=round((ms_p - ms_e) / ms_p, 4), same_tokens=tok_p == tok_e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--window", type=float, default=1.0, help="seconds of timed calls per measurement")
    ap.add_argument("--requests", type=int, default=32)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    enc = T5Encoder(T5Config(**CFG), tokenizer=_Words()).to("cuda", torch.bfloat16).eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for k, p in enc.state_dict().items():
            r = torch.randn(p.shape, generator=g, device="cuda")
            p.copy_(1 + 0.1 * r if k.endswith("layer_norm.weight") else (r if p.dim() == 1 or "relative" in k or k == "shared.weight"
                                                                           else r / math.sqrt(p.shape[1])))
    sd = enc.state_dict()
    ocfg = dict(num_layers=24, num_heads=32, d_kv=64, num_buckets=32, max_distance=128, eps=1e-6)
    try:
        import transformers
        hf = transformers.T5EncoderModel(transformers.T5Config(num_layers=24, feed_forward_proj="gated-gelu", dropout_rate=0.0,
                                                               **{k: v for k, v in CFG.items() if k != "num_layers"}))
        hf.load_state_dict(sd, strict=False)
        hf = hf.to("cuda", torch.bfloat16).eval()
    except ImportError:
        hf = None
    T = 120
    for B in args.batches:
        ids = torch.randint(0, CFG["vocab_size"], (B, T), device="cuda")
        mask = torch.ones(B, T, dtype=torch.long, device="cuda")
        ms = timed(lambda: enc.encode(ids, mask), args.window)
        with torch.no_grad():
            ms_oracle = timed(lambda: t5_encoder_oracle(sd, ocfg, ids, mask, torch.bfloat16), args.window)
            ms_hf = timed(lambda: hf(input_ids=ids, attention_mask=mask), args.window) if hf is not None else None
        f = flops(B, T, CFG)
        print(json.dumps(dict(B=B, T=T, engine_ms=round(ms, 3), engine_tflops=round(f / ms / 1e9, 1), oracle_bf16_ms=round(ms_oracle, 3),
                              hf_bf16_ms=None if ms_hf is None else round(ms_hf, 3), gpu=q)))
    del hf
    torch.cuda.empty_cache()
    print(json.dumps(dict(serve_share(enc, args.requests), gpu=q)))


if __name__ == "__main__":
    main()
