"""The reference's language/extract_t5_feature.py on the engine: caption features for --cond-npy / --t5-feature-dir.

    python -m llamagen_b200.sample.extract_t5_feature --data-path DIR --t5-path OUT --data-start 0 --data-end 3 \\
        [--caption-key blip] [--trunc-caption] [--t5-model-path ./pretrained_models/t5-ckpt] [--t5-model-type flan-t5-xl] \\
        [--precision bf16|none] [--batch-size 64]

reads the *.jsonl files of DIR (sorted, [data-start, data-end]) and writes <t5-path>/<jsonl stem>/<line>.npy, fp32
[1, valid_len, d_model]: the same files as the reference. `--prompt-csv FILE` instead writes <t5-path>/<row>.npy per row of
sample_t2i_ddp.read_prompts(FILE), the layout `sample_t2i_ddp --t5-feature-dir` reads. One process; captions are encoded in batches
by t5.T5Encoder (the HuggingFace tokenizer of the checkpoint directory, no caption cleaning, as the reference's call)."""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

CAPTION_KEY = {"blip": 0, "llava": 1, "llava_first": 2}


def read_captions(lst_dir, start, end, caption_key, trunc_caption=False):
    """(caption, jsonl stem, line index) of every line, in the reference's CustomDataset order."""
    out = []
    for name in sorted(os.listdir(lst_dir))[start: end + 1]:
        if not name.endswith(".jsonl"):
            continue
        path = os.path.join(lst_dir, name)
        with open(path) as f:
            for i, line in enumerate(f):
                caption = json.loads(line)["text"][CAPTION_KEY[caption_key]]
                if trunc_caption:
                    caption = caption.split(".")[0]
                out.append((caption, name.split(".")[0], i))
    return out


def write_features(encoder, items, out_dir, batch_size):
    """items: (caption, sub-directory or None, file stem). Writes <out_dir>[/<sub>]/<stem>.npy, fp32 [1, valid_len, d_model]."""
    for s in range(0, len(items), batch_size):
        chunk = items[s: s + batch_size]
        embs, mask = encoder([c for c, _, _ in chunk])
        valid = mask.sum(dim=1).tolist()
        feats = embs.float().cpu()
        for (_, sub, stem), n, f in zip(chunk, valid, feats):
            d = os.path.join(out_dir, sub) if sub else out_dir
            os.makedirs(d, exist_ok=True)
            np.save(os.path.join(d, f"{stem}.npy"), f[None, : int(n)].numpy())


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--data-path", type=str, default=None)
    p.add_argument("--t5-path", type=str, required=True)
    p.add_argument("--data-start", type=int, default=0)
    p.add_argument("--data-end", type=int, default=0)
    p.add_argument("--caption-key", type=str, default="blip", choices=list(CAPTION_KEY))
    p.add_argument("--trunc-caption", action="store_true", default=False)
    p.add_argument("--t5-model-path", type=str, default="./pretrained_models/t5-ckpt")
    p.add_argument("--t5-model-type", type=str, default="flan-t5-xl")
    p.add_argument("--precision", type=str, default="bf16", choices=["none", "bf16"])
    p.add_argument("--max-length", type=int, default=120, help="tokens per caption (T5Embedder's model_max_length)")
    p.add_argument("--batch-size", type=int, default=64)
    p.add_argument("--prompt-csv", type=str, default=None, help="write <row>.npy per prompt of this tab-separated file instead")
    args = p.parse_args(argv)
    if (args.data_path is None) == (args.prompt_csv is None):
        p.error("give exactly one of --data-path and --prompt-csv")
    if not torch.cuda.is_available():
        raise SystemExit("llamagen_b200 has no CPU path: a CUDA (sm_90a) device is required")
    from ..t5 import T5Encoder
    if args.prompt_csv:
        from .sample_t2i_ddp import read_prompts
        items = [(c, None, i) for i, c in enumerate(read_prompts(args.prompt_csv))]
    else:
        items = read_captions(args.data_path, args.data_start, args.data_end, args.caption_key, args.trunc_caption)
    dtype = {"none": torch.float32, "bf16": torch.bfloat16}[args.precision]
    enc = T5Encoder.from_pretrained(os.path.join(args.t5_model_path, args.t5_model_type), dtype=dtype, device="cuda",
                                    max_length=args.max_length)
    os.makedirs(args.t5_path, exist_ok=True)
    print(f"{len(items)} captions")
    with torch.no_grad():
        write_features(enc, items, args.t5_path, args.batch_size)


if __name__ == "__main__":
    main()
