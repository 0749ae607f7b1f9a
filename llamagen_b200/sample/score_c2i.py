"""Score class-conditional token codes with a GPT checkpoint: the validation loss of autoregressive/train/train_c2i.py:194 in one
teacher-forced pass per batch (llamagen_b200.score).

Reads a code directory in the layout autoregressive/train/extract_codes_c2i.py writes: `<name>_codes/{i}.npy` ([1, num_aug,
grid * grid] token ids) and `<name>_labels/{i}.npy` (the class label), and prints one JSON line: the mean NLL per token in nats,
the same in bits, and the number of images. The checkpoint is loaded as sample_c2i loads it.

    python -m llamagen_b200.sample.score_c2i --code-path /path/to/codes --gpt-model GPT-L --gpt-ckpt c2i_L_256.pt --image-size 256
"""
from __future__ import annotations

import argparse
import glob
import json
import math
import os

import numpy as np
import torch

from .. import score
from .common import add_common_args, load_gpt


def code_files(code_path: str):
    """[(codes .npy, labels .npy)] of a code directory, in image-index order. It must hold exactly one `*_codes` and one `*_labels`
    directory, with the same indices."""
    codes = [d for d in glob.glob(os.path.join(code_path, "*_codes")) if os.path.isdir(d)]
    labels = [d for d in glob.glob(os.path.join(code_path, "*_labels")) if os.path.isdir(d)]
    if len(codes) != 1 or len(labels) != 1:
        raise SystemExit(f"{code_path}: expected one *_codes and one *_labels directory, found {len(codes)} and {len(labels)}")
    def indices(d):
        out = {}
        for f in os.listdir(d):
            stem, ext = os.path.splitext(f)
            if ext == ".npy" and stem.isdigit():
                out[int(stem)] = os.path.join(d, f)
        return out
    ci, li = indices(codes[0]), indices(labels[0])
    if set(ci) != set(li):
        raise SystemExit(f"{code_path}: code and label files differ ({len(ci)} vs {len(li)} indices)")
    if not ci:
        raise SystemExit(f"{code_path}: no code files")
    return [(ci[i], li[i]) for i in sorted(ci)]


def load_item(codes_file: str, label_file: str, aug_index: int):
    """(token ids int64 [grid * grid], class label int) of one image: augmentation `aug_index` of its [1, num_aug, grid * grid]
    codes (dataset/imagenet.py CustomDataset reads the same arrays)."""
    codes = np.load(codes_file)
    if codes.ndim != 3 or codes.shape[0] != 1:
        raise SystemExit(f"{codes_file}: expected codes of shape [1, num_aug, grid * grid], got {codes.shape}")
    if not 0 <= aug_index < codes.shape[1]:
        raise SystemExit(f"{codes_file}: --aug-index {aug_index} outside the {codes.shape[1]} augmentations")
    label = np.asarray(np.load(label_file)).reshape(-1)
    return torch.from_numpy(codes[0, aug_index].astype(np.int64)), int(label[0])


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    add_common_args(parser, t2i=False)
    parser.add_argument("--code-path", type=str, required=True, help="directory holding <name>_codes/ and <name>_labels/")
    parser.add_argument("--aug-index", type=int, default=0, help="which augmentation of every image to score (0 = the plain crop)")
    parser.add_argument("--batch-size", type=int, default=64)
    parser.add_argument("--max-images", type=int, default=0, help="score only the first N images (0 = all)")
    parser.set_defaults(cfg_scale=1.0, image_size=256)
    args = parser.parse_args(argv)
    torch.manual_seed(args.seed)
    device = "cuda"
    latent_size = args.image_size // args.downsample_size
    files = code_files(args.code_path)
    if args.max_images > 0:
        files = files[: args.max_images]
    gpt_model = load_gpt(args, device, latent_size)
    total, count = 0.0, 0
    for i in range(0, len(files), args.batch_size):
        items = [load_item(c, l, args.aug_index) for c, l in files[i:i + args.batch_size]]
        tokens = torch.stack([t for t, _ in items]).to(device)
        if tokens.shape[1] != latent_size ** 2:
            raise SystemExit(f"codes hold {tokens.shape[1]} tokens, --image-size / --downsample-size give {latent_size ** 2}")
        labels = torch.tensor([y for _, y in items], device=device)
        nll = score(gpt_model, labels, tokens, cfg_scale=args.cfg_scale)
        total += float(nll.double().sum())
        count += nll.numel()
    mean = total / count
    print(json.dumps({"mean_nll": mean, "bits_per_token": mean / math.log(2), "images": len(files), "tokens": count,
                      "cfg_scale": args.cfg_scale, "gpt_model": args.gpt_model}))


if __name__ == "__main__":
    main()
