"""`torchrun --nproc_per_node=N -m llamagen_b200.sample.sample_t2i_ddp` — replica data-parallel text-to-image sampler
with the flags of autoregressive/sample/sample_t2i_ddp.py:199-227: prompts from a tab-separated file with a `Prompt`
column (:115-116), prompt index i*world+rank+total with "a cute dog" past the end (:134-138), per-rank seed
global_seed*world+rank (:34), PNGs under <folder>/images, rank-0 result.jsonl + captions.txt (:174-193).

Differences: weights are broadcast from rank 0 over NCCL once; left-padding is batched on the device (cond.py); the VQ
decode, pixel finishing and PNG encoding of batch i overlap the sampling of batch i+1 (pipeline.py, postprocess.py).
Text features: the HF Flan-T5 encoder (--t5-path), or `--t5-feature-dir` holding one extract_t5_feature.py .npy per
prompt row (`<row>.npy`), or `--synthetic-cond` (seeded random features; no T5 weights exist offline)."""
import argparse
import csv
import json
import math
import os

import torch
import torch.distributed as dist

from .. import distributed as lgd
from ..cond import HFT5Encoder, load_t5_feature_files, prepare_condition, synthetic_features
from ..pipeline import SamplePipeline
from ..postprocess import AsyncPngWriter
from .common import add_common_args, load_gpt, load_vq

FALLBACK_PROMPT = "a cute dog"      # sample_t2i_ddp.py:138


def read_prompts(path):
    with open(path, newline="") as f:
        return [row["Prompt"] for row in csv.DictReader(f, delimiter="\t")]


def prompt_indices(n, rank, world, total):
    return [lgd.image_index(i, rank, world, total) for i in range(n)]


def main(args):
    if not torch.cuda.is_available():
        raise SystemExit("llamagen_b200 has no CPU path: a CUDA (sm_90a) device is required")
    torch.set_grad_enabled(False)
    rank, world, local = lgd.init_from_env("nccl")
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    seed = lgd.rank_seed(args.global_seed, rank, world)
    torch.manual_seed(args.global_seed)            # identical init on every rank before the broadcast
    print(f"Starting rank={rank}, seed={seed}, world_size={world}.")
    latent_size = args.image_size // args.downsample_size
    if rank != 0:
        args_nockpt = argparse.Namespace(**{**vars(args), "gpt_ckpt": None, "vq_ckpt": None})
        vq_model, gpt_model = load_vq(args_nockpt, device), load_gpt(args_nockpt, device, latent_size)
    else:
        vq_model, gpt_model = load_vq(args, device), load_gpt(args, device, latent_size)
    nbytes = lgd.broadcast_module(gpt_model) + lgd.broadcast_module(vq_model)
    if rank == 0:
        print(f"broadcast {nbytes / 1e6:.1f} MB of weights over NCCL")
    torch.manual_seed(seed)
    precision = gpt_model.tok_embeddings.weight.dtype
    T, C = args.t5_feature_max_len, args.t5_feature_dim
    t5 = None
    if not (args.synthetic_cond or args.t5_feature_dir):
        assert os.path.exists(args.t5_path), "--t5-path not found (use --t5-feature-dir or --synthetic-cond without T5 weights)"
        t5 = HFT5Encoder(args.t5_path, args.t5_model_type, T, device, precision)

    prompt_list = read_prompts(args.prompt_csv)
    ckpt_name = os.path.basename(args.gpt_ckpt or "random-init").replace(".pth", "").replace(".pt", "")
    prompt_name = args.prompt_csv.split("/")[-1].split(".")[0].lower()
    folder = (f"{args.gpt_model.replace('/', '-')}-{ckpt_name}-{prompt_name}-size-{args.image_size}-size-{args.image_size}-"
              f"{args.vq_model}-topk-{args.top_k}-topp-{args.top_p}-temperature-{args.temperature}-cfg-{args.cfg_scale}-"
              f"seed-{args.global_seed}")
    sample_folder_dir = f"{args.sample_dir}/{folder}"
    if rank == 0:
        os.makedirs(f"{sample_folder_dir}/images", exist_ok=True)
        print(f"Saving .png samples at {sample_folder_dir}/images")
    if world > 1:
        dist.barrier()

    n = args.per_proc_batch_size
    global_batch = n * world
    num_fid_samples = min(args.num_fid_samples, len(prompt_list))
    total_samples = int(math.ceil(num_fid_samples / global_batch) * global_batch)
    if rank == 0:
        print(f"Total number of images that will be sampled: {total_samples}")
    iterations = total_samples // world // n

    def features(indices):
        if args.synthetic_cond:
            return synthetic_features(n, T, C, seed * 1000003 + indices[0], device, precision)
        if args.t5_feature_dir:
            # rows past the end of the list fall back to row 0's file (the reference substitutes a fixed prompt there)
            paths = [os.path.join(args.t5_feature_dir, f"{i if i < len(prompt_list) else 0}.npy") for i in indices]
            embs, masks = load_t5_feature_files(paths, T, C)
            return embs.to(device, precision), masks.to(device)
        return t5([prompt_list[i] if i < len(prompt_list) else FALLBACK_PROMPT for i in indices])

    pipe = SamplePipeline(gpt_model, vq_model, args.codebook_embed_dim, cfg_scale=args.cfg_scale, temperature=args.temperature,
                          top_k=args.top_k, top_p=args.top_p, sample_logits=True)
    px = args.image_size
    host = [torch.empty(n, px, px, 3, dtype=torch.uint8).pin_memory() for _ in range(2)]

    def flush(job, writer):
        done, buf, indices = job
        done.synchronize()
        for i, index in enumerate(indices):
            writer.submit(buf[i].numpy().copy(), f"{sample_folder_dir}/images/{index:06d}.png")

    total = 0
    with AsyncPngWriter(args.png_workers) as writer:
        pending = None
        for it in range(iterations):
            indices = prompt_indices(n, rank, world, total)
            caption_embs, emb_masks = features(indices)
            c_indices, c_emb_masks = prepare_condition(caption_embs, emb_masks, left_padding=not args.no_left_padding)
            buf = host[it % 2]
            pipe.submit(c_indices, latent_size, to_uint8_host=buf, emb_masks=c_emb_masks)
            done = torch.cuda.Event()
            done.record(pipe.decode_stream)
            if pending is not None:
                flush(pending, writer)
            pending = (done, buf, indices)
            total += global_batch
        if pending is not None:
            flush(pending, writer)

    if world > 1:
        dist.barrier()
    if rank == 0:
        with open(os.path.join(sample_folder_dir, "result.jsonl"), "w") as f:
            for idx, prompt in enumerate(prompt_list):
                f.write(json.dumps({"text": prompt, "image_path": os.path.join(sample_folder_dir, "images", f"{idx:06d}.png")}) + "\n")
        with open(os.path.join(sample_folder_dir, "captions.txt"), "w") as f:
            for prompt in prompt_list:
                f.write(f"{prompt}\n")
        print("Done.")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return sample_folder_dir


def build_parser():
    parser = add_common_args(argparse.ArgumentParser(), t2i=True)
    parser.add_argument("--prompt-csv", type=str, default="evaluations/t2i/PartiPrompts.tsv")
    parser.add_argument("--t5-path", type=str, default="pretrained_models/t5-ckpt")
    parser.add_argument("--t5-model-type", type=str, default="flan-t5-xl")
    parser.add_argument("--t5-feature-max-len", type=int, default=120)
    parser.add_argument("--t5-feature-dim", type=int, default=2048)
    parser.add_argument("--no-left-padding", action="store_true", default=False)
    parser.add_argument("--sample-dir", type=str, default="samples_parti", help="samples_coco or samples_parti")
    parser.add_argument("--per-proc-batch-size", type=int, default=32)
    parser.add_argument("--num-fid-samples", type=int, default=30000)
    parser.add_argument("--global-seed", type=int, default=0)
    parser.add_argument("--t5-feature-dir", type=str, default=None, help="extension: <row>.npy files from extract_t5_feature.py")
    parser.add_argument("--synthetic-cond", action="store_true", help="extension: seeded random T5-shaped features")
    parser.add_argument("--png-workers", type=int, default=8, help="extension: host threads encoding PNGs")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
