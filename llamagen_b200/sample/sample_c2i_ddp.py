"""`torchrun --nproc_per_node=N -m llamagen_b200.sample.sample_c2i_ddp` — replica data-parallel sampler with the
flags of autoregressive/sample/sample_c2i_ddp.py:161-187: per-rank seed global_seed*world+rank (:47), per-rank
generate() + decode_code(), PNG index i*world+rank+total (:147), rank-0 .npz (:21-35). Differences: weights are
loaded / initialised by rank 0 and broadcast over NCCL once, instead of every rank reading the checkpoint; the pixel
finishing (:141-143) is one CUDA kernel and the PNG encoders run on host threads under the next batch's sampling."""
import argparse
import math
import os

import numpy as np
import torch
import torch.distributed as dist

from .. import distributed as lgd
from ..pipeline import SamplePipeline
from ..postprocess import AsyncPngWriter
from .common import (add_common_args, add_compose_class_arg, add_inpaint_args, check_compose_args, check_inpaint_args, compose_class_cond,
                     guidance_kwargs, inpaint_kwargs, load_gpt, load_vq)


def create_npz_from_sample_folder(sample_dir, num=50_000):
    from PIL import Image
    samples = np.stack([np.asarray(Image.open(f"{sample_dir}/{i:06d}.png")).astype(np.uint8) for i in range(num)])
    assert samples.shape == (num, samples.shape[1], samples.shape[2], 3)
    np.savez(f"{sample_dir}.npz", arr_0=samples)
    print(f"Saved .npz file to {sample_dir}.npz [shape={samples.shape}].")
    return f"{sample_dir}.npz"


def main(args):
    assert torch.cuda.is_available(), "Sampling with DDP requires at least one GPU"
    torch.set_grad_enabled(False)
    rank, world, local = lgd.init_from_env("nccl")
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    seed = lgd.rank_seed(args.global_seed, rank, world)
    torch.manual_seed(args.global_seed)            # identical init on every rank before the broadcast
    print(f"Starting rank={rank}, seed={seed}, world_size={world}.")
    latent_size = args.image_size // args.downsample_size
    check_inpaint_args(args, latent_size)
    check_compose_args(args, args.num_classes)
    if rank != 0:                                   # only rank 0 touches the disk
        args_nockpt = argparse.Namespace(**{**vars(args), "vq_ckpt": None, "gpt_ckpt": None})
        vq_model, gpt_model = load_vq(args_nockpt, device), load_gpt(args_nockpt, device, latent_size)
    else:
        vq_model, gpt_model = load_vq(args, device), load_gpt(args, device, latent_size)
    nbytes = lgd.broadcast_module(gpt_model) + lgd.broadcast_module(vq_model)
    if rank == 0:
        print(f"broadcast {nbytes / 1e6:.1f} MB of weights over NCCL")
    # every rank keeps the same cells of the same image (none without --inpaint-image)
    ik = inpaint_kwargs(args, vq_model, args.per_proc_batch_size, latent_size, device)
    torch.manual_seed(seed)

    # folder name of sample_c2i_ddp.py:100-107 (model, checkpoint name, sizes, sampling knobs); "random-init" when no ckpt is given
    model_name = args.gpt_model.replace("/", "-")
    ckpt = args.gpt_ckpt or "random-init"
    if getattr(args, "from_fsdp", False) and args.gpt_ckpt and len(args.gpt_ckpt.split("/")) > 1:
        ckpt_name = args.gpt_ckpt.split("/")[-2]
    else:
        ckpt_name = os.path.basename(ckpt).replace(".pth", "").replace(".pt", "")
    folder = (f"{model_name}-{ckpt_name}-size-{args.image_size}-size-{args.image_size_eval}-{args.vq_model}-topk-{args.top_k}-topp-{args.top_p}-"
              f"temperature-{args.temperature}-cfg-{args.cfg_scale}-seed-{args.global_seed}")
    sample_folder_dir = f"{args.sample_dir}/{folder}"
    if rank == 0:
        os.makedirs(sample_folder_dir, exist_ok=True)
        print(f"Saving .png samples at {sample_folder_dir}")
    if world > 1:
        dist.barrier()
    n = args.per_proc_batch_size
    global_batch = n * world
    total_samples = int(math.ceil(args.num_fid_samples / global_batch) * global_batch)
    iterations = total_samples // world // n
    total = 0
    # Steady-state loop of sample_c2i_ddp.py:128-149, reorganised (SURVEY §8 f-1): the VQ decode + pixel finishing +
    # D2H of batch i run on a second stream under the AR sampling of batch i+1, and the PNG encoders run on host
    # threads; file names and contents are the reference's.
    pipe = SamplePipeline(gpt_model, vq_model, args.codebook_embed_dim, **guidance_kwargs(args), temperature=args.temperature, top_k=args.top_k, top_p=args.top_p, sample_logits=True, **ik)
    eval_px = args.image_size_eval
    host = [torch.empty(n, eval_px, eval_px, 3, dtype=torch.uint8).pin_memory() for _ in range(2)]

    def flush(job, writer):
        done, buf, base = job
        done.synchronize()
        for i in range(n):
            writer.submit(buf[i].numpy().copy(), f"{sample_folder_dir}/{lgd.image_index(i, rank, world, base):06d}.png")

    with AsyncPngWriter(args.png_workers) as writer:
        pending = None
        for it in range(iterations):
            c_indices = torch.randint(0, args.num_classes, (n,), device=device)
            buf = host[it % 2]
            pipe.submit(compose_class_cond(args, c_indices), latent_size, to_uint8_host=buf)
            done = torch.cuda.Event()
            done.record(pipe.decode_stream)
            if pending is not None:
                flush(pending, writer)
            pending = (done, buf, total)
            total += global_batch
        if pending is not None:
            flush(pending, writer)
    if world > 1:
        dist.barrier()
    if rank == 0:
        create_npz_from_sample_folder(sample_folder_dir, args.num_fid_samples)
        print("Done.")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def build_parser():
    parser = add_compose_class_arg(add_inpaint_args(add_common_args(argparse.ArgumentParser(), t2i=False)))
    parser.add_argument("--cfg-interval", type=float, default=-1)
    parser.add_argument("--image-size-eval", type=int, choices=[256, 384, 512], default=256)
    parser.add_argument("--sample-dir", type=str, default="samples")
    parser.add_argument("--per-proc-batch-size", type=int, default=32)
    parser.add_argument("--num-fid-samples", type=int, default=50000)
    parser.add_argument("--global-seed", type=int, default=0)
    parser.add_argument("--png-workers", type=int, default=8, help="host threads encoding PNGs (extra flag, not in the reference)")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
