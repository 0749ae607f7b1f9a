"""Shared CLI helpers: checkpoint key dispatch (sample_c2i.py:48-58) and model construction."""
from __future__ import annotations

import torch

from .. import GPT_models, VQ_models


def pick_model_weight(checkpoint, from_fsdp: bool):
    if from_fsdp:                       # fsdp: bare state_dict (train_c2i_fsdp.py:321-325)
        return checkpoint
    for key in ("model", "module", "state_dict"):   # ddp / deepspeed / generic
        if key in checkpoint:
            return checkpoint[key]
    raise Exception("please check model weight, maybe add --from-fsdp to run command")   # sample_c2i.py:58


def load_vq(args, device):
    vq_model = VQ_models[args.vq_model](codebook_size=args.codebook_size, codebook_embed_dim=args.codebook_embed_dim)
    vq_model.to(device)
    vq_model.eval()
    if args.vq_ckpt:
        checkpoint = torch.load(args.vq_ckpt, map_location="cpu", weights_only=False)
        vq_model.load_state_dict(checkpoint["model"])
        del checkpoint
    else:
        print("WARNING: no --vq-ckpt given, using random-init tokenizer weights")
    print("image tokenizer is loaded")
    return vq_model


def load_gpt(args, device, latent_size):
    precision = {"none": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}[args.precision]
    kv_cache_dtype = getattr(args, "kv_cache_dtype", "auto")
    if kv_cache_dtype == "fp8" and precision == torch.float32:
        raise SystemExit("--kv-cache-dtype fp8 needs --precision bf16 or fp16 (fp32 models keep an fp32 KV cache)")
    gpt_model = GPT_models[args.gpt_model](
        vocab_size=args.codebook_size, block_size=latent_size ** 2, num_classes=args.num_classes,
        cls_token_num=args.cls_token_num, model_type=args.gpt_type).to(device=device, dtype=precision)
    if args.gpt_ckpt:
        checkpoint = torch.load(args.gpt_ckpt, map_location="cpu", weights_only=False)
        gpt_model.load_state_dict(pick_model_weight(checkpoint, args.from_fsdp), strict=False)
        del checkpoint
    else:
        print("WARNING: no --gpt-ckpt given, using random-init weights with a normal(0.02) output head")
        gpt_model.output.weight.data.normal_(std=0.02)
    gpt_model.eval()
    gpt_model.set_kv_cache(kv_cache_dtype)
    print("gpt model is loaded")
    if args.compile:
        print("--compile is accepted for CLI compatibility; the engine already replays one CUDA graph per decode step")
    return gpt_model


def add_common_args(parser, t2i: bool):
    parser.add_argument("--gpt-model", type=str, choices=list(GPT_models.keys()), default="GPT-XL" if t2i else "GPT-B")
    parser.add_argument("--gpt-ckpt", type=str, default=None)
    parser.add_argument("--gpt-type", type=str, choices=["c2i", "t2i"], default="t2i" if t2i else "c2i",
                        help="class-conditional or text-conditional")
    parser.add_argument("--from-fsdp", action="store_true")
    parser.add_argument("--cls-token-num", type=int, default=120 if t2i else 1, help="max token number of condition input")
    parser.add_argument("--precision", type=str, default="bf16", choices=["none", "fp16", "bf16"])
    parser.add_argument("--kv-cache-dtype", type=str, default="auto", choices=["auto", "fp8"],
                        help="KV-cache storage: the model dtype (auto) or fp8 e4m3 (half the cache bytes; bf16 / fp16 models)")
    parser.add_argument("--compile", action="store_true", default=False)
    parser.add_argument("--vq-model", type=str, choices=list(VQ_models.keys()), default="VQ-16")
    parser.add_argument("--vq-ckpt", type=str, default=None, help="ckpt path for vq model")
    parser.add_argument("--codebook-size", type=int, default=16384, help="codebook size for vector quantization")
    parser.add_argument("--codebook-embed-dim", type=int, default=8, help="codebook dimension for vector quantization")
    parser.add_argument("--image-size", type=int, choices=[256, 384, 512], default=512 if t2i else 384)
    parser.add_argument("--downsample-size", type=int, choices=[8, 16], default=16)
    parser.add_argument("--num-classes", type=int, default=1000)
    parser.add_argument("--cfg-scale", type=float, default=7.5 if t2i else 4.0)
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--top-k", type=int, default=1000 if t2i else 2000, help="top-k value to sample with")
    parser.add_argument("--temperature", type=float, default=1.0, help="temperature value to sample with")
    parser.add_argument("--top-p", type=float, default=1.0, help="top-p value to sample with")
    return parser
