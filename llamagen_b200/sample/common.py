"""Shared CLI helpers: checkpoint key dispatch (sample_c2i.py:48-58) and model construction."""
from __future__ import annotations

import os

import numpy as np
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
    weight_dtype = getattr(args, "weight_dtype", "auto")
    if weight_dtype == "fp8" and precision == torch.float32:
        raise SystemExit("--weight-dtype fp8 needs --precision bf16 or fp16 (fp32 models keep fp32 weights)")
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
    gpt_model.set_weight_dtype(weight_dtype)
    print("gpt model is loaded")
    if args.compile:
        print("--compile is accepted for CLI compatibility; the engine already replays one CUDA graph per decode step")
    return gpt_model


def add_sjd_arg(parser):
    parser.add_argument("--sjd-window", type=int, default=None,
                        help="extension: speculative Jacobi decoding with this many tokens per forward pass (2..64)")
    return parser


def sjd_kwargs(args) -> dict:
    """generate() keywords of --sjd-window (none when it is not given, so the default path is unchanged)."""
    return {} if args.sjd_window is None else {"sjd_window": args.sjd_window}


def add_prefix_args(parser):
    parser.add_argument("--prefix-image", type=str, default=None,
                        help="extension: complete this image: it is centre-cropped to --image-size and encoded, the first "
                             "--prefix-rows rows of its latent grid are kept for every image of the batch and the rest is generated")
    parser.add_argument("--prefix-rows", type=int, default=None, help="extension: latent rows of --prefix-image kept (1 .. grid - 1)")
    return parser


def check_prefix_args(args, latent_size: int):
    """Rejects a --prefix-image / --prefix-rows combination that generate() cannot run, before any model is loaded."""
    if args.prefix_image is None and args.prefix_rows is None:
        return
    if args.prefix_image is None or args.prefix_rows is None:
        raise SystemExit("--prefix-image and --prefix-rows go together")
    if not 1 <= args.prefix_rows <= latent_size - 1:
        raise SystemExit(f"--prefix-rows must lie in [1, {latent_size - 1}] (the latent grid has {latent_size} rows)")
    if getattr(args, "sjd_window", None) is not None:
        raise SystemExit("--prefix-image cannot be combined with --sjd-window")
    if not os.path.isfile(args.prefix_image):
        raise SystemExit(f"--prefix-image {args.prefix_image!r} is not a file")


def prefix_kwargs(args, vq_model, batch: int, latent_size: int, device) -> dict:
    """generate() keywords of --prefix-image / --prefix-rows: the first rows * grid codes of the encoded image (raster order), the
    same for every image of the batch; none when no prefix is given, so the default path is unchanged."""
    if args.prefix_image is None:
        return {}
    codes = _encode_image(args.prefix_image, args.image_size, vq_model, device)[: args.prefix_rows * latent_size]
    return {"prefix": codes.view(1, -1).expand(batch, -1).contiguous()}


def _encode_image(path, image_size: int, vq_model, device):
    """The latent codes of the image at `path`, centre-cropped to image_size and encoded, in raster order."""
    from PIL import Image
    from .vq_demo import center_crop
    img = center_crop(Image.open(path).convert("RGB"), image_size)
    x = torch.from_numpy(2.0 * (np.array(img) / 255.0) - 1.0).permute(2, 0, 1)[None].float().to(device)
    _, _, [_, _, indices] = vq_model.encode(x)
    return indices.reshape(-1)


def add_inpaint_args(parser):
    parser.add_argument("--inpaint-image", type=str, default=None,
                        help="extension: redraw one box of this image: it is centre-cropped to --image-size and encoded, every latent "
                             "cell outside --inpaint-box is kept for every image of the batch and the box is generated")
    parser.add_argument("--inpaint-box", type=int, nargs=4, default=None, metavar=("TOP", "LEFT", "BOTTOM", "RIGHT"),
                        help="extension: the latent-grid cells to redraw, rows TOP .. BOTTOM - 1 and columns LEFT .. RIGHT - 1 (a "
                             "redrawn cell sees the cells above and to its left, not the rows below the box)")
    return parser


def check_inpaint_args(args, latent_size: int):
    """Rejects an --inpaint-image / --inpaint-box combination that generate() cannot run, before any model is loaded."""
    if args.inpaint_image is None and args.inpaint_box is None:
        return
    if args.inpaint_image is None or args.inpaint_box is None:
        raise SystemExit("--inpaint-image and --inpaint-box go together")
    top, left, bottom, right = args.inpaint_box
    if not (0 <= top < bottom <= latent_size and 0 <= left < right <= latent_size):
        raise SystemExit(f"--inpaint-box TOP LEFT BOTTOM RIGHT must satisfy 0 <= TOP < BOTTOM <= {latent_size} and "
                         f"0 <= LEFT < RIGHT <= {latent_size} (the latent grid is {latent_size} x {latent_size})")
    if getattr(args, "prefix_image", None) is not None:
        raise SystemExit("--inpaint-image cannot be combined with --prefix-image")
    if getattr(args, "sjd_window", None) is not None:
        raise SystemExit("--inpaint-image cannot be combined with --sjd-window")
    if not os.path.isfile(args.inpaint_image):
        raise SystemExit(f"--inpaint-image {args.inpaint_image!r} is not a file")


def inpaint_mask(box, latent_size: int) -> torch.Tensor:
    """given_mask [grid * grid] of --inpaint-box: True (kept) outside the box, False (redrawn) inside, raster order."""
    top, left, bottom, right = box
    m = torch.ones(latent_size, latent_size, dtype=torch.bool)
    m[top:bottom, left:right] = False
    return m.reshape(-1)


def inpaint_kwargs(args, vq_model, batch: int, latent_size: int, device) -> dict:
    """generate() keywords of --inpaint-image / --inpaint-box: the encoded image's codes, the same for every image of the batch, and the
    mask that keeps every cell outside the box; none when no image is given, so the default path is unchanged."""
    if args.inpaint_image is None:
        return {}
    codes = _encode_image(args.inpaint_image, args.image_size, vq_model, device)
    return {"given": codes.view(1, -1), "given_mask": inpaint_mask(args.inpaint_box, latent_size)}


def add_compose_class_arg(parser):
    parser.add_argument("--compose-class", type=str, nargs=2, action="append", default=None, metavar=("LABEL", "WEIGHT"),
                        help="extension: composable guidance: add this class to every image with this weight (any sign; repeatable, "
                             "up to 7 times); each image's own class keeps weight --cfg-scale")
    return parser


def add_compose_prompt_args(parser):
    parser.add_argument("--compose-prompt", type=str, nargs=2, action="append", default=None, metavar=("TEXT", "WEIGHT"),
                        help="extension: composable guidance: add this caption to every image with this weight (any sign; "
                             "repeatable), encoded by the --t5-path encoder; each image's own caption keeps weight --cfg-scale")
    parser.add_argument("--compose-cond-npy", type=str, nargs=2, action="append", default=None, metavar=("PATH", "WEIGHT"),
                        help="extension: as --compose-prompt, with the caption's T5 features in one .npy (extract_t5_feature's "
                             "layout); these conditions follow the --compose-prompt ones")
    return parser


def compose_entries(args) -> list:
    """The (value, weight string) pairs of --compose-class, or of --compose-prompt then --compose-cond-npy; [] without them."""
    return (list(getattr(args, "compose_class", None) or []) + list(getattr(args, "compose_prompt", None) or [])
            + list(getattr(args, "compose_cond_npy", None) or []))


def check_compose_args(args, num_classes: int = 0):
    """Rejects --compose-* flags that generate() cannot run, before any model is loaded: weights that are not finite numbers, more
    than 7 added conditions, class labels outside [0, num_classes), missing feature files, --sjd-window, and --cfg-interval with
    added conditions."""
    from .. import _lib
    entries = compose_entries(args)
    if not entries:
        return
    if len(entries) > _lib.MAX_COMPOSE - 1:
        raise SystemExit(f"at most {_lib.MAX_COMPOSE - 1} --compose-* conditions (every image has {_lib.MAX_COMPOSE} at most), "
                         f"got {len(entries)}")
    for value, w in entries:
        try:
            wf = float(w)
        except ValueError:
            raise SystemExit(f"--compose-* weight {w!r} is not a number") from None
        if not (np.isfinite(wf) and abs(wf) <= float(np.finfo(np.float32).max)):
            raise SystemExit(f"--compose-* weight {w!r} is not finite")
    for label, _ in getattr(args, "compose_class", None) or []:
        try:
            lab = int(label)
        except ValueError:
            raise SystemExit(f"--compose-class label {label!r} is not an integer") from None
        if not 0 <= lab < num_classes:
            raise SystemExit(f"--compose-class label {lab} must lie in [0, {num_classes})")
    for path, _ in getattr(args, "compose_cond_npy", None) or []:
        if not os.path.isfile(path):
            raise SystemExit(f"--compose-cond-npy {path!r} is not a file")
    if getattr(args, "sjd_window", None) is not None:
        raise SystemExit("--compose-* cannot be combined with --sjd-window")
    if getattr(args, "cfg_interval", -1) != -1:
        raise SystemExit("--cfg-interval applies to plain guidance only; it cannot be combined with --compose-*")


def guidance_kwargs(args, cfg_interval: bool = True) -> dict:
    """generate()'s guidance keywords: cfg_scale (and cfg_interval) as before without --compose-*, else cond_weights: --cfg-scale for
    each image's own condition, then the added conditions' weights in flag order."""
    entries = compose_entries(args)
    if not entries:
        return {"cfg_scale": args.cfg_scale, **({"cfg_interval": args.cfg_interval} if cfg_interval else {})}
    return {"cond_weights": [float(args.cfg_scale)] + [float(w) for _, w in entries]}


def compose_class_cond(args, c_indices):
    """c2i cond of generate(): the labels [B] as they are without --compose-class, else [B, K] with the added classes after each
    image's own."""
    extra = [int(label) for label, _ in getattr(args, "compose_class", None) or []]
    if not extra:
        return c_indices
    add = torch.tensor(extra, dtype=c_indices.dtype, device=c_indices.device).view(1, -1).expand(len(c_indices), -1)
    return torch.cat([c_indices.view(-1, 1), add], 1)


def compose_caption_cond(cond, emb_masks, extra):
    """t2i cond / emb_masks of generate(): as they are without added captions (extra empty), else [B, K, T, C] / [B, K, T] with the
    added prepared captions (each ([1, T, C], [1, T])) after each image's own."""
    if not extra:
        return cond, emb_masks
    B = cond.shape[0]
    c = torch.stack([cond] + [e.to(cond.dtype).expand(B, -1, -1) for e, _ in extra], 1)
    m = torch.stack([emb_masks] + [mk.to(emb_masks.dtype).expand(B, -1) for _, mk in extra], 1)
    return c, m


def compose_caption_features(args, encode, device, precision) -> list:
    """The added captions of --compose-prompt (encoded by `encode`, a list-of-strings -> (features, masks) text encoder, or None when
    the sampler has none) then --compose-cond-npy, each prepared as the prompts are: [(cond [1, T, C], mask [1, T]), ...]."""
    from ..cond import load_t5_feature_files, prepare_condition
    T, C = args.t5_feature_max_len, args.t5_feature_dim
    feats = []
    prompts = [text for text, _ in getattr(args, "compose_prompt", None) or []]
    if prompts:
        if encode is None:
            raise SystemExit("--compose-prompt needs the text encoder (--t5-path); use --compose-cond-npy with precomputed features")
        embs, masks = encode(prompts)
        feats += [(embs[i:i + 1], masks[i:i + 1]) for i in range(len(prompts))]
    for path, _ in getattr(args, "compose_cond_npy", None) or []:
        embs, masks = load_t5_feature_files([path], T, C)
        feats.append((embs.to(device, precision), masks.to(device)))
    return [prepare_condition(e, mk, left_padding=not args.no_left_padding) for e, mk in feats]


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
    parser.add_argument("--weight-dtype", type=str, default="auto", choices=["auto", "fp8"],
                        help="storage of the transformer's GEMM weights: the model dtype (auto) or fp8 e4m3 codes with per-row "
                             "power-of-two scales (half the weight bytes; bf16 / fp16 models)")
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
