"""`python -m llamagen_b200.sample.sample_t2i` — flags of autoregressive/sample/sample_t2i.py:130-155.

The Flan-T5 encoder is upstream of the hot path (SURVEY §2 row 7): with `--t5-path` the HF encoder produces the
[B,120,2048] features exactly like language/t5.py; `--cond-npy` takes features precomputed by
language/extract_t5_feature.py (fp32 [1, valid_len, 2048] .npy, one file per prompt); `--synthetic-cond`
draws seeded random features (what the benchmarks use, there are no T5 weights offline).

A negative prompt (`--negative-prompt TEXT`, encoded by the `--t5-path` encoder, or `--negative-cond-npy FILE` in
extract_t5_feature's layout) takes the place of the null condition in classifier-free guidance for every prompt.

Composable guidance (`--compose-prompt TEXT WEIGHT`, `--compose-cond-npy FILE WEIGHT`, repeatable) adds weighted captions to every
image; each image's own caption keeps weight --cfg-scale."""
import argparse
import os
import time

import torch

from .. import generate
from ..cond import HFT5Encoder, load_t5_feature_files, prepare_condition, synthetic_features
from .common import (add_common_args, add_compose_prompt_args, add_inpaint_args, add_prefix_args, add_sjd_arg, check_compose_args,
                     check_inpaint_args, check_prefix_args, compose_caption_cond, compose_caption_features, compose_entries,
                     guidance_kwargs, inpaint_kwargs, load_gpt, load_vq, prefix_kwargs, sjd_kwargs)

PROMPTS = [
    "A portrait photo of a kangaroo wearing an orange hoodie and blue sunglasses standing on the grassin front of the Sydney Opera House holding a sign on the chest that says Welcome Friends!",
    "A blue Porsche 356 parked in front of a yellow brick wall.",
    "A photo of an astronaut riding a horse in the forest. There is a river in front of them with water lilies.",
    "A map of the United States made out of sushi. It is on a table next to a glass of red wine.",
]


def t5_features(args, device, precision):
    T, C = args.t5_feature_max_len, args.t5_feature_dim
    if args.cond_npy:
        embs, masks = load_t5_feature_files(args.cond_npy, T, C)
        return embs.to(device, precision), masks.to(device)
    if args.synthetic_cond:
        return synthetic_features(len(PROMPTS), T, C, args.seed, device, precision)
    return _hf_encoder(args, device, precision)(PROMPTS)


def negative_features(args, device, precision):
    """The negative prompt's (features [1, T, C], mask [1, T]), or None without one."""
    T, C = args.t5_feature_max_len, args.t5_feature_dim
    if args.negative_cond_npy:
        embs, masks = load_t5_feature_files([args.negative_cond_npy], T, C)
        return embs.to(device, precision), masks.to(device)
    if args.negative_prompt:
        return _hf_encoder(args, device, precision)([args.negative_prompt])
    return None


_ENCODERS = {}


def _hf_encoder(args, device, precision):
    """The --t5-path encoder, loaded once for the prompts and the negative prompt."""
    key = (args.t5_path, args.t5_model_type, args.t5_feature_max_len, str(device), precision)
    if key not in _ENCODERS:
        assert os.path.exists(args.t5_path), "--t5-path not found (use --cond-npy or --synthetic-cond without T5 weights)"
        _ENCODERS[key] = HFT5Encoder(args.t5_path, args.t5_model_type, args.t5_feature_max_len, device, precision)
    return _ENCODERS[key]


def check_negative_args(args):
    if args.negative_prompt and args.negative_cond_npy:
        raise SystemExit("pass --negative-prompt or --negative-cond-npy, not both")
    if (args.negative_prompt or args.negative_cond_npy) and not args.cfg_scale > 1.0 and not compose_entries(args):
        raise SystemExit("a negative prompt replaces the unconditional half of classifier-free guidance: it needs --cfg-scale > 1 "
                         "(or --compose-*)")


def main(args):
    torch.manual_seed(args.seed)
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("llamagen_b200 has no CPU path: a CUDA (sm_90a) device is required")
    device = "cuda"
    latent_size = args.image_size // args.downsample_size
    check_prefix_args(args, latent_size)
    check_inpaint_args(args, latent_size)
    check_negative_args(args)
    check_compose_args(args)
    vq_model = load_vq(args, device)
    gpt_model = load_gpt(args, device, latent_size)
    precision = gpt_model.tok_embeddings.weight.dtype
    caption_embs, emb_masks = t5_features(args, device, precision)

    if not args.no_left_padding:            # sample_t2i.py:92-103, batched on the device (cond.left_pad_features)
        print("processing left-padding...")
        for idx, valid in enumerate(emb_masks.sum(dim=-1).tolist()):
            print(f"  prompt {idx} token len: {int(valid)}")
    c_indices, emb_masks = prepare_condition(caption_embs, emb_masks, left_padding=not args.no_left_padding)
    neg = negative_features(args, device, precision)
    nk = {}
    if neg is not None:   # prepared as the prompts are; one negative for every prompt
        nk["negative_cond"], nk["negative_emb_masks"] = prepare_condition(*neg, left_padding=not args.no_left_padding)
    encode = (lambda texts: _hf_encoder(args, device, precision)(texts)) if args.compose_prompt else None
    c_indices, emb_masks = compose_caption_cond(c_indices, emb_masks, compose_caption_features(args, encode, device, precision))
    qzshape = [len(c_indices), args.codebook_embed_dim, latent_size, latent_size]

    pk = {**prefix_kwargs(args, vq_model, len(c_indices), latent_size, device),
          **inpaint_kwargs(args, vq_model, len(c_indices), latent_size, device)}
    torch.cuda.synchronize()
    t1 = time.time()
    index_sample = generate(gpt_model, c_indices, latent_size ** 2, emb_masks, **guidance_kwargs(args, cfg_interval=False),
                            temperature=args.temperature, top_k=args.top_k, top_p=args.top_p, sample_logits=True,
                            **sjd_kwargs(args), **pk, **nk)
    torch.cuda.synchronize()
    print(f"Full sampling takes about {time.time() - t1:.2f} seconds.")
    t2 = time.time()
    samples = vq_model.decode_code(index_sample, qzshape)
    torch.cuda.synchronize()
    print(f"decoder takes about {time.time() - t2:.2f} seconds.")
    from torchvision.utils import save_image
    save_image(samples, "sample_{}.png".format(args.gpt_type), nrow=4, normalize=True, value_range=(-1, 1))
    print(f"image is saved to sample_{args.gpt_type}.png")


def build_parser():
    parser = add_compose_prompt_args(add_inpaint_args(add_prefix_args(add_sjd_arg(add_common_args(argparse.ArgumentParser(), t2i=True)))))
    parser.add_argument("--t5-path", type=str, default="pretrained_models/t5-ckpt")
    parser.add_argument("--t5-model-type", type=str, default="flan-t5-xl")
    parser.add_argument("--t5-feature-max-len", type=int, default=120)
    parser.add_argument("--t5-feature-dim", type=int, default=2048)
    parser.add_argument("--no-left-padding", action="store_true", default=False)
    parser.add_argument("--cond-npy", type=str, nargs="+", default=None, help="extension: precomputed T5 feature files")
    parser.add_argument("--synthetic-cond", action="store_true", help="extension: seeded random T5-shaped features")
    parser.add_argument("--negative-prompt", type=str, default=None,
                        help="extension: a negative prompt for every image, encoded by the --t5-path encoder (needs --cfg-scale > 1)")
    parser.add_argument("--negative-cond-npy", type=str, default=None,
                        help="extension: the negative prompt's T5 features, one .npy in extract_t5_feature's layout")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
