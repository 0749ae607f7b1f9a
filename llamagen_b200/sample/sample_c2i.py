"""`python -m llamagen_b200.sample.sample_c2i` — same flags and output file as
autoregressive/sample/sample_c2i.py:101-123 (sample_{gpt_type}.png), executed by the sm_90a engine."""
import argparse
import time

import torch

from .. import generate
from .common import add_common_args, load_gpt, load_vq


def main(args):
    torch.manual_seed(args.seed)
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("llamagen_b200 has no CPU path: a CUDA (sm_90a) device is required")
    device = "cuda"
    vq_model = load_vq(args, device)
    latent_size = args.image_size // args.downsample_size
    gpt_model = load_gpt(args, device, latent_size)

    class_labels = args.class_labels or [207, 360, 387, 974, 88, 979, 417, 279]      # sample_c2i.py:77
    c_indices = torch.tensor(class_labels, device=device)
    qzshape = [len(class_labels), args.codebook_embed_dim, latent_size, latent_size]

    torch.cuda.synchronize()
    t1 = time.time()
    index_sample = generate(gpt_model, c_indices, latent_size ** 2, cfg_scale=args.cfg_scale, cfg_interval=args.cfg_interval,
                            temperature=args.temperature, top_k=args.top_k, top_p=args.top_p, sample_logits=True)
    torch.cuda.synchronize()
    print(f"gpt sampling takes about {time.time() - t1:.2f} seconds.")
    t2 = time.time()
    samples = vq_model.decode_code(index_sample, qzshape)     # output value is between [-1, 1] for trained weights
    torch.cuda.synchronize()
    print(f"decoder takes about {time.time() - t2:.2f} seconds.")
    from torchvision.utils import save_image
    save_image(samples, "sample_{}.png".format(args.gpt_type), nrow=4, normalize=True, value_range=(-1, 1))
    print(f"image is saved to sample_{args.gpt_type}.png")


def build_parser():
    parser = add_common_args(argparse.ArgumentParser(), t2i=False)
    parser.add_argument("--cfg-interval", type=float, default=-1)
    parser.add_argument("--class-labels", type=int, nargs="+", default=None,
                        help="extension: override the 8 hard-coded ImageNet labels (batch size = number of labels)")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
