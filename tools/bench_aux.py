"""Measurements for the widened rows of SURVEY §8(f): VQ encode (f-2) and pixel finishing (f-1), one JSON line.

  python tools/bench_aux.py [--batch 64] [--size 256] [--iters 10]

Timed with CUDA events on the launching stream after warm-up; inputs (fp32 images, 50-200 MB per call) exceed nothing
special, so an L2 flush (a 256 MB memset) runs between timed iterations. Peaks come from MEASURED_PEAKS.json."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def encoder_flops(m, size):
    """2*MACs of Encoder.forward + quant_conv for one image (vq_model.py:64-124), from the parameter shapes."""
    sd = m.state_dict()
    n = len(m.config.encoder_ch_mult)
    fl, res = 0, size

    def conv(name, r):
        w = sd[name + ".weight"]
        return 2 * w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3] * r * r

    def resblock(p, r):
        f = conv(p + ".conv1", r) + conv(p + ".conv2", r)
        return f + (conv(p + ".nin_shortcut", r) if p + ".nin_shortcut.weight" in sd else 0)

    def attn(p, r):
        c = sd[p + ".q.weight"].shape[0]
        return 4 * conv(p + ".q", r) + 2 * 2 * (r * r) * (r * r) * c

    fl += conv("encoder.conv_in", res)
    for i in range(n):
        for j in range(2):
            fl += resblock(f"encoder.conv_blocks.{i}.res.{j}", res)
            if i == n - 1:
                fl += attn(f"encoder.conv_blocks.{i}.attn.{j}", res)
        if i != n - 1:
            res //= 2
            fl += conv(f"encoder.conv_blocks.{i}.downsample.conv", res)
    fl += resblock("encoder.mid.0", res) + attn("encoder.mid.1", res) + resblock("encoder.mid.2", res)
    fl += conv("encoder.conv_out", res) + conv("quant_conv", res)
    return fl


def timed(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        total += a.elapsed_time(b)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from llamagen_b200 import VQ_models
    from llamagen_b200.postprocess import to_uint8_nhwc
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    # fallback: H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense bf16 at 700 W), not rates measured here
    hbm = float(peaks.get("hbm_gbs", peaks.get("hbm_GBps", 3350.0))) if isinstance(peaks, dict) else 3350.0
    tf = float(peaks.get("bf16_tflops_sustained", 989.0)) if isinstance(peaks, dict) else 989.0
    torch.manual_seed(0)
    m = VQ_models["VQ-16"](codebook_size=16384, codebook_embed_dim=8).cuda().eval()
    B, S = args.batch, args.size
    x = torch.rand(B, 3, S, S, device="cuda") * 2 - 1
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ms_enc = timed(lambda: m.encode(x), args.iters, flush)
    fl = encoder_flops(m, S) * B
    pix = torch.randn(B, 3, S, S, device="cuda")
    out = torch.empty(B, S, S, 3, dtype=torch.uint8, device="cuda")
    ms_pix = timed(lambda: to_uint8_nhwc(pix, out=out), args.iters, flush)
    pix_bytes = pix.numel() * 4 + out.numel()
    big = torch.randn(B, 3, 384, 384, device="cuda")
    ms_res = timed(lambda: to_uint8_nhwc(big, size=256, out=out), args.iters, flush)
    res_bytes = big.numel() * 4 + out.numel()
    idx = torch.randint(0, 16384, (B, (S // 16) ** 2), device="cuda")
    ms_dec = timed(lambda: m.decode_code(idx, [B, 8, S // 16, S // 16]), args.iters, flush)
    print(json.dumps({
        "tool": "bench_aux", "batch": B, "image_size": S, "l2": "256 MB memset between timed iterations",
        "encode": {"ms": ms_enc, "images_per_s": B / ms_enc * 1e3, "tflops": fl / ms_enc / 1e9, "peak_tflops": tf,
                   "frac_tensor": fl / ms_enc / 1e9 / tf, "gflop_per_image": fl / B / 1e9},
        "decode": {"ms": ms_dec, "images_per_s": B / ms_dec * 1e3},
        "pixels_to_u8": {"ms": ms_pix, "gbs": pix_bytes / ms_pix / 1e6, "peak_gbs": hbm, "frac_hbm": pix_bytes / ms_pix / 1e6 / hbm,
                         "bytes": pix_bytes},
        "pixels_to_u8_bicubic_384_to_256": {"ms": ms_res, "gbs": res_bytes / ms_res / 1e6, "frac_hbm": res_bytes / ms_res / 1e6 / hbm,
                                            "bytes": res_bytes},
    }))


if __name__ == "__main__":
    main()
