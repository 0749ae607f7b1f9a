"""Two-stage sampling pipeline: AR generation of batch i+1 overlaps the VQ decode of batch i.

The AR decode loop is latency-bound (≈ 220 short dependent kernels per token) and leaves most SMs idle, while the
VQ decode is a dense tensor-core burst; running them on two streams lets the decode fill the idle machine.
This is the steady-state loop of the reference's DDP sampler (sample_c2i_ddp.py:128-149), reorganised:
    for labels in batches: tokens = generate(labels); pixels = decode_code(tokens); emit(pixels)
"""
from __future__ import annotations

import os

import torch

from . import _lib
from .generate import generate
from .postprocess import to_uint8_nhwc


class SamplePipeline:
    def __init__(self, gpt_model, vq_model, codebook_embed_dim: int = 8, **sampling_kwargs):
        self.gpt, self.vq = gpt_model, vq_model
        self.kw = sampling_kwargs
        self.embed_dim = codebook_embed_dim
        dev = gpt_model.tok_embeddings.weight.device
        self.dev = dev
        self.decode_stream = torch.cuda.Stream(device=dev)
        self._last = None
        # While batch i is decoded the AR loop of batch i+1 is running. LG_PIPE_CONV_CTAS = N > 0 runs the decoder's convolutions as
        # N persistent CTAs (a cap on the SMs they occupy); 0 = one CTA per tile (default): the sampler loses more from a long-lived
        # background decode than from a short full-machine burst, so the cap stays off; what does help is the sampler's stream priority.
        self.conv_ctas = int(os.environ.get("LG_PIPE_CONV_CTAS", "0"))

    def submit(self, cond, grid: int, to_uint8_host=None, emb_masks=None):
        """Enqueue generate() on the current stream and decode_code() on the decode stream. Returns the pixel tensor
        (fp32 NCHW; uint8 NHWC when `to_uint8_host` has the decoder's own resolution); it is complete once `self.decode_stream` (or `wait()`) has been synchronised. When
        `to_uint8_host` (a pinned uint8 [B,H',W',3] tensor) is given, the pixel finishing of sample_c2i_ddp.py:141-143
        (bicubic resize to H' x W' when that differs from the decoder's output, clamp, uint8, NHWC — one kernel,
        postprocess.to_uint8_nhwc) and the device-to-host copy are enqueued behind the decode as well."""
        main = torch.cuda.current_stream(self.dev)
        tokens = generate(self.gpt, cond, grid * grid, emb_masks, **self.kw)
        ready = torch.cuda.Event()
        ready.record(main)
        self.decode_stream.wait_event(ready)
        tokens.record_stream(self.decode_stream)
        with torch.cuda.stream(self.decode_stream):
            if self.conv_ctas > 0:
                _lib.load().lg_vq_set_cta_budget(self.conv_ctas)     # read at launch time by every conv of this decode
            shape = [tokens.shape[0], self.embed_dim, grid, grid]
            up = 2 ** (len(self.vq.config.decoder_ch_mult) - 1)
            if to_uint8_host is not None and tuple(to_uint8_host.shape[1:3]) == (grid * up, grid * up):
                # no resize wanted: conv_out's drain writes the uint8 NHWC bytes directly (SURVEY 8 f-1), no fp32 image in HBM
                pixels = self.vq.decode_code_uint8(tokens, shape)
                to_uint8_host.copy_(pixels, non_blocking=True)
            else:
                pixels = self.vq.decode_code(tokens, shape)
                if to_uint8_host is not None:
                    u8 = to_uint8_nhwc(pixels, size=(to_uint8_host.shape[1], to_uint8_host.shape[2]))
                    to_uint8_host.copy_(u8, non_blocking=True)
            if self.conv_ctas > 0:
                _lib.load().lg_vq_set_cta_budget(0)
        self._last = pixels
        return pixels

    def wait(self):
        """Make the current stream wait for every decode submitted so far."""
        torch.cuda.current_stream(self.dev).wait_stream(self.decode_stream)
