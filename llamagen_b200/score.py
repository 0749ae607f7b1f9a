"""Likelihood of complete token sequences in one teacher-forced pass (lg_score in include/llamagen_b200.h): the per-token negative
log-likelihood of Transformer.forward(idx, cond_idx, targets) (gpt.py:341-382, eval mode), optionally under classifier-free
guidance with generate()'s CFG mix. One batched forward over every position instead of the S sequential decode steps of
generate(..., teacher=tokens)."""
from __future__ import annotations

import torch

from .gpt import Transformer


@torch.no_grad()
def score(model, cond, tokens, emb_masks=None, cfg_scale=1.0, return_logits=False):
    """Per-token NLL of `tokens` [B, S] (S <= block_size) given `cond` (c2i: labels [B]; t2i: caption features [B, T, C]).

    Position s is scored from the condition and tokens[:, :s]: nll[b, s] = -log_softmax(logits[b, s])[tokens[b, s]], with the
    logits rounded to the model dtype as the reference's `.float()` of its head output. cfg_scale > 1 scores the guided
    distribution uncond + (cond - uncond) * cfg_scale (generate.py:79-82), the null condition filling the unconditional half.
    emb_masks [B, T] (t2i) mask condition padding as in generate(). The scratch lives on the model (llamagen_b200.gpt.SCORE_SCRATCH_CAP
    bytes at most; larger batches are scored in image chunks). Returns nll fp32 [B, S], and the logits fp32 [B, S, V] with
    return_logits."""
    if not isinstance(model, Transformer):
        raise TypeError("llamagen_b200.score needs a llamagen_b200 GPT_models[...] instance")
    if tokens.dim() != 2 or tokens.shape[0] != cond.shape[0]:
        raise ValueError(f"tokens must be [B, S] with B = {cond.shape[0]}, got {tuple(tokens.shape)}")
    idx = tokens[:, :-1] if tokens.shape[1] > 1 else None
    logits, nll = model._score(cond, idx, tokens, emb_masks, float(cfg_scale), bool(return_logits), True)
    return (nll, logits) if return_logits else nll
