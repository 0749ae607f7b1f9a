"""Drop-in for autoregressive/models/generate.py: same `generate()` signature and return value
(int32 [B, max_new_tokens] on cond.device, generate.py:126-176), executed by ONE C-ABI call: prefill,
the S-1 KV-cached decode steps, CFG mixing and top-k/top-p sampling all stay on the device
(lg_generate in include/llamagen_b200.h); the reference's Python loop of S host iterations is gone.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .gpt import Transformer


def _draw_seed() -> int:
    # torch.multinomial consumes torch's global generator in the reference (generate.py:63); we take one
    # 62-bit draw from the same generator so `torch.manual_seed(s)` keeps runs reproducible.
    return int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())


def _is_rows(x) -> bool:
    """Whether a temperature / top_k / top_p argument is per image (a sequence, array or tensor with a dimension) rather than a number."""
    return isinstance(x, (list, tuple)) or (isinstance(x, (torch.Tensor, np.ndarray)) and x.ndim > 0)


def _filters(temperature, top_k, top_p, B):
    """generate()'s and sample()'s temperature, top_k and top_p. Plain numbers keep the scalar path: (temperature, top_k, top_p, None)
    converted as always. When any of them is a 1-D sequence, array or tensor, each is B per-image values (a number is repeated),
    checked on the host (it is outside input): temperature finite and >= 0, top_k integral (k <= 0: off), top_p not NaN. Returns
    (temperature, top_k, top_p, rows) with rows = (f32 [B], int32 [B], f32 [B]) on the host; the scalars are then unused."""
    if not any(_is_rows(x) for x in (temperature, top_k, top_p)):
        return float(temperature), int(top_k or 0), float(top_p), None

    def rows(name, x):
        try:
            t = torch.as_tensor(x.detach().cpu() if torch.is_tensor(x) else np.asarray(0 if x is None else x))
        except (TypeError, ValueError) as e:
            raise ValueError(f"{name} must hold real numbers, got {x!r}") from e
        if t.dtype == torch.bool or t.dtype.is_complex:
            raise ValueError(f"{name} must hold real numbers, got dtype {t.dtype}")
        if t.dim() > 1 or (t.dim() == 1 and t.shape[0] != B):
            raise ValueError(f"{name} must be a number or {B} values, one per image, got shape {tuple(t.shape)}")
        return t.to(torch.float64).expand(B)
    t, k, p = rows("temperature", temperature), rows("top_k", top_k), rows("top_p", top_p)
    if not bool(torch.isfinite(t).all()) or bool((t < 0).any()):
        raise ValueError(f"temperature must be finite and >= 0, got {t.tolist()}")
    if not bool(torch.isfinite(k).all()) or not bool((k == k.round()).all()):
        raise ValueError(f"top_k must hold integers, got {k.tolist()}")
    if bool(torch.isnan(p).any()):
        raise ValueError(f"top_p must not be NaN, got {p.tolist()}")
    return 1.0, 0, 1.0, (t.float().contiguous(), k.clamp(0, 2 ** 31 - 1).to(torch.int32).contiguous(), p.float().contiguous())


def _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev):
    """The call's SampleCfg, and the device copies of its per-image filter rows (None without them), which the caller keeps alive for
    the call. Draws the seed from torch's generator when seed is None."""
    sc = _lib.SampleCfg(float(cfg_scale), int(cfg_interval), temperature, top_k, top_p, 0 if sample_logits else 1,
                        _draw_seed() if seed is None else int(seed))
    if rows is None:
        return sc, None
    keep = tuple(r.to(dev) for r in rows)
    sc.temperature_rows, sc.top_k_rows, sc.top_p_rows = (r.data_ptr() for r in keep)
    return sc, keep


def sample(logits, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, sample_logits=True, seed=None):
    """generate.py:57-66 on the device: logits [B, T, V] (last position used) -> (idx int64 [B,1], probs [B,V]). temperature, top_k
    and top_p may each be B per-row values (see generate())."""
    lib = _lib.load()
    x = _lib.require_cuda(logits, "sample")[:, -1, :].float().contiguous()
    B, V = x.shape
    idx = torch.empty(B, dtype=torch.int32, device=x.device)
    probs = torch.empty(B, V, dtype=torch.float32, device=x.device)
    temperature, top_k, top_p, rows = _filters(temperature, top_k, top_p, B)
    sc, keep = _sample_cfg(1.0, -1, temperature, top_k, top_p, sample_logits, seed, rows, x.device)
    _lib.check(lib.lg_sample(_lib.ptr(x), B, V, 0, _lib.LG_DTYPE_F32, ctypes.byref(sc), 0, _lib.ptr(idx),
                             _lib.ptr(probs), _lib.current_stream(x.device)), "lg_sample")
    return idx.long().unsqueeze(-1), probs


@torch.no_grad()
def generate(model, cond, max_new_tokens, emb_masks=None, cfg_scale=1.0, cfg_interval=-1, **sampling_kwargs):
    """Same contract as the reference generate() (generate.py:126-176).

    temperature, top_k and top_p may each also be a 1-D sequence, array or tensor of B values, one per image (c2i with CFG: the B
    conditional images; cond_weights: per image, not per condition). Image b then draws exactly what image b of the same call draws
    with the plain number set to value b, on every path below (sjd_window, prefix, given, negatives, cond_weights, return_logprobs,
    teacher, fp16, fp8). Checked on the host with ValueError: B values, temperature finite and >= 0, top_k integral (<= 0: off), top_p
    not NaN. Plain numbers keep the scalar path.

    Extra keyword-only knobs (ignored by the reference signature, all optional):
      seed=int             explicit RNG seed for the multinomial draw
      return_logits=True   also return the per-step CFG-mixed logits [S, B, V] (fp32) for parity tests
      teacher=int tensor   [B, S] tokens fed back instead of the sampled ones (teacher forcing)
      sjd_window=L         speculative Jacobi decoding: up to L tokens per forward pass (2 <= L <= 64; a window longer than
                           max_new_tokens - 1 is shortened to it). The same distribution as plain sampling but other draws for a
                           seed, except token 0; greedy decoding gives the same tokens.
      return_stats=True    with sjd_window: return (tokens, {"iterations": passes, "tokens_per_iteration": ...})
      prefix=int tensor    [B, P] tokens 0 .. P - 1 of every image (1 <= P <= max_new_tokens - 1; e.g. the first rows of an encoded
                           image): the condition and the prefix are prefilled in one forward pass and tokens P .. are sampled as
                           plain generation samples them (same RNG key per token index), so out[:, :P] == prefix. With
                           return_logits, rows k < P of the logits are zero.
      negative_cond=tensor t2i with cfg_scale > 1: a negative prompt, [1, T, C] (one for every image) or [B, T, C], prepared as cond
                           is (cond.pack_t5_features + cond.prepare_condition). It replaces the null condition of the unconditional
                           rows, so the mix uncond + (cond - uncond) * cfg_scale pushes away from it. Works on the plain, prefix and
                           sjd_window paths; not with teacher.
      negative_emb_masks=tensor  [1, T] or [B, T]: the negative's emb-mask (the unconditional rows attend with it). Either of
                           emb_masks / negative_emb_masks left out counts as all ones.
      return_logprobs=True return (tokens, logprobs): f32 [B, S], the log-probability of every drawn token under the distribution the
                           sampler drew it from (logits rounded to the model dtype, CFG-mixed with cfg_interval, divided by
                           temperature, top-k / top-p applied; a greedy draw reports that distribution's value too). Rows k < P of a
                           prefix are 0, so logprobs.sum(1) is the cumulative logprob of the drawn tokens. The tokens are those of the
                           same call without it. Works on the plain, CFG, negative and prefix paths; not with sjd_window, teacher (use
                           score() for given tokens) or return_logits.
      given=int tensor, given_mask=bool tensor
                           inpainting: given [B, S] or [1, S] (one for every image) holds token ids, read only where given_mask
                           ([B, S], [1, S] or [S]) is True; those ids must lie in [0, vocab_size) and at least one mask entry must be
                           False. out[b, k] == given[b, k] wherever the mask is True; every other token is drawn as plain generation
                           draws token k of image b (same RNG key per token index, cfg_interval by token index, the same filters), from
                           a model that has seen every token before k, given or drawn. A raster-order model never sees the given tokens
                           after k (e.g. the rows below a hole): a redrawn region follows what lies above and left of it. The leading
                           run given to every image is prefilled in one pass (as prefix), and every later run given to every image is
                           appended in one window pass instead of one decode step per token. An all-False mask gives exactly the tokens
                           of the call without it, and a mask of the first P columns exactly those of prefix=given[:, :P]. Works with
                           c2i and t2i, emb_masks, negative prompts, fp8 KV caches and fp8 weights; not with prefix, teacher,
                           sjd_window, return_logits or return_logprobs.
      top_logprobs=N       1 <= N <= 20, with return_logprobs: return (tokens, logprobs, {"ranks": int32 [B, S], "top_ids": int32
                           [B, S, N], "top_logprobs": f32 [B, S, N]}). rank = 1 + the number of tokens with a larger processed logit;
                           the top ids are the N kept tokens with the largest logits (ties: lower id first), -1 with logprob -inf past
                           the last kept token. Prefix rows: rank 0, ids -1, logprobs -inf.
      cond_weights=floats  composable guidance (Liu et al. 2022 on logits): K weighted conditions per image, 1 <= K <= 8. cond is
                           int [B, K] class ids in [0, num_classes) (c2i) or [B, K, T, C] captions prepared as cond is (t2i; emb_masks
                           [B, K, T] or None); cond_weights is [K] (every image) or [B, K] (per image, e.g. an interpolation strip),
                           finite, any sign, zeros allowed. Every token is drawn from x = u + d, d = w_1 (c_1 - u) + w_2 (c_2 - u) + ...
                           accumulated left to right in fp32, c_i the logits under condition i and u those of the null condition (or
                           negative_cond), every row rounded to the model dtype first; u attends with the emb-mask of condition 1, or
                           with negative_emb_masks when a negative is given. Temperature, top-k / top-p, greedy and the RNG key (seed,
                           token index, image index) are those of plain generation, so K = 1 with cond_weights=[s], s > 1, gives the
                           tokens of cfg_scale=s bit for bit, and a zero weight drops its condition exactly. The call always mixes:
                           cfg_scale must stay at its default; cfg_interval only with K = 1. Combines with negative_cond /
                           negative_emb_masks ([1 or B, T, C] / [1 or B, T]), prefix ([B, P]), given / given_mask, return_logprobs /
                           top_logprobs (of the composed distribution), fp16, fp8 KV caches and fp8 weights; not with sjd_window,
                           teacher or return_logits. An image runs 2K rows through the model, of which K + 1 are read.
    """
    if not isinstance(model, Transformer):
        raise TypeError("llamagen_b200.generate needs a llamagen_b200 GPT_models[...] instance")
    temperature = sampling_kwargs.pop("temperature", 1.0)
    top_k = sampling_kwargs.pop("top_k", 0)
    top_p = sampling_kwargs.pop("top_p", 1.0)
    sample_logits = bool(sampling_kwargs.pop("sample_logits", True))
    seed = sampling_kwargs.pop("seed", None)
    return_logits = bool(sampling_kwargs.pop("return_logits", False))
    teacher = sampling_kwargs.pop("teacher", None)
    sjd_window = sampling_kwargs.pop("sjd_window", None)
    return_stats = bool(sampling_kwargs.pop("return_stats", False))
    prefix = sampling_kwargs.pop("prefix", None)
    negative_cond = sampling_kwargs.pop("negative_cond", None)
    negative_emb_masks = sampling_kwargs.pop("negative_emb_masks", None)
    return_logprobs = bool(sampling_kwargs.pop("return_logprobs", False))
    top_logprobs = sampling_kwargs.pop("top_logprobs", None)
    given = sampling_kwargs.pop("given", None)
    given_mask = sampling_kwargs.pop("given_mask", None)
    cond_weights = sampling_kwargs.pop("cond_weights", None)
    if sampling_kwargs:
        raise TypeError(f"unexpected sampling kwargs: {sorted(sampling_kwargs)}")
    if top_logprobs is not None:
        if not return_logprobs:
            raise ValueError("top_logprobs needs return_logprobs=True")
        if not _is_int(top_logprobs) or not 1 <= int(top_logprobs) <= _lib.MAX_TOP_LOGPROBS:
            raise ValueError(f"top_logprobs must be an integer in [1, {_lib.MAX_TOP_LOGPROBS}], got {top_logprobs!r}")
    if return_logprobs:
        if sjd_window is not None:
            raise ValueError("return_logprobs cannot be combined with sjd_window")
        if teacher is not None:
            raise ValueError("return_logprobs cannot be combined with teacher: score() gives the log-likelihood of given tokens")
        if return_logits:
            raise ValueError("return_logprobs cannot be combined with return_logits")
    if sjd_window is not None:
        if isinstance(sjd_window, bool) or int(sjd_window) != sjd_window or not 2 <= int(sjd_window) <= 64:
            raise ValueError(f"sjd_window must be an integer in [2, 64], got {sjd_window!r}")
        if teacher is not None or return_logits:
            raise ValueError("sjd_window cannot be combined with teacher or return_logits")
    elif return_stats:
        raise ValueError("return_stats needs sjd_window")
    if cond_weights is not None:
        for name, on in (("sjd_window", sjd_window is not None), ("teacher", teacher is not None), ("return_logits", return_logits),
                         ("return_stats", return_stats)):
            if on:
                raise ValueError(f"cond_weights cannot be combined with {name}")
        return _generate_composed(model, cond, int(max_new_tokens), emb_masks, cfg_scale, cfg_interval, cond_weights,
                                  temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits, seed=seed,
                                  prefix=prefix, negative_cond=negative_cond, negative_emb_masks=negative_emb_masks,
                                  return_logprobs=return_logprobs, top_logprobs=top_logprobs, given=given, given_mask=given_mask)
    if prefix is not None and (teacher is not None or sjd_window is not None):
        raise ValueError("prefix cannot be combined with teacher or sjd_window")
    pf = _check_prefix(prefix, cond.shape[0], int(max_new_tokens), model.vocab_size) if prefix is not None else None
    gv = None
    if given is not None or given_mask is not None:
        for name, on in (("prefix", prefix is not None), ("teacher", teacher is not None), ("sjd_window", sjd_window is not None),
                         ("return_logits", return_logits), ("return_logprobs", return_logprobs)):
            if on:
                raise ValueError(f"given / given_mask cannot be combined with {name}")
        gv = _check_given(given, given_mask, cond.shape[0], int(max_new_tokens), model.vocab_size)
    if negative_cond is not None or negative_emb_masks is not None:
        _check_negative(model, cond, emb_masks, negative_cond, negative_emb_masks, cfg_scale, teacher)

    dev = model.tok_embeddings.weight.device
    _lib.require_cuda(model.tok_embeddings.weight, "generate")
    if model.model_type == "c2i":
        T = 1
        cond_dev = cond.to(device=dev, dtype=torch.int32).contiguous()
        if cond_dev.dim() != 1:
            raise ValueError("c2i cond must be a 1-D tensor of class labels")
    elif model.model_type == "t2i":
        T = cond.shape[1]
        cond_dev = cond.to(device=dev, dtype=model.tok_embeddings.weight.dtype).contiguous()
    else:
        raise Exception("please check model type")            # generate.py:143
    B = cond.shape[0]
    S = int(max_new_tokens)
    use_cfg = cfg_scale > 1.0
    temperature, top_k, top_p, rows = _filters(temperature, top_k, top_p, B)

    em = None
    if emb_masks is not None:
        assert emb_masks.shape[0] == B                          # generate.py:155-156
        assert emb_masks.shape[-1] == T
        em = emb_masks.to(device=dev, dtype=torch.float32).contiguous()
    neg = nm = None
    if negative_cond is not None:                                # both halves get a mask: a missing one is all ones
        neg = negative_cond.to(device=dev, dtype=cond_dev.dtype).expand(B, T, cond_dev.shape[2]).contiguous()
        ones = torch.ones(B, T, dtype=torch.float32, device=dev)
        em = ones if em is None else em
        nm = ones if negative_emb_masks is None else negative_emb_masks.to(device=dev, dtype=torch.float32).expand(B, T).contiguous()

    if sjd_window is not None and S < 3:
        raise ValueError(f"sjd_window needs max_new_tokens >= 3, got {S}")
    model.setup_caches(max_batch_size=2 * B if use_cfg else B, max_seq_length=T + S, dtype=model.tok_embeddings.weight.dtype)
    lib, handle = _lib.load(), model.engine()
    out = torch.empty((B, S), dtype=torch.int32, device=dev)
    if gv is not None:
        sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
        ws, ws_bytes = model._given_scratch(gv, T, use_cfg)
        _lib.check(lib.lg_generate_given(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, T, S, ctypes.byref(sc),
                                         _lib.ptr(gv), ws, ws_bytes, _lib.ptr(out), _lib.current_stream(dev)), "lg_generate_given")
        return out.to(cond.device) if cond.device != dev else out
    if sjd_window is not None:
        sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
        return _generate_sjd(model, lib, handle, cond, cond_dev, em, B, T, S, out, min(int(sjd_window), S - 1), use_cfg, return_stats,
                             sc, neg=neg, nm=nm)
    if return_logprobs:
        sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
        return _generate_logprobs(model, lib, handle, cond, cond_dev, em, neg, nm, pf, B, T, S, sc, out, use_cfg,
                                  None if top_logprobs is None else int(top_logprobs))
    if pf is not None:
        P = pf.shape[1]
        dbg = torch.zeros((S, B, model.vocab_size), dtype=torch.float32, device=dev) if return_logits else None
        pf_dev = pf.to(device=dev, dtype=torch.int32).contiguous()
        ws, ws_bytes = model._prefix_scratch(2 * B if use_cfg else B, T + P, 2 if use_cfg else 1)
        sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
        if neg is None:
            _lib.check(lib.lg_generate_prefix(handle, _lib.ptr(cond_dev), _lib.ptr(em), B, T, S, ctypes.byref(sc), _lib.ptr(pf_dev), P, ws,
                                              ws_bytes, _lib.ptr(out), _lib.ptr(dbg), _lib.current_stream(dev)), "lg_generate_prefix")
        else:
            _lib.check(lib.lg_generate_prefix_neg(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, T, S,
                                                  ctypes.byref(sc), _lib.ptr(pf_dev), P, ws, ws_bytes, _lib.ptr(out), _lib.ptr(dbg),
                                                  _lib.current_stream(dev)), "lg_generate_prefix_neg")
        if cond.device != dev:
            out = out.to(cond.device)
        return (out, dbg) if return_logits else out
    dbg = torch.empty((S, B, model.vocab_size), dtype=torch.float32, device=dev) if return_logits else None
    tf = teacher.to(device=dev, dtype=torch.int32).contiguous() if teacher is not None else None
    if tf is not None and tuple(tf.shape) != (B, S):
        raise ValueError("teacher must be [B, max_new_tokens]")
    sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
    if neg is None:
        _lib.check(lib.lg_generate(handle, _lib.ptr(cond_dev), _lib.ptr(em), B, T, S, ctypes.byref(sc), _lib.ptr(out),
                                   _lib.ptr(dbg), _lib.ptr(tf), _lib.current_stream(dev)), "lg_generate")
    else:
        _lib.check(lib.lg_generate_neg(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, T, S, ctypes.byref(sc),
                                       _lib.ptr(out), _lib.ptr(dbg), None, _lib.current_stream(dev)), "lg_generate_neg")
    if cond.device != dev:
        out = out.to(cond.device)
    return (out, dbg) if return_logits else out


def _check_cond_weights(cfg_scale, cfg_interval, cond_weights):
    """The checks of cond_weights, and of the cfg_scale / cfg_interval beside it, that do not depend on cond (serve.LLM makes them on
    a request's SamplingParams). Returns (weights f64 host [K] or [B, K], K)."""
    if cfg_scale != 1.0:
        raise ValueError(f"cond_weights are the guidance scales of a composed call; leave cfg_scale at its default (got {cfg_scale})")
    w = torch.as_tensor(cond_weights)
    if w.dtype == torch.bool or w.dtype.is_complex:
        raise ValueError(f"cond_weights must be real numbers, got dtype {w.dtype}")
    w = w.detach().to("cpu", torch.float64)
    if w.dim() not in (1, 2):
        raise ValueError(f"cond_weights must be [K] or [B, K], got {tuple(w.shape)}")
    K = w.shape[-1]
    if not 1 <= K <= _lib.MAX_COMPOSE:
        raise ValueError(f"cond_weights has K={K} conditions per image; K must lie in [1, {_lib.MAX_COMPOSE}]")
    if not bool(torch.isfinite(w).all()) or not bool(torch.isfinite(w.float()).all()):
        raise ValueError("cond_weights must be finite (in fp32)")
    if cfg_interval != -1 and K > 1:
        raise ValueError(f"cfg_interval applies to a composed call only with K = 1 (got K={K}, cfg_interval={cfg_interval})")
    return w, K


def _check_compose(model, cond, S, emb_masks, cfg_scale, cfg_interval, cond_weights, negative_cond, negative_emb_masks):
    """generate(cond_weights=...)'s checks, before anything reaches the device. Returns (B, K, T, weights f32 host [B, K])."""
    if not isinstance(model, Transformer):
        raise TypeError("llamagen_b200.generate needs a llamagen_b200 GPT_models[...] instance")
    w, K = _check_cond_weights(cfg_scale, cfg_interval, cond_weights)
    if not torch.is_tensor(cond):
        raise ValueError("cond must be a tensor")
    if model.model_type == "c2i":
        if cond.dtype.is_floating_point or cond.dtype.is_complex or cond.dtype == torch.bool:
            raise ValueError(f"c2i cond of a composed call must be an integer tensor of class ids, got dtype {cond.dtype}")
        if cond.dim() != 2 or cond.shape[1] != K or cond.shape[0] < 1:
            raise ValueError(f"c2i cond of a composed call must be [B, K] = [B, {K}], got {tuple(cond.shape)}")
        c = cond.detach().to("cpu", torch.int64)
        if bool(((c < 0) | (c >= model.num_classes)).any()):
            raise ValueError(f"class ids must lie in [0, num_classes={model.num_classes})")
        if emb_masks is not None or negative_cond is not None or negative_emb_masks is not None:
            raise ValueError("emb_masks and negative prompts apply to text-conditional (t2i) models")
        T = 1
    elif model.model_type == "t2i":
        T, C = model.cls_token_num, model.config.caption_dim
        if cond.dim() != 4 or cond.shape[0] < 1 or tuple(cond.shape[1:]) != (K, T, C):
            raise ValueError(f"t2i cond of a composed call must be [B, K, T, C] = [B, {K}, {T}, {C}], got {tuple(cond.shape)}")
        B = cond.shape[0]
        if emb_masks is not None and tuple(emb_masks.shape) != (B, K, T):
            raise ValueError(f"emb_masks of a composed call must be [B, K, T] = [{B}, {K}, {T}], got {tuple(emb_masks.shape)}")
        if negative_emb_masks is not None and negative_cond is None:
            raise ValueError("negative_emb_masks needs negative_cond")
        if negative_cond is not None and (negative_cond.dim() != 3 or negative_cond.shape[0] not in (1, B)
                                          or tuple(negative_cond.shape[1:]) != (T, C)):
            raise ValueError(f"negative_cond must be [1, T, C] or [B, T, C] = [{B}, {T}, {C}], got {tuple(negative_cond.shape)}")
        if negative_emb_masks is not None and (negative_emb_masks.dim() != 2 or negative_emb_masks.shape[0] not in (1, B)
                                               or negative_emb_masks.shape[1] != T):
            raise ValueError(f"negative_emb_masks must be [1, T] or [B, T] = [{B}, {T}], got {tuple(negative_emb_masks.shape)}")
    else:
        raise Exception("please check model type")
    B = cond.shape[0]
    if w.dim() == 2 and w.shape[0] != B:
        raise ValueError(f"cond_weights must be [K] or [B, K] = [{B}, {K}], got {tuple(w.shape)}")
    if S < 1:
        raise ValueError(f"max_new_tokens must be >= 1, got {S}")
    return B, K, T, w.float().expand(B, K).contiguous()


def _generate_composed(model, cond, S, emb_masks, cfg_scale, cfg_interval, cond_weights, *, temperature, top_k, top_p, sample_logits,
                       seed, prefix, negative_cond, negative_emb_masks, return_logprobs, top_logprobs, given, given_mask):
    """generate(cond_weights=...): lg_generate_composed over B * K conditional rows (image-major) and as many unconditional rows."""
    B, K, T, w = _check_compose(model, cond, S, emb_masks, cfg_scale, cfg_interval, cond_weights, negative_cond, negative_emb_masks)
    temperature, top_k, top_p, rows = _filters(temperature, top_k, top_p, B)   # per image, not per condition
    if prefix is not None and (given is not None or given_mask is not None):
        raise ValueError("given / given_mask cannot be combined with prefix")
    if return_logprobs and (given is not None or given_mask is not None):
        raise ValueError("given / given_mask cannot be combined with return_logprobs")
    pf = _check_prefix(prefix, B, S, model.vocab_size) if prefix is not None else None
    gv = _check_given(given, given_mask, B, S, model.vocab_size) if given is not None or given_mask is not None else None

    dev = model.tok_embeddings.weight.device
    _lib.require_cuda(model.tok_embeddings.weight, "generate")
    R = B * K
    if model.model_type == "c2i":
        cond_dev = cond.reshape(R).to(device=dev, dtype=torch.int32).contiguous()
    else:
        cond_dev = cond.reshape(R, T, cond.shape[3]).to(device=dev, dtype=model.tok_embeddings.weight.dtype).contiguous()
    em = None if emb_masks is None else emb_masks.reshape(R, T).to(device=dev, dtype=torch.float32).contiguous()
    neg = nm = None
    if negative_cond is not None:   # an image's negative and its mask repeat on its K rows; a missing mask is all ones
        neg = negative_cond.to(device=dev, dtype=cond_dev.dtype).expand(B, T, cond_dev.shape[2]).repeat_interleave(K, 0).contiguous()
        ones = torch.ones(R, T, dtype=torch.float32, device=dev)
        em = ones if em is None else em
        nm = ones if negative_emb_masks is None else \
            negative_emb_masks.to(device=dev, dtype=torch.float32).expand(B, T).repeat_interleave(K, 0).contiguous()
    w_dev = w.to(dev)
    model.setup_caches(max_batch_size=2 * R, max_seq_length=T + S, dtype=model.tok_embeddings.weight.dtype)
    lib, handle = _lib.load(), model.engine()
    out = torch.empty((B, S), dtype=torch.int32, device=dev)
    sc, keep = _sample_cfg(cfg_scale, cfg_interval, temperature, top_k, top_p, sample_logits, seed, rows, dev)
    P, pf_dev, g_rows, ws, ws_bytes = 0, None, None, None, 0
    if pf is not None:
        P = pf.shape[1]
        pf_dev = pf.repeat_interleave(K, 0).to(device=dev, dtype=torch.int32).contiguous()
        ws, ws_bytes = model._prefix_scratch(2 * R, T + P, 2)
    if gv is not None:
        g_rows = gv.repeat_interleave(K, 0).contiguous()
        ws, ws_bytes = model._given_scratch(g_rows, T, True)
    extra, spec = None, None
    if return_logprobs:
        top_n = None if top_logprobs is None else int(top_logprobs)
        lp = torch.empty((B, S), dtype=torch.float32, device=dev)
        if top_n is not None:
            extra = {"ranks": torch.empty((B, S), dtype=torch.int32, device=dev),
                     "top_ids": torch.empty((B, S, top_n), dtype=torch.int32, device=dev),
                     "top_logprobs": torch.empty((B, S, top_n), dtype=torch.float32, device=dev)}
        spec = _lib.Logprobs(lp.data_ptr(), *((extra["ranks"].data_ptr(), extra["top_ids"].data_ptr(), extra["top_logprobs"].data_ptr(),
                                               top_n) if extra else (0, 0, 0, 0)))
    _lib.check(lib.lg_generate_composed(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, K, T, S,
                                        ctypes.byref(sc), _lib.ptr(w_dev), _lib.ptr(pf_dev), P, _lib.ptr(g_rows), ws, ws_bytes,
                                        None if spec is None else ctypes.byref(spec), _lib.ptr(out), _lib.current_stream(dev)),
               "lg_generate_composed")
    if cond.device != dev:
        out = out.to(cond.device)
    if not return_logprobs:
        return out
    lp = lp.to(out.device)
    if extra is None:
        return out, lp
    return out, lp, {k: v.to(out.device) for k, v in extra.items()}


def _is_int(x) -> bool:
    return isinstance(x, int) and not isinstance(x, bool)


def _generate_logprobs(model, lib, handle, cond, cond_dev, em, neg, nm, pf, B, T, S, sc, out, use_cfg, top_n):
    """lg_generate_logprobs: generate() with return_logprobs (top_n: None or top_logprobs)."""
    dev = out.device
    lp = torch.empty((B, S), dtype=torch.float32, device=dev)
    extra = None
    if top_n is not None:
        extra = {"ranks": torch.empty((B, S), dtype=torch.int32, device=dev),
                 "top_ids": torch.empty((B, S, top_n), dtype=torch.int32, device=dev),
                 "top_logprobs": torch.empty((B, S, top_n), dtype=torch.float32, device=dev)}
    spec = _lib.Logprobs(lp.data_ptr(), *((extra["ranks"].data_ptr(), extra["top_ids"].data_ptr(), extra["top_logprobs"].data_ptr(),
                                           top_n) if extra else (0, 0, 0, 0)))
    P, pf_dev, ws, ws_bytes = 0, None, None, 0
    if pf is not None:
        P = pf.shape[1]
        pf_dev = pf.to(device=dev, dtype=torch.int32).contiguous()
        ws, ws_bytes = model._prefix_scratch(2 * B if use_cfg else B, T + P, 2 if use_cfg else 1)
    _lib.check(lib.lg_generate_logprobs(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, T, S, ctypes.byref(sc),
                                        _lib.ptr(pf_dev), P, ws, ws_bytes, ctypes.byref(spec), _lib.ptr(out), _lib.current_stream(dev)),
               "lg_generate_logprobs")
    if cond.device != dev:
        out, lp = out.to(cond.device), lp.to(cond.device)
        extra = None if extra is None else {k: v.to(cond.device) for k, v in extra.items()}
    return (out, lp) if extra is None else (out, lp, extra)


def _check_negative(model, cond, emb_masks, negative_cond, negative_emb_masks, cfg_scale, teacher):
    """generate()'s checks of a negative prompt, before anything reaches the device."""
    if model.model_type != "t2i":
        raise ValueError("negative_cond applies to text-conditional (t2i) models; a c2i model has no negative class")
    if negative_cond is None:
        raise ValueError("negative_emb_masks needs negative_cond")
    if not cfg_scale > 1.0:
        raise ValueError(f"a negative prompt replaces the unconditional half of classifier-free guidance: it needs cfg_scale > 1, "
                         f"got {cfg_scale}")
    if teacher is not None:
        raise ValueError("negative_cond cannot be combined with teacher")
    B, T, C = cond.shape[0], cond.shape[1], cond.shape[2]
    if negative_cond.dim() != 3 or negative_cond.shape[0] not in (1, B) or tuple(negative_cond.shape[1:]) != (T, C):
        raise ValueError(f"negative_cond must be [1, T, C] or [B, T, C] = [{B}, {T}, {C}], got {tuple(negative_cond.shape)}")
    if negative_emb_masks is not None and (negative_emb_masks.dim() != 2 or negative_emb_masks.shape[0] not in (1, B)
                                           or negative_emb_masks.shape[1] != T):
        raise ValueError(f"negative_emb_masks must be [1, T] or [B, T] = [{B}, {T}], got {tuple(negative_emb_masks.shape)}")


def _check_prefix(prefix, B, S, V):
    """The prefix as an int64 host tensor [B, P], checked on the host (it is outside input): integer ids in [0, V), 1 <= P <= S - 1."""
    pf = torch.as_tensor(prefix)
    if pf.dtype.is_floating_point or pf.dtype.is_complex or pf.dtype == torch.bool:
        raise ValueError(f"prefix must be an integer tensor of token ids, got dtype {pf.dtype}")
    if pf.dim() != 2 or pf.shape[0] != B:
        raise ValueError(f"prefix must be [B, P] = [{B}, P], got {tuple(pf.shape)}")
    if not 1 <= pf.shape[1] <= S - 1:
        raise ValueError(f"prefix length P={pf.shape[1]} must lie in [1, max_new_tokens - 1 = {S - 1}]")
    pf = pf.detach().to("cpu", torch.int64)
    if bool(((pf < 0) | (pf >= V)).any()):
        raise ValueError(f"prefix token ids must lie in [0, vocab_size={V})")
    return pf


def _check_given(given, given_mask, B, S, V):
    """given / given_mask as one int32 host tensor [B, S]: the given token where the mask is True, -1 where the token is drawn; checked
    on the host (it is outside input): integer ids in [0, V) where given, shapes [B, S] / [1, S] (and [S] for the mask), at least one
    drawn token."""
    if given is None or given_mask is None:
        raise ValueError("given and given_mask go together")
    g = torch.as_tensor(given)
    m = torch.as_tensor(given_mask)
    if g.dtype.is_floating_point or g.dtype.is_complex or g.dtype == torch.bool:
        raise ValueError(f"given must be an integer tensor of token ids, got dtype {g.dtype}")
    if m.dtype != torch.bool:
        raise ValueError(f"given_mask must be a bool tensor, got dtype {m.dtype}")
    if g.dim() != 2 or g.shape[0] not in (1, B) or g.shape[1] != S:
        raise ValueError(f"given must be [B, S] or [1, S] = [{B}, {S}], got {tuple(g.shape)}")
    if m.dim() not in (1, 2) or (m.dim() == 2 and m.shape[0] not in (1, B)) or m.shape[-1] != S:
        raise ValueError(f"given_mask must be [B, S], [1, S] or [S] = [{B}, {S}], got {tuple(m.shape)}")
    g = g.detach().to("cpu", torch.int64).expand(B, S)
    m = m.detach().to("cpu").reshape(-1, S).expand(B, S)
    if bool(m.all()):
        raise ValueError("given_mask is True everywhere: at least one token must be drawn")
    if bool((m & ((g < 0) | (g >= V))).any()):
        raise ValueError(f"given token ids must lie in [0, vocab_size={V}) where given_mask is True")
    return torch.where(m, g, torch.full_like(g, -1)).to(torch.int32).contiguous()


def _generate_sjd(model, lib, handle, cond, cond_dev, em, B, T, S, out, L, use_cfg, return_stats, sc, dbg_probs=None, neg=None, nm=None):
    """lg_generate_sjd with window L (already clamped to S - 1); dbg_probs: None or f32 [S - 1, B, L, V] for replay tests; neg, nm:
    a negative prompt and its mask, [B, T, C] and [B, T] on the device (lg_generate_sjd_neg), or None."""
    dev = out.device
    ws, ws_bytes = model._sjd_scratch(B, use_cfg, L)
    iters = torch.zeros(1, dtype=torch.int32, device=dev)
    if neg is None:
        _lib.check(lib.lg_generate_sjd(handle, _lib.ptr(cond_dev), _lib.ptr(em), B, T, S, ctypes.byref(sc), L, ws, ws_bytes, _lib.ptr(out),
                                       _lib.ptr(iters), _lib.ptr(dbg_probs), _lib.current_stream(dev)), "lg_generate_sjd")
    else:
        _lib.check(lib.lg_generate_sjd_neg(handle, _lib.ptr(cond_dev), _lib.ptr(em), _lib.ptr(neg), _lib.ptr(nm), B, T, S, ctypes.byref(sc),
                                           L, ws, ws_bytes, _lib.ptr(out), _lib.ptr(iters), _lib.ptr(dbg_probs), _lib.current_stream(dev)),
                   "lg_generate_sjd_neg")
    if cond.device != dev:
        out = out.to(cond.device)
    if not return_stats:
        return out
    n = int(iters.item())
    return out, {"iterations": n, "tokens_per_iteration": (S - 1) / max(n, 1)}
