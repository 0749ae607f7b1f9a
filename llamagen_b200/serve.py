"""Continuous-batching front end for class-conditional sampling (SURVEY §8 f-4) with the call surface of the reference's
vLLM-fork entry point: `LLM.generate(prompt_token_ids=..., sampling_params=...)` (autoregressive/serve/llm.py:138-221,
used by autoregressive/serve/sample_c2i.py:39-63) returning `RequestOutput`-shaped objects sorted by request id (:266), and
the engine-style `add_request()` / `step()` loop of autoregressive/serve/llm_engine.py:511.

Iteration-level scheduling: the engine holds `max_num_seqs` sequence slots (slot i = KV-cache rows i and, under CFG, B + i).
Every `step()` (1) admits waiting requests into free slots — they JOIN MID-SEQUENCE of the others, starting at position 0 with
their class embedding — (2) runs ONE decode step for all slots through `lg_decode_rows` (per-row positions: RoPE, cache write
and attention length are per sequence), (3) samples every slot with its own RNG stream (`lg_sample_rows`: request r draws with
seed `base_seed + r`, exactly what a batch-of-one `generate(seed=...)` would draw), and (4) returns the requests that reached
`max_tokens`. Requests have no EOS, so the host knows every sequence's depth without reading the device; the only device->host
copy is the token row of a finished request.

Classifier-free guidance follows the reference's serving protocol (serve/sample_c2i.py:35-37, serve/sampler.py:54-58): the
caller appends one `[num_classes]` (null-class) prompt per conditional prompt; the second half is recognised as the
unconditional twins, the pair is sampled once, and both requests receive the same tokens (the reference samples the two
copies of the mixed logits independently and the caller discards the second half, serve/sample_c2i.py:66-67).

Text-conditional models are served the same way, with one caption's T5 features per request (`add_request(prompt_embeds=...)`,
`LLM.generate(prompt_embeds=[...])`). The condition is built as the samplers build it (cond.pack_t5_features, then
cond.prepare_condition with left padding). A step (1) decodes and samples the running slots through `lg_decode_rows_t2i` and
`lg_sample_rows`, then (2) admits waiting requests into free slots: `lg_prefill_slot` prefills the caption (and, under CFG, the
null condition) into the slot's cache rows alone, and token 0 is drawn from its logits with step 0. A join has the same shapes
whatever else joins or runs, so a request's tokens do not depend on the schedule, and request r draws token k with the key
`generate(seed=base_seed + r)` uses for image 0. CFG is internal: the unconditional row takes the learned null condition, and no
twin requests are involved. temperature=0 decodes greedily (generate's sample_logits=False) on this path.

With a text encoder (`LLM(gpt_t2i, text_encoder=t5.T5Encoder)`), a t2i request may bring its caption as a string
(`LLM.generate(prompts=[...])`, `add_request(prompt=...)`): the batch of strings is one encoder call on the device, and each request is
enqueued exactly as `prompt_embeds` = its valid feature rows would be, so its tokens equal those of that path.

Image completion: a request may bring its first P image tokens (`add_request(..., prefix=ids)`, `LLM.generate(..., prefixes=[...])`,
1 <= P <= max_tokens - 1). Its join is `lg_prefill_slot_prefix`: the condition and the P tokens are prefilled into the slot's cache rows
alone (one row of T + P positions each), token P is drawn from its logits with step P, and the request continues from position T + P
with token index P + 1 — the draws generate(prefix=..., seed=base_seed + r) makes for image 0. A t2i completion request joins where a
caption request joins; a c2i one joins in the admission phase (a c2i request without a prefix still starts at position 0 in the
decode) and takes part in the same step's decode. A request whose join draws its last token (P = max_tokens - 1) finishes at its join.
Null-class twins mirror their conditional request's prefix.

Negative prompts (t2i with cfg_scale > 1): a request may bring a negative caption (`add_request(..., negative_prompt_embeds=...)`,
`LLM.generate(..., negative_prompt_embeds=[...])`, and with a text encoder `negative_prompt=` / `negative_prompts=`, encoded in the same
encoder call as the prompts). It is prepared as the condition is, and the request's unconditional row is prefilled with it and attends
with its mask (`lg_prefill_slot_prefix_neg`, `lg_decode_rows_t2i_neg`), so the request draws what generate(negative_cond=...,
seed=base_seed + r) draws for image 0. Requests with and without a negative share the running batch: a slot without one keeps the null
condition and its caption's mask in its unconditional row.

Per-request guidance and seeds: SamplingParams(cfg_scale=, cfg_interval=, seed=) (None: the LLM's cfg_scale, -1, base_seed + r). The
running set shares only (temperature, top_p, top_k, max_tokens) (with per_request_sampling, max_tokens alone); a change of these waits
for the set to drain, a change of cfg_scale, cfg_interval or seed does not. Under CFG every slot's scale and interval sit in device
arrays (st["cfg"], st["interval"]) that its request's join writes before its first draw, and every draw is lg_sample_rows_guided over
them: a row mixes only when its scale is > 1 and its interval allows it, so a request draws the tokens it draws alone in an LLM built
with its cfg_scale (generate(cfg_scale=c, cfg_interval=k, seed=s) for image 0). A request's seed replaces base_seed + r in st["seeds"]. A
scale > 1 needs an LLM built with cfg_scale > 1 (the unconditional rows); a request at scale <= 1 in such an LLM keeps its
unconditional row running, unread.

Speculative Jacobi decoding (LLM(..., sjd_window=L), 2 <= L <= 64): every step() runs one SJD pass over all slots instead of one decode
step, and makes up to L tokens of every running request final (generate(sjd_window=L)'s pass on per-slot state: lg_sjd_pass_slots).
A request's window is min(L, max_tokens - 1); it draws token 0 at its join as a plain request does (a c2i join is
lg_prefill_slot_prefix with P = 0), then lg_sjd_slot_start keys its window with its own seed and a pass counter from 0, so request r draws
what generate(cond_r, sjd_window=L, seed=s_r) draws for image 0, whatever ran beside it. A step enqueues its pass, then reads the
previous pass's final counts (a pinned copy and an event): a finished request leaves, and its slot is reused, one step after its last
pass; its slot is frozen meanwhile. prefix= requests are refused (as generate() refuses prefix with sjd_window).

Parallel sampling (SamplingParams(n=k), 1 <= k <= max_num_seqs; vLLM's `n`): a request takes k sequence slots (max_num_seqs counts
sequences) and returns one RequestOutput whose outputs are k CompletionOutputs, index 0 .. k - 1. Sample j draws what image j of
generate(cond repeated k times, seed=s) draws (s: the request's seed), with the same guidance, prefix, negative and sjd_window; n = 1 is
image 0, as before. The request joins when k slots are free, all at once, in FIFO order (a later request does not overtake it). A join
that prefills (t2i, a prefix, every SJD join) prefills once, into the first slot; lg_copy_slot_kv then copies positions [0, T + P) of
its K / V rows to the other k - 1 slots (a prefill writes the same bytes whatever the slot), their host-side state is copied too, and the
join's logits are drawn once per slot with the slot's image index (lg_sample_rows_keyed). A plain c2i join has no prefill: its k slots
start at position 0 with the same class. Samples finish independently (under SJD at different passes); a finished sample frees its slot
at once, and the request is returned when its last sample finishes. Null-class twins mirror the request's k outputs.

Token log-probabilities (SamplingParams(logprobs=N), 0 <= N <= 20; vLLM's field): every CompletionOutput then carries
cumulative_logprob and one dict per token_ids entry, None for a given prefix token, otherwise {drawn token: Logprob(logprob, rank)} plus
the N kept tokens with the largest processed logits (Logprob(logprob, 1 .. N)). The numbers are the sample kernel's own, on the
distribution the token was drawn from: the logits rounded to the model dtype, mixed with the request's guidance, divided by temperature
and filtered by top-k / top-p (generate(return_logprobs=True, top_logprobs=N) for image j of the request). Two differences from vLLM:
a greedy (temperature 0, t2i) draw reports that distribution, not the temperature-1 one, and a slot past the last token top-k / top-p
keep is left out rather than filled with arbitrary -inf tokens. Requests with and without logprobs share the running batch; a draw
switches to lg_sample_rows_logprobs only while a running or joining slot needs logprobs, and asks for 20 alternatives whenever one asks
for any (the device rows hold 20 per token). best_of = m (n <= m <= max_num_seqs) draws images 0 .. m - 1 as n = m would and returns
the n with the largest cumulative_logprob, sorted descending (ties: the lower image index first), each with its image index; without
best_of the outputs stay in index order (vLLM always sorts). cumulative_logprob is filled whenever logprobs or best_of is set: the sum of
the drawn tokens' logprobs in float64. Neither field goes with sjd_window.

Inpainting (add_request(..., given=ids, given_mask=mask), LLM.generate(..., givens=[...], given_masks=[...]); c2i and t2i): ids and
mask have shape [max_tokens], checked as generate()'s given / given_mask at B = 1, and the request's token_ids hold ids[k] wherever
mask[k] is True. The request follows the engine's own plan of generate(given=...) at B = 1 (lg_test_given_plan): its leading given run
of P tokens is its prefix (a join through lg_prefill_slot_prefix, P = 0: a plain join); its drawn tokens are drawn by the running
batch's decode and draw; each interior given run [a, a + K) is one window pass over the slot alone (lg_extend_slot: tokens a - 1 ..
a + K - 1 at positions T + a - 1 ..), enqueued after the step's batched decode, whose row for the slot is rewritten by it, and token
a + K is drawn from its logits with the slot's seed, guidance and image index at step a + K; a trailing given run needs no step, the
request finishes when its last drawn token is drawn. While a running or joining slot has given tokens, every draw is
lg_sample_rows_given over the slots' given rows, so a row whose token is given takes it; requests without given draw as before. A
request's passes and their shapes depend only on the request, whatever ran beside it. At cfg_scale 1 they are the passes of
generate(cond, given=ids, given_mask=mask, seed=base_seed + r) at B = 1, so the tokens are that call's bit for bit; under CFG each half
runs its own window pass, so the logits agree with that call's up to rounding. With n = k, sample j is keyed as image j. given goes with everything generate(given=) goes with; prefix=, sjd_window, logprobs and best_of are refused.
Null-class twins mirror their conditional request's given tokens.

Composable guidance (SamplingParams(cond_weights=(w_1, .., w_K)), 1 <= K <= 8, on an LLM built with cfg_scale > 1): a c2i request brings
K class ids (prompt_token_ids=[c_1, .., c_K]), a t2i request K captions (prompt_embeds=[f_1, .., f_K], or prompt=[s_1, .., s_K] with a
text encoder; a bare one when K = 1), and every token is drawn from u + w_1 (c_1 - u) + .. + w_K (c_K - u), as generate(cond_weights=)
draws it: sample j draws what image j of generate(cond repeated n times, cond_weights=w, seed=s) draws, whatever runs beside it. The
request takes n K slots, the lowest free ones at once (sample j's condition i in the (j K + i)-th); condition 1's slot is the sample's
lead (its seed, image index, token row and unconditional row: the null condition or the negative), the others are condition slots
whose unconditional rows run unread. A t2i or prefix join prefills sample 0's K slots alone, fans their K / V out to the other samples
and draws token P once per sample; a c2i join without a prefix enters its K classes at position 0. While a running or joining slot is
composed, every draw is lg_sample_rows_composed over a gather table (st["mix_rows"], st["mix_w"]: -2 for a condition slot, -1 for a
plain one, the lead's rows and weights otherwise), and the leads' tokens become their condition slots' inputs on the device. A sample
frees its K slots together. Not with cfg_scale (the weights are the scales), cfg_interval when K > 1, given / given_mask or sjd_window.
Null-class twins mirror their conditional request's cond_weights and keep the single null class as their prompt.

Per-request sampling filters (LLM(..., per_request_sampling=True)): requests that differ in temperature, top_k or top_p share the running
batch, as requests that differ in cfg_scale or seed do; only a change of max_tokens (which sizes the KV, token and given rows and the SJD
window) still waits for the running set to drain. Without the flag a change of any of the four drains, as before. In both modes every
join writes its slots' temperature, top_k, top_p and greedy flag to device arrays (st["temp"], st["topk"], st["topp"], st["greedy"]) before
its first draw, and every draw, SJD passes included, reads them through SampleCfg's row arrays, so a request draws what it draws alone in
an LLM whose running set shares its filters (generate(cond, seed=s, temperature=t, top_k=k, top_p=p) for image j). A t2i request at
temperature 0 is greedy; c2i keeps the reference's temperature. Under the flag add_request checks the three values as generate() checks
per-image filters (top_k -1 or 0: off), and a null-class twin must carry its request's filters.

While requests are in flight the LLM owns the model's KV-cache workspace (a `generate()` call on the same model would reset it)."""
from __future__ import annotations

import itertools
import math
import numbers
from collections import deque
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import ctypes

import numpy as np
import torch

from . import _lib
from .cond import pack_t5_features, prepare_condition
from .generate import _check_cond_weights, _check_given, _check_prefix, _filters


@dataclass(frozen=True)
class SamplingParams:
    """The vllm.SamplingParams fields the reference sets (serve/sample_c2i.py:47-49). top_k=-1 / 0 disables top-k.
    Per-request guidance and seed (requests that differ only in these share the running batch):
    cfg_scale: None = the LLM's cfg_scale; a finite number, > 1 only on an LLM built with cfg_scale > 1 (it has the unconditional rows).
    cfg_interval: None = -1; an integer >= -1, generate()'s cfg_interval (the mix is dropped after decode iteration cfg_interval).
    seed: None = the LLM's seed + request id; an integer in [0, 2**63), the key generate(seed=...) draws image 0 with.
    n: the number of images of the request, an integer in [1, max_num_seqs]; image j is what image j of generate(cond repeated n times,
    seed=seed) draws. Requests that differ in n share the running batch.
    logprobs: None, or an integer in [0, 20]: return every drawn token's logprob and rank and its `logprobs` most likely alternatives.
    best_of: None, or an integer in [n, max_num_seqs]: draw best_of images and return the n with the largest cumulative_logprob.
    Requests that differ in logprobs or best_of share the running batch.
    cond_weights: None, or K finite weights (1 <= K <= 8, any sign, zeros allowed; stored as a tuple): composable guidance, every token
    drawn from u + w_1 (c_1 - u) + ... + w_K (c_K - u) over the request's K conditions (generate(cond_weights=)). Needs an LLM built
    with cfg_scale > 1 and no sjd_window; not with cfg_scale (the weights are the scales), given / given_mask, or cfg_interval when
    K > 1. A request takes n * K sequence slots. Requests that differ in cond_weights share the running batch.
    temperature, top_k, top_p: the request's filters (top_k -1 or 0: off; temperature 0 on a t2i LLM: greedy). A change of them waits
    for the running set to drain, unless the LLM was built with per_request_sampling=True: then they are per request, checked when
    the request is added (temperature finite and >= 0, top_k an integer, top_p not NaN), and requests that differ in them share the
    running batch."""
    temperature: float = 1.0
    top_p: float = 1.0
    top_k: int = -1
    max_tokens: int = 256
    cfg_scale: Optional[float] = None
    cfg_interval: Optional[int] = None
    seed: Optional[int] = None
    n: int = 1
    logprobs: Optional[int] = None
    best_of: Optional[int] = None
    cond_weights: Optional[Sequence[float]] = None

    def __post_init__(self):
        if self.cond_weights is not None and not isinstance(self.cond_weights, (str, bytes)):
            try:
                object.__setattr__(self, "cond_weights", tuple(self.cond_weights))
            except TypeError:   # not a sequence: refused when a request is added
                pass


def _wants_logprobs(p: SamplingParams) -> bool:
    """Whether a request's draws need the device's logprob outputs."""
    return p.logprobs is not None or p.best_of is not None


def _batch_key(p: SamplingParams):
    """The parameters every request of a running set shares; a change of these waits for the set to drain."""
    return (p.temperature, p.top_p, p.top_k, p.max_tokens)


def _is_int(x) -> bool:
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


@dataclass
class Logprob:
    """vLLM's Logprob without the decoded text: a token's log-probability and its rank among the processed logits (1 = largest)."""
    logprob: float
    rank: int


@dataclass
class CompletionOutput:
    index: int
    token_ids: List[int]
    finish_reason: str = "length"
    cumulative_logprob: Optional[float] = None
    logprobs: Optional[List[Optional[Dict[int, Logprob]]]] = None


@dataclass
class RequestOutput:
    request_id: str
    prompt_token_ids: List[int]
    outputs: List[CompletionOutput] = field(default_factory=list)
    finished: bool = False


@dataclass
class _Request:
    request_id: str
    prompt_token_ids: List[int]
    params: SamplingParams
    twin_of: Optional[str] = None      # request id of the conditional request this null-class request mirrors
    cond: Optional[torch.Tensor] = None   # t2i: the prepared condition, fp32 [T, caption_dim] on the host
    mask: Optional[torch.Tensor] = None   # t2i: its emb-mask, fp32 [T]
    prefix: Optional[torch.Tensor] = None  # image completion: the given tokens 0 .. P - 1, int64 [P] on the host
    neg: Optional[torch.Tensor] = None     # t2i: a negative prompt's prepared condition, fp32 [T, caption_dim] on the host, or None
    neg_mask: Optional[torch.Tensor] = None   # and its emb-mask, fp32 [T]
    cfg: float = 1.0                       # the request's guidance scale, cfg_interval and RNG seed, resolved at enqueue
    interval: int = -1
    seed: int = 0
    n: int = 1                             # its images (sequence slots): best_of, else n
    done: dict = field(default_factory=dict)   # image index -> token ids of every finished sample
    done_lp: dict = field(default_factory=dict)   # image index -> (logprob, rank, top ids, top logprobs) rows, when it wants them
    given: Optional[torch.Tensor] = None   # inpainting: int32 [S] on the host, the given token where given, -1 where drawn
    extends: dict = field(default_factory=dict)   # inpainting: start a of every interior given run -> its length K
    end: int = 0                           # the index after the last drawn token (max_tokens without a trailing given run)
    weights: Optional[tuple] = None        # composable guidance: the K weights (fp32 values), or None
    conds: Optional[list] = None           # t2i composed: the K prepared (condition, emb-mask) pairs; conds[0] is (cond, mask)

    @property
    def K(self) -> int:
        """Conditions per image: a sample takes K sequence slots."""
        return 1 if self.weights is None else len(self.weights)


def _plen(req: _Request) -> int:
    """P, the number of given image tokens of a request (0 without a prefix)."""
    return 0 if req.prefix is None else int(req.prefix.numel())


def _given_plan(given: torch.Tensor):
    """The engine's plan of generate(given=...) at B = 1 for one request's given row (int32 [S], -1: drawn), lg_test_given_plan:
    (P, {a: K} of every EXTEND, the index after the last drawn token)."""
    S = int(given.numel())
    row = np.ascontiguousarray(given.numpy(), dtype=np.int32)
    segs = np.zeros((S + 1, 3), dtype=np.int32)
    n = _lib.load().lg_test_given_plan(row.ctypes.data_as(ctypes.c_void_p), 1, S, segs.ctypes.data_as(ctypes.c_void_p), S + 1)
    _lib.check(n, "lg_test_given_plan")
    segs = segs[:n].tolist()
    tail = [ln for kind, _, ln in segs if kind == 3]
    return segs[0][2], {a: K for kind, a, K in segs if kind == 2}, S - sum(tail)


class LLM:
    def __init__(self, gpt_model, cfg_scale: float = 1.0, num_classes: int = 1000, max_num_seqs: int = 64, seed: Optional[int] = None,
                 kv_cache_dtype: Optional[str] = None, weight_dtype: Optional[str] = None, text_encoder=None, sjd_window: Optional[int] = None,
                 per_request_sampling: bool = False):
        """kv_cache_dtype: None keeps the model's KV-cache setting (Transformer.set_kv_cache, scales included); "auto" (the model
        dtype) or "fp8" (e4m3) sets it. Passing the dtype the model already has keeps its scales.
        weight_dtype: None keeps the model's GEMM-weight storage (Transformer.set_weight_dtype, its head choice included); "auto" or
        "fp8" sets it.
        A t2i model serves caption requests (prompt_embeds); num_classes does not apply to it.
        text_encoder (t2i only): a t5.T5Encoder whose d_model is the model's caption_dim. Requests may then bring caption strings
        (generate(prompts=...), add_request(prompt=...)); each is encoded on the device and enqueued exactly as prompt_embeds = its
        valid feature rows would be.
        sjd_window: None, or an integer L in [2, 64]: every step() runs one speculative Jacobi decoding pass over all slots (up to
        min(L, max_tokens - 1) tokens of every running request per step; max_tokens >= 3, no prefix requests). sjd_passes counts the
        passes run, sjd_tokens the tokens they made final, sjd_request_passes the passes of every finished request.
        per_request_sampling: False (the default) keeps one (temperature, top_k, top_p) per running set: a request with other filters
        waits until every running request finished. True makes them per request: requests that differ in them share the running batch,
        and only a change of max_tokens drains."""
        if sjd_window is not None and (not _is_int(sjd_window) or not 2 <= int(sjd_window) <= 64):
            raise ValueError(f"sjd_window must be an integer in [2, 64], got {sjd_window!r}")
        self.sjd_window = None if sjd_window is None else int(sjd_window)
        self.per_request_sampling = bool(per_request_sampling)
        self.sjd_passes = 0
        self.sjd_tokens = 0
        self.sjd_request_passes: dict[str, int] = {}
        if gpt_model.model_type not in ("c2i", "t2i"):
            raise ValueError(f"serve.LLM handles c2i and t2i models, got model_type {gpt_model.model_type!r}")
        self.t2i = gpt_model.model_type == "t2i"
        if text_encoder is not None:
            if not self.t2i:
                raise ValueError("a text_encoder goes with a text-conditional (t2i) model; a c2i model takes class ids")
            if int(text_encoder.d_model) != gpt_model.config.caption_dim:
                raise ValueError(f"text_encoder.d_model {text_encoder.d_model} != the model's caption_dim {gpt_model.config.caption_dim}")
        self.text_encoder = text_encoder
        if kv_cache_dtype is not None and kv_cache_dtype != getattr(gpt_model, "_kv_cache", ("auto", None))[0]:
            gpt_model.set_kv_cache(kv_cache_dtype)
        if weight_dtype is not None and weight_dtype != getattr(gpt_model, "_weight_dtype", ("auto", True))[0]:
            gpt_model.set_weight_dtype(weight_dtype)
        self.model = gpt_model
        self.cfg_scale = float(cfg_scale)
        self.num_classes = int(num_classes)
        self.max_num_seqs = int(max_num_seqs)
        self.request_counter = itertools.count()
        self._waiting: deque[_Request] = deque()
        self._twins: dict[str, _Request] = {}
        self._seed = int(torch.randint(0, 2 ** 31, (1,)).item()) if seed is None else int(seed)
        self._slots: List[Optional[_Request]] = [None] * self.max_num_seqs
        self._depth = [0] * self.max_num_seqs          # tokens sampled so far per slot (== position of the next input)
        self._img = [0] * self.max_num_seqs            # image index of every slot's sample within its request
        self._lead = list(range(self.max_num_seqs))    # the lead slot of every slot's sample (itself, except for condition slots)
        self._params: Optional[SamplingParams] = None  # sampling parameters of the running set
        self._state = None                             # device tensors, allocated for (max_num_seqs, max_tokens)
        self.steps_run = 0

    # ------------------------------------------------------------------ engine-style surface (llm_engine.py)
    def add_request(self, prompt_token_ids: Optional[Sequence[int]] = None, sampling_params: Optional[SamplingParams] = None, twin_of=None,
                    prompt_embeds=None, prefix=None, prompt: Optional[str] = None, negative_prompt_embeds=None,
                    negative_prompt: Optional[str] = None, given=None, given_mask=None) -> str:
        """c2i: prompt_token_ids = [class id] (twin_of: see LLM.generate). t2i: prompt_embeds = one caption's T5 features, [n, caption_dim]
        or the .npy layout [1, n, caption_dim] (array or tensor, n >= 1, truncated at cls_token_num).
        prefix: image completion, the first P image tokens (1-D integer ids in [0, vocab_size), 1 <= P <= max_tokens - 1); the
        request's token_ids start with them. A null-class twin takes its conditional request's prefix (passing another one is an error).
        prompt: a caption string, with a text_encoder only (instead of prompt_embeds).
        negative_prompt_embeds (t2i, cfg_scale > 1): a negative caption's T5 features, shaped as prompt_embeds; the request's
        unconditional row takes it instead of the null condition. negative_prompt: its string, with a text_encoder only (one encoder
        call with prompt).
        given, given_mask: inpainting, token ids [max_tokens] and a bool mask [max_tokens] with at least one False (generate()'s checks
        at B = 1); the request keeps given[k] wherever given_mask[k] is True and draws the rest. Not with prefix, sjd_window, logprobs
        or best_of. A null-class twin takes its conditional request's (passing other ones is an error).
        With SamplingParams.cond_weights of K weights: c2i prompt_token_ids = [c_1, .., c_K] (class ids in [0, num_classes); a twin's
        prompt stays [num_classes]); t2i prompt_embeds = a list of K captions (or one when K = 1), prompt = a list of K strings."""
        composed = sampling_params is not None and sampling_params.cond_weights is not None
        if prompt is not None or negative_prompt is not None:
            many = composed and isinstance(prompt, (list, tuple))   # a composed request's K caption strings
            texts = (list(prompt) if many else [t for t in (prompt,) if t is not None]) + [t for t in (negative_prompt,) if t is not None]
            if prompt is not None and prompt_embeds is not None:
                raise ValueError("pass caption strings (prompts) or their features (prompt_embeds), not both")
            if negative_prompt is not None and negative_prompt_embeds is not None:
                raise ValueError("pass negative_prompt or negative_prompt_embeds, not both")
            feats = self._encode_prompts(texts)
            if prompt is not None:
                prompt_embeds = feats[:len(prompt)] if many else feats.pop(0)
                feats = feats[len(prompt):] if many else feats
            if negative_prompt is not None:
                negative_prompt_embeds = feats.pop(0)
        if self.t2i:
            if prompt_token_ids is not None or twin_of is not None:
                raise ValueError("a t2i LLM takes prompt_embeds (T5 caption features), not prompt_token_ids; CFG needs no twin requests")
            scale = self._guidance(sampling_params)[0]
            if composed:
                conds = self._captions(prompt_embeds, sampling_params)
                negative = self._negative(negative_prompt_embeds, scale)
                pf = self._prefix(prefix, sampling_params)
                self._given(given, given_mask, sampling_params, pf)
                return self._enqueue_t2i(conds[0], sampling_params, pf, negative, conds=conds)
            caption = self._caption(prompt_embeds)
            negative = self._negative(negative_prompt_embeds, scale)
            pf = self._prefix(prefix, sampling_params)
            gv = self._given(given, given_mask, sampling_params, pf)
            if gv is not None:
                return self._enqueue_t2i(caption, sampling_params, pf, negative, gv)
            return self._enqueue_t2i(caption, sampling_params, pf) if negative is None else self._enqueue_t2i(caption, sampling_params, pf,
                                                                                                              negative)
        if negative_prompt_embeds is not None:
            raise ValueError("negative prompts apply to text-conditional (t2i) models")
        if prompt_embeds is not None:
            raise ValueError("prompt_embeds apply to text-conditional (t2i) models; a c2i prompt is prompt_token_ids = [class id]")
        if prompt_token_ids is None:
            raise ValueError("a c2i request needs prompt_token_ids = [class id]")
        ids = self._class_ids(prompt_token_ids, sampling_params, twin_of)
        self._guidance(sampling_params)
        if twin_of is None:
            pf = self._prefix(prefix, sampling_params)
            gv = self._given(given, given_mask, sampling_params, pf)
        else:
            gv = self._twin_given(twin_of, given, given_mask, sampling_params, prefix)
            pf = self._twin_prefix(twin_of, prefix, sampling_params)
            self._twin_guidance(twin_of, sampling_params)
        rid = str(next(self.request_counter))
        req = self._guided(_Request(rid, ids, sampling_params or SamplingParams(), twin_of, prefix=pf))
        self._set_given(req, gv)
        if twin_of is None:
            self._waiting.append(req)
        else:
            self._twins[twin_of] = req
        return rid

    def _class_ids(self, prompt_token_ids, sampling_params: Optional[SamplingParams], twin_of=None) -> List[int]:
        """A c2i prompt's class ids: one id in [0, num_classes] (num_classes: the null class), or for a composed request (not a twin,
        which keeps the single null class) K ids in [0, num_classes), one per weight."""
        if sampling_params is not None and sampling_params.cond_weights is not None and twin_of is None:
            K = len(self._weights(sampling_params, self._guidance(sampling_params)[1]))
            ids = list(prompt_token_ids)
            if len(ids) != K or not all(_is_int(c) and 0 <= int(c) < self.num_classes for c in ids):
                raise ValueError(f"a composed c2i prompt is K = {K} class ids in [0, {self.num_classes}), one per weight, got {ids}")
            return [int(c) for c in ids]
        if len(prompt_token_ids) != 1 or not (0 <= int(prompt_token_ids[0]) <= self.num_classes):
            raise ValueError(f"a c2i prompt is one class id in [0, {self.num_classes}], got {list(prompt_token_ids)}")
        return [int(prompt_token_ids[0])]

    @staticmethod
    def _composed(sampling_params, i: int) -> bool:
        """Whether request i of an LLM.generate call (sampling_params: one SamplingParams, a list, or None) has cond_weights."""
        sp = sampling_params[i] if isinstance(sampling_params, list) and i < len(sampling_params) else sampling_params
        return isinstance(sp, SamplingParams) and sp.cond_weights is not None

    def _encode_prompts(self, prompts, prompt_embeds=None):
        """Caption strings -> one [valid_len, d_model] feature tensor each (one text_encoder call for the batch)."""
        if self.text_encoder is None:
            raise ValueError("prompts must be None: the image models have no tokenizer (skip_tokenizer_init=True)")
        if prompt_embeds is not None:
            raise ValueError("pass caption strings (prompts) or their features (prompt_embeds), not both")
        prompts = [prompts] if isinstance(prompts, str) else list(prompts)
        if not prompts or not all(isinstance(p, str) for p in prompts):
            raise ValueError("prompts must be a non-empty list of caption strings")
        embs, mask = self.text_encoder(prompts)
        return [embs[i][mask[i] != 0] for i in range(len(prompts))]

    def _caption(self, feats):
        """One caption's (condition fp32 [T, caption_dim], emb-mask fp32 [T]) on the host, exactly as the samplers build a batch row:
        cond.pack_t5_features (truncation at T), then cond.prepare_condition with left padding."""
        T, C = self.model.cls_token_num, self.model.config.caption_dim
        if feats is None:
            raise ValueError("a t2i request needs prompt_embeds (one caption's T5 features)")
        f = feats.detach().cpu() if torch.is_tensor(feats) else torch.as_tensor(np.asarray(feats))
        if f.dim() == 3 and f.shape[0] == 1:
            f = f[0]
        if f.dim() != 2 or f.shape[1] != C:
            raise ValueError(f"prompt_embeds must be [n, {C}] or [1, n, {C}], got {tuple(f.shape)}")
        if f.shape[0] == 0:
            raise ValueError("prompt_embeds holds an empty caption (n = 0)")
        embs, masks = pack_t5_features([f], max_len=T, dim=C)
        cond, mask = prepare_condition(embs, masks, left_padding=True)
        return cond[0], mask[0]

    def _captions(self, feats, sampling_params: SamplingParams) -> list:
        """A composed t2i request's K captions, [(condition, emb-mask)] prepared as _caption prepares one: feats is a list of K
        prompt_embeds, or, when K = 1, one bare prompt_embeds."""
        K = len(self._weights(sampling_params, -1 if sampling_params.cfg_interval is None else sampling_params.cfg_interval))
        if feats is None:
            raise ValueError(f"a composed t2i request needs prompt_embeds = a list of K = {K} captions' T5 features")
        many = isinstance(feats, (list, tuple))
        if not many and K != 1:
            raise ValueError(f"a composed t2i request takes a list of K = {K} captions, one per weight; got one caption")
        feats = list(feats) if many else [feats]
        if len(feats) != K:
            raise ValueError(f"a composed t2i request takes K = {K} captions, one per weight; got {len(feats)}")
        return [self._caption(f) for f in feats]

    def _negative(self, feats, scale: Optional[float] = None):
        """A negative caption's (condition fp32 [T, caption_dim], emb-mask fp32 [T]) on the host, prepared as _caption prepares the
        condition; None stays None. A negative replaces the null condition of CFG: it needs cfg_scale > 1, the LLM's and the request's
        (scale, its effective cfg_scale; None: the LLM's)."""
        if feats is None:
            return None
        if not self.cfg_scale > 1.0:
            raise ValueError(f"a negative prompt replaces the unconditional half of classifier-free guidance: it needs cfg_scale > 1, "
                             f"this LLM has {self.cfg_scale}")
        if scale is not None and not scale > 1.0:
            raise ValueError(f"a negative prompt replaces the unconditional half of classifier-free guidance: it needs cfg_scale > 1, "
                             f"the request has {scale}")
        return self._caption(feats)

    def _guidance(self, sampling_params: Optional[SamplingParams]):
        """A request's (cfg_scale, cfg_interval, seed or None) with the LLM's defaults applied, checked before anything is queued."""
        sp = sampling_params or SamplingParams()
        scale = self.cfg_scale if sp.cfg_scale is None else sp.cfg_scale
        if isinstance(scale, (bool, np.bool_)) or not isinstance(scale, numbers.Real) or not math.isfinite(scale):
            raise ValueError(f"SamplingParams.cfg_scale must be a finite number, got {sp.cfg_scale!r}")
        scale = float(scale)
        if scale > 1.0 and not self.cfg_scale > 1.0:
            raise ValueError(f"SamplingParams.cfg_scale {scale} > 1 needs an LLM built with cfg_scale > 1 (this one has {self.cfg_scale} and "
                             f"runs no unconditional rows)")
        interval = -1 if sp.cfg_interval is None else sp.cfg_interval
        if not _is_int(interval) or interval < -1:
            raise ValueError(f"SamplingParams.cfg_interval must be an integer >= -1, got {sp.cfg_interval!r}")
        if sp.seed is not None and (not _is_int(sp.seed) or not 0 <= sp.seed < 2 ** 63):
            raise ValueError(f"SamplingParams.seed must be an integer in [0, 2**63), got {sp.seed!r}")
        if self.sjd_window is not None and int(sp.max_tokens) < 3:
            raise ValueError(f"sjd_window needs max_tokens >= 3, got {sp.max_tokens}")
        if not _is_int(sp.n) or not 1 <= sp.n <= self.max_num_seqs:
            raise ValueError(f"SamplingParams.n must be an integer in [1, max_num_seqs = {self.max_num_seqs}], got {sp.n!r}")
        if sp.logprobs is not None and (not _is_int(sp.logprobs) or not 0 <= sp.logprobs <= _lib.MAX_TOP_LOGPROBS):
            raise ValueError(f"SamplingParams.logprobs must be None or an integer in [0, {_lib.MAX_TOP_LOGPROBS}], got {sp.logprobs!r}")
        if sp.best_of is not None and (not _is_int(sp.best_of) or not sp.n <= sp.best_of <= self.max_num_seqs):
            raise ValueError(f"SamplingParams.best_of must be None or an integer in [n = {sp.n}, max_num_seqs = {self.max_num_seqs}], "
                             f"got {sp.best_of!r}")
        if self.sjd_window is not None and _wants_logprobs(sp):
            raise ValueError("logprobs and best_of cannot be combined with sjd_window")
        self._weights(sp, int(interval))
        if self.per_request_sampling:   # generate()'s checks of per-image filters, at B = 1
            _filters((sp.temperature,), (sp.top_k,), (sp.top_p,), 1)
        return scale, int(interval), None if sp.seed is None else int(sp.seed)

    def _weights(self, sp: SamplingParams, interval: int) -> Optional[tuple]:
        """A request's cond_weights as a tuple of fp32 values (None without them), checked as generate(cond_weights=) checks them at
        B = 1, with the LLM's own conditions: unconditional rows (cfg_scale > 1), no sjd_window, and n * K, best_of * K slots."""
        if sp.cond_weights is None:
            return None
        if not self.cfg_scale > 1.0:
            raise ValueError(f"SamplingParams.cond_weights mixes each condition with the unconditional rows: it needs an LLM built with "
                             f"cfg_scale > 1, this one has {self.cfg_scale}")
        if sp.cfg_scale is not None:
            raise ValueError("SamplingParams.cond_weights are the request's guidance scales; leave SamplingParams.cfg_scale at None")
        if self.sjd_window is not None:
            raise ValueError("SamplingParams.cond_weights cannot be combined with sjd_window")
        if isinstance(sp.cond_weights, (str, bytes)) or not isinstance(sp.cond_weights, tuple):
            raise ValueError(f"SamplingParams.cond_weights must be a sequence of K weights, got {sp.cond_weights!r}")
        try:
            w, K = _check_cond_weights(1.0, interval, sp.cond_weights)
        except (TypeError, RuntimeError) as e:
            raise ValueError(f"SamplingParams.cond_weights must be a sequence of K real numbers, got {sp.cond_weights!r}") from e
        if w.dim() != 1:
            raise ValueError(f"SamplingParams.cond_weights must be a sequence of K weights, got shape {tuple(w.shape)}")
        m = sp.n if sp.best_of is None else sp.best_of
        if m * K > self.max_num_seqs:
            raise ValueError(f"a composed request takes {'best_of' if sp.best_of is not None else 'n'} * K = {m} * {K} sequence slots, more "
                             f"than max_num_seqs = {self.max_num_seqs}")
        return tuple(float(x) for x in w.float())

    def _guided(self, req: _Request) -> _Request:
        """req with its guidance, seed (None: the LLM's seed + request id) and image count resolved."""
        req.cfg, req.interval, seed = self._guidance(req.params)
        req.seed = self._seed + int(req.request_id) if seed is None else seed
        req.n = int(req.params.n if req.params.best_of is None else req.params.best_of)
        req.weights = self._weights(req.params, req.interval) if req.twin_of is None else None
        return req

    def _twin_guidance(self, twin_of, sampling_params: Optional[SamplingParams]):
        """A null-class twin mirrors its conditional request: its params may not carry another cfg_scale, cfg_interval, seed, n,
        logprobs or best_of."""
        owner = self._owner(twin_of)
        sp = sampling_params or SamplingParams()
        mirror = lambda p: (p.cfg_scale, p.cfg_interval, p.seed, p.n, p.logprobs, p.best_of, p.cond_weights)   # noqa: E731
        if owner is not None and mirror(sp) != mirror(owner.params):
            raise ValueError(f"a null-class twin mirrors its conditional request {twin_of!r}: its cfg_scale, cfg_interval, seed, n, "
                             f"logprobs, best_of and cond_weights must be the request's")
        filters = lambda p: (p.temperature, p.top_k, p.top_p)   # noqa: E731
        if self.per_request_sampling and owner is not None and filters(sp) != filters(owner.params):
            raise ValueError(f"a null-class twin mirrors its conditional request {twin_of!r}: its temperature, top_k and top_p must be "
                             f"the request's")

    def _prefix(self, prefix, sampling_params: Optional[SamplingParams]) -> Optional[torch.Tensor]:
        """A request's prefix as int64 [P] on the host, checked as generate(prefix=...) checks it: integer ids in [0, vocab_size),
        1 <= P <= max_tokens - 1. None stays None."""
        if prefix is None:
            return None
        if self.sjd_window is not None:
            raise ValueError("prefix cannot be combined with sjd_window")
        pf = prefix if torch.is_tensor(prefix) else torch.as_tensor(np.asarray(prefix))
        if pf.dim() != 1:
            raise ValueError(f"a request's prefix is 1-D, [P] image token ids, got shape {tuple(pf.shape)}")
        S = int((sampling_params or SamplingParams()).max_tokens)
        return _check_prefix(pf[None], 1, S, self.model.vocab_size)[0]

    def _given(self, given, given_mask, sampling_params: Optional[SamplingParams], prefix) -> Optional[torch.Tensor]:
        """A request's given tokens as int32 [max_tokens] on the host, -1 where drawn, checked as generate(given=, given_mask=) checks
        them at B = 1; None without them."""
        if given is None and given_mask is None:
            return None
        if self.sjd_window is not None:
            raise ValueError("given / given_mask cannot be combined with sjd_window")
        if prefix is not None:
            raise ValueError("given / given_mask cannot be combined with prefix (a leading given run already is a prefix)")
        sp = sampling_params or SamplingParams()
        if _wants_logprobs(sp):
            raise ValueError("given / given_mask cannot be combined with SamplingParams.logprobs or best_of")
        if sp.cond_weights is not None:
            raise ValueError("given / given_mask cannot be combined with SamplingParams.cond_weights")
        S = int(sp.max_tokens)
        g, m = [None if x is None else x.detach().cpu() if torch.is_tensor(x) else torch.as_tensor(np.asarray(x)) for x in (given, given_mask)]
        for name, x in (("given", g), ("given_mask", m)):
            if x is not None and x.dim() != 1:
                raise ValueError(f"a request's {name} is 1-D, [max_tokens = {S}], got shape {tuple(x.shape)}")
        return _check_given(None if g is None else g[None], m, 1, S, self.model.vocab_size)[0]

    def _set_given(self, req: _Request, gv: Optional[torch.Tensor]) -> _Request:
        """req with its given tokens and plan (_given_plan); the leading given run becomes its prefix (its join is a prefix join)."""
        req.end = int(req.params.max_tokens)
        if gv is not None:
            P, req.extends, req.end = _given_plan(gv)
            req.given = gv
            req.prefix = gv[:P].to(torch.int64) if P > 0 else None
        return req

    def _twin_given(self, twin_of, given, given_mask, sampling_params: Optional[SamplingParams], prefix) -> Optional[torch.Tensor]:
        """The given tokens of a null-class twin: its conditional request's. Given tokens passed for the twin must equal them."""
        owner = self._owner(twin_of)
        mine = None if owner is None else owner.given
        if given is not None or given_mask is not None:
            gv = self._given(given, given_mask, sampling_params, prefix)
            if mine is None or not torch.equal(gv, mine):
                raise ValueError(f"a null-class twin mirrors the given tokens of its conditional request {twin_of!r}; it was given other ones")
        return mine

    def _owner(self, twin_of) -> Optional[_Request]:
        """The waiting or running conditional request a null-class twin mirrors, or None."""
        return next((r for r in itertools.chain(self._waiting, self._slots) if r is not None and r.request_id == twin_of), None)

    def _twin_prefix(self, twin_of, prefix, sampling_params: Optional[SamplingParams]) -> Optional[torch.Tensor]:
        """The prefix of a null-class twin: its conditional request's. A prefix passed for the twin must equal it."""
        owner = self._owner(twin_of)
        mine = None if owner is None or owner.given is not None else owner.prefix
        if prefix is not None:
            pf = self._prefix(prefix, sampling_params)
            if mine is None or not torch.equal(pf, mine):
                raise ValueError(f"a null-class twin mirrors the prefix of its conditional request {twin_of!r}; it was given another one")
        return mine

    def _enqueue_t2i(self, caption, sampling_params: Optional[SamplingParams], prefix: Optional[torch.Tensor] = None, negative=None,
                     given: Optional[torch.Tensor] = None, conds: Optional[list] = None) -> str:
        rid = str(next(self.request_counter))
        neg, neg_mask = negative if negative is not None else (None, None)
        self._waiting.append(self._set_given(self._guided(_Request(rid, [], sampling_params or SamplingParams(), cond=caption[0],
                                                                   mask=caption[1], prefix=prefix, neg=neg, neg_mask=neg_mask,
                                                                   conds=conds)), given))
        return rid

    def _running(self) -> int:
        return sum(r is not None for r in self._slots)

    def has_unfinished_requests(self) -> bool:
        return bool(self._waiting) or self._running() > 0

    def get_num_unfinished_requests(self) -> int:
        return len(self._waiting) + len({id(r) for r in self._slots if r is not None}) + len(self._twins)

    def _admit(self, params: SamplingParams):
        """Admission: the waiting requests that share the running set's sampling parameters, in FIFO order, each into its n K lowest free
        slots (image j's condition i in the (j K + i)-th; K = 1 without cond_weights); the first request without n K free slots waits,
        and every request behind it. Returns [(slots, req)]."""
        free = [i for i in range(self.max_num_seqs) if self._slots[i] is None]
        joined = []
        while (self._waiting and self._key(self._waiting[0].params) == self._key(params) and
               len(free) >= self._waiting[0].n * self._waiting[0].K):
            req = self._waiting.popleft()
            K = req.K
            slots, free = free[:req.n * K], free[req.n * K:]
            for k, i in enumerate(slots):
                self._slots[i], self._img[i], self._lead[i] = req, k // K, slots[k - k % K]
            joined.append((slots, req))
        return joined

    def _key(self, p: SamplingParams):
        """The parameters every request of the running set shares: _batch_key, or with per_request_sampling max_tokens alone."""
        return (p.max_tokens,) if self.per_request_sampling else _batch_key(p)

    def _sample_slots(self, lead: int) -> List[int]:
        """The slots of the sample whose lead slot is `lead`: itself, then its condition slots."""
        return [lead] + [s for s in range(self.max_num_seqs) if s != lead and self._lead[s] == lead and self._slots[s] is not None]

    def _ensure_state(self, params: SamplingParams):
        m, B = self.model, self.max_num_seqs
        dev = m.tok_embeddings.weight.device
        R = 2 * B if self.cfg_scale > 1.0 else B
        S = int(params.max_tokens)
        if self._state is not None and self._state["S"] == S:
            return self._state
        m.setup_caches(max_batch_size=R, max_seq_length=m.cls_token_num + S, dtype=m.tok_embeddings.weight.dtype)
        self._state = dict(
            S=S, R=R, dev=dev,
            tok=torch.zeros(B, dtype=torch.int32, device=dev),          # label (position 0) or previous token of every slot
            pos=torch.zeros(R, dtype=torch.int32, device=dev),          # per-row positions
            active=torch.zeros(R, dtype=torch.int32, device=dev),       # 1 for rows of occupied slots
            seeds=torch.zeros(B, dtype=torch.int64, device=dev),
            img=torch.zeros(B, dtype=torch.int32, device=dev),          # every slot's image index (lg_sample_rows_keyed)
            img_host=[0] * B,                                           # what st["img"] holds
            out=torch.zeros(B, S, dtype=torch.int32, device=dev),
            logits=torch.empty(R, m.vocab_size, dtype=torch.float32, device=dev),
            join_logits=torch.empty(R // B, m.vocab_size, dtype=torch.float32, device=dev),   # a join's logits (one request's rows)
            join_step=torch.zeros(1, dtype=torch.int32, device=dev),  # a completion request's join draws token P: its step
            # every slot's sampling filters (SampleCfg's row arrays), written by its request's join
            temp=torch.ones(B, dtype=torch.float32, device=dev), topk=torch.zeros(B, dtype=torch.int32, device=dev),
            topp=torch.ones(B, dtype=torch.float32, device=dev), greedy=torch.zeros(B, dtype=torch.int32, device=dev))
        if R == 2 * B:   # every slot's guidance scale and cfg_interval (lg_sample_rows_guided), written by its request's join
            self._state.update(cfg=torch.full((B,), self.cfg_scale, dtype=torch.float32, device=dev),
                               interval=torch.full((B,), -1, dtype=torch.int32, device=dev))
        if self.t2i:
            T, C = m.cls_token_num, m.config.caption_dim
            self._state.update(
                step=torch.zeros(B, dtype=torch.int32, device=dev),       # index of the token every slot samples next
                cond=torch.zeros(B, T, C, dtype=m.tok_embeddings.weight.dtype, device=dev),   # every slot's condition
                mask=torch.zeros(B, T, dtype=torch.float32, device=dev),   # and emb-mask (row r of a decode reads mask row r % B)
                step0=torch.zeros(1, dtype=torch.int32, device=dev),      # the step of token 0, drawn by a join
                # negative prompts: a slot's negative condition and the mask its unconditional row B + s attends with (the slot's own
                # mask without a negative); has_neg: on the host, whether the slot's request brought one
                neg=torch.zeros(B, T, C, dtype=m.tok_embeddings.weight.dtype, device=dev),
                neg_mask=torch.zeros(B, T, dtype=torch.float32, device=dev),
                has_neg=[False] * B)
        if self.sjd_window is not None:
            # the window, this LLM's own per-slot SJD scratch (every slot free) and the host's pass bookkeeping: passes enqueued, and the
            # first pass of every slot's request
            self._state.update(L=min(self.sjd_window, S - 1), passes=0, first_pass=[0] * B, nfin_host=None, events=None, sjd_ws=None,
                               copy_stream=None)
            self._device_sjd_reset(self._state)
        return self._state

    def _filter_values(self, p: SamplingParams) -> tuple:
        """A request's (temperature, top_k, top_p, greedy) as its slots hold them: top_k <= 0 is off (0); t2i: temperature 0 is greedy
        decoding (the argmax of the mixed logits); the c2i path keeps the reference's temperature."""
        return float(p.temperature), min(max(0, int(p.top_k)), 2 ** 31 - 1), float(p.top_p), 1 if self.t2i and p.temperature == 0 else 0

    def _sample_cfg(self, st, params: SamplingParams, slots: slice):
        """The SampleCfg of a draw over `slots`: the row arrays point at their slots' filters (st["temp"], st["topk"], st["topp"],
        st["greedy"]), which the kernel reads in place of the scalars; those stay the running set's."""
        sc = _lib.SampleCfg(self.cfg_scale, -1, *self._filter_values(params), 0)
        sc.temperature_rows, sc.top_k_rows, sc.top_p_rows, sc.greedy_rows = (st[k][slots].data_ptr()
                                                                             for k in ("temp", "topk", "topp", "greedy"))
        return sc

    def _write_guidance(self, st, flat: List[tuple]):
        """The joining requests' seeds, image indices, sampling filters and, under CFG, guidance scales and cfg_intervals, to their slots
        (flat: [(slot, request)]) before their draws. The image indices are written only when one of them changes (a slot at image 0
        that held image 0 writes nothing). Returns the slots as a device index."""
        dev = st["dev"]
        idx = torch.tensor([i for i, _ in flat], dtype=torch.long, device=dev)
        st["seeds"][idx] = torch.tensor([r.seed for _, r in flat], dtype=torch.int64, device=dev)
        f = [self._filter_values(r.params) for _, r in flat]
        for j, (k, dt) in enumerate((("temp", torch.float32), ("topk", torch.int32), ("topp", torch.float32), ("greedy", torch.int32))):
            st[k][idx] = torch.tensor([v[j] for v in f], dtype=dt, device=dev)
        if "cfg" in st:
            st["cfg"][idx] = torch.tensor([r.cfg for _, r in flat], dtype=torch.float32, device=dev)
            st["interval"][idx] = torch.tensor([r.interval for _, r in flat], dtype=torch.int32, device=dev)
        slots = [i for i, _ in flat]
        if any(st["img_host"][i] != self._img[i] for i in slots):
            st["img"][idx] = torch.tensor([self._img[i] for i in slots], dtype=torch.int32, device=dev)
            for i in slots:
                st["img_host"][i] = self._img[i]
        return idx

    def _draw(self, st, params: SamplingParams, logits, slots: slice, step_rows, out, mix=None):
        """One draw for each slot in `slots` from logits (its rows, cond rows first) with the slot's seed at token index step_rows:
        result -> st["tok"][slots] and out[slot, step] (out: st["out"] rows from slots.start). Under CFG each slot mixes with its own
        scale and cfg_interval (lg_sample_rows_guided with st["cfg"], st["interval"]), otherwise lg_sample_rows. When a running slot
        among them holds an image index > 0 (parallel sampling), every slot draws as its image (lg_sample_rows_keyed with st["img"]).
        While a slot among them wants logprobs, the draw is lg_sample_rows_logprobs into st["lp"] ... at the same index as out. While a
        slot among them has given tokens, it is lg_sample_rows_given over st["given"] (a row whose token is given takes it). While a slot
        among them is composed, or for a composed join (mix: its gather table, weights and logits row count), it is
        lg_sample_rows_composed over the gather table st["mix_rows"], st["mix_w"]; a batch draw then hands every lead's token to its
        condition slots' next input (st["lead"]), on the device."""
        lib, m, n = _lib.load(), self.model, slots.stop - slots.start
        use_cfg = 1 if st["R"] == 2 * self.max_num_seqs else 0
        sc = self._sample_cfg(st, params, slots)
        dt = _lib.dtype_code(m.tok_embeddings.weight.dtype)   # 16-bit models round the head's logits to their dtype
        head = (_lib.ptr(logits), n, m.vocab_size, use_cfg, dt, ctypes.byref(sc), _lib.ptr(st["seeds"][slots]), _lib.ptr(step_rows))
        tail = (_lib.ptr(st["tok"][slots]), _lib.ptr(out), st["S"], _lib.current_stream(st["dev"]))
        keyed = any(self._slots[i] is not None and self._img[i] > 0 for i in range(slots.start, slots.stop))
        wants = [self._slots[i].params for i in range(slots.start, slots.stop)
                 if self._slots[i] is not None and _wants_logprobs(self._slots[i].params)]
        if mix is not None or any(self._slots[i] is not None and self._slots[i].weights is not None for i in range(slots.start, slots.stop)):
            rows, weights, nrows = mix if mix is not None else (st["mix_rows"][slots], st["mix_w"][slots], st["R"])
            spec = self._logprob_spec(st, slots.start, any(p.logprobs for p in wants)) if wants else None
            _lib.check(lib.lg_sample_rows_composed(_lib.ptr(logits), nrows, n, m.vocab_size, dt, ctypes.byref(sc), *head[6:],
                                                   _lib.ptr(st["cfg"][slots]), _lib.ptr(st["interval"][slots]),
                                                   _lib.ptr(st["img"][slots]), _lib.ptr(st["given"][slots]) if "given" in st else None,
                                                   _lib.ptr(rows), _lib.ptr(weights), None if spec is None else ctypes.byref(spec), *tail),
                       "lg_sample_rows_composed")
            if mix is None:
                st["tok"].copy_(st["tok"][st["lead"]])
        elif any(self._slots[i] is not None and self._slots[i].given is not None for i in range(slots.start, slots.stop)):
            spec = self._logprob_spec(st, slots.start, any(p.logprobs for p in wants)) if wants else None
            guide = (_lib.ptr(st["cfg"][slots]), _lib.ptr(st["interval"][slots])) if use_cfg else (None, None)
            _lib.check(lib.lg_sample_rows_given(*head, *guide, _lib.ptr(st["img"][slots]) if keyed else None, _lib.ptr(st["given"][slots]),
                                                None if spec is None else ctypes.byref(spec), *tail), "lg_sample_rows_given")
        elif wants:
            spec = self._logprob_spec(st, slots.start, any(p.logprobs for p in wants))
            guide = (_lib.ptr(st["cfg"][slots]), _lib.ptr(st["interval"][slots])) if use_cfg else (None, None)
            _lib.check(lib.lg_sample_rows_logprobs(*head, *guide, _lib.ptr(st["img"][slots]) if keyed else None, ctypes.byref(spec), *tail),
                       "lg_sample_rows_logprobs")
        elif keyed:
            guide = (_lib.ptr(st["cfg"][slots]), _lib.ptr(st["interval"][slots])) if use_cfg else (None, None)
            _lib.check(lib.lg_sample_rows_keyed(*head, *guide, _lib.ptr(st["img"][slots]), *tail), "lg_sample_rows_keyed")
        elif use_cfg:
            _lib.check(lib.lg_sample_rows_guided(*head, _lib.ptr(st["cfg"][slots]), _lib.ptr(st["interval"][slots]), *tail),
                       "lg_sample_rows_guided")
        else:
            _lib.check(lib.lg_sample_rows(*head, *tail), "lg_sample_rows")

    def _logprob_spec(self, st, row: int, top: bool):
        """lg_logprobs over the state's logprob rows from slot `row` on (allocated at the first draw that needs them: [B, S], and
        [B, S, 20] for the alternatives, which a draw asks for whenever a request wants any)."""
        B, S, dev, N = self.max_num_seqs, st["S"], st["dev"], _lib.MAX_TOP_LOGPROBS
        if "lp" not in st:
            st.update(lp=torch.zeros(B, S, dtype=torch.float32, device=dev), rank=torch.zeros(B, S, dtype=torch.int32, device=dev),
                      top_ids=torch.full((B, S, N), -1, dtype=torch.int32, device=dev),
                      top_lp=torch.full((B, S, N), -math.inf, dtype=torch.float32, device=dev))
        return _lib.Logprobs(st["lp"][row].data_ptr(), st["rank"][row].data_ptr(), st["top_ids"][row].data_ptr() if top else 0,
                             st["top_lp"][row].data_ptr() if top else 0, N if top else 0)

    def _host_rows(self, st, done: List[int]):
        """The token rows of the slots in `done` on the host, and for each the logprob rows of its request ((logprob, rank, top ids,
        top logprobs), all [S] / [S, 20]) or None when it did not ask: one device->host copy each."""
        idx = torch.tensor(done, dtype=torch.long, device=st["dev"])
        toks = st["out"][idx].cpu().tolist()
        want = [_wants_logprobs(self._slots[i].params) for i in done]
        lps: List[Optional[tuple]] = [None] * len(done)
        if any(want):
            sel = [j for j, w in enumerate(want) if w]
            rows = [st[k][idx[sel]].cpu().numpy() for k in ("lp", "rank", "top_ids", "top_lp")]
            for n, j in enumerate(sel):
                lps[j] = tuple(r[n] for r in rows)
        return toks, lps

    def _device_decode_t2i(self, st, params: SamplingParams):
        """lg_decode_rows_t2i + a draw (_draw) on every slot: the logits of every row at its own position under its slot's emb-mask, then
        one draw per slot with step st["step"][slot], written to st["out"][slot, step] and, in place, to st["tok"][slot]."""
        B, R, dev = self.max_num_seqs, st["R"], st["dev"]
        lib, handle = _lib.load(), self.model.engine()
        use_cfg = 1 if R == 2 * B else 0
        stream = _lib.current_stream(dev)
        if use_cfg:   # row B + s reads neg_mask[s]: a negative's mask, or the slot's own mask
            _lib.check(lib.lg_decode_rows_t2i_neg(handle, _lib.ptr(st["tok"]), _lib.ptr(st["pos"]), _lib.ptr(st["mask"]), _lib.ptr(st["neg_mask"]),
                                                  B, use_cfg, _lib.ptr(st["logits"]), stream), "lg_decode_rows_t2i_neg")
        else:
            _lib.check(lib.lg_decode_rows_t2i(handle, _lib.ptr(st["tok"]), _lib.ptr(st["pos"]), _lib.ptr(st["mask"]), B, use_cfg,
                                              _lib.ptr(st["logits"]), stream), "lg_decode_rows_t2i")
        self._draw(st, params, st["logits"], slice(0, B), st["step"], st["out"])

    def _device_prefill(self, st, slot: int, P: int, logits):
        """The prefill of a join into slot's cache rows alone, its logits ([2, V] under CFG, else [1, V]) to `logits`: t2i without a
        prefix, lg_prefill_slot of st["cond"][slot], st["mask"][slot]; otherwise lg_prefill_slot_prefix of the slot's condition (c2i: the
        class id in st["tok"][slot]; t2i: st["cond"][slot] and st["mask"][slot]) and the P given tokens in st["out"][slot, :P]. A t2i slot
        with a negative prefills its unconditional row with it and its mask (lg_prefill_slot_prefix_neg)."""
        B, R, dev = self.max_num_seqs, st["R"], st["dev"]
        m = self.model
        lib, handle = _lib.load(), m.engine()
        use_cfg = 1 if R == 2 * B else 0
        stream = _lib.current_stream(dev)
        if self.t2i and P == 0:
            if st["has_neg"][slot]:   # the unconditional row takes the slot's negative and its mask
                ws, ws_bytes = m._slot_prefix_scratch(use_cfg, 0)
                _lib.check(lib.lg_prefill_slot_prefix_neg(handle, _lib.ptr(st["cond"][slot]), _lib.ptr(st["mask"][slot]),
                                                          _lib.ptr(st["neg"][slot]), _lib.ptr(st["neg_mask"][slot]), m.cls_token_num, None, 0,
                                                          slot, B, use_cfg, ws, ws_bytes, _lib.ptr(logits), stream), "lg_prefill_slot_prefix_neg")
            else:
                ws, ws_bytes = m._slot_scratch(use_cfg)
                _lib.check(lib.lg_prefill_slot(handle, _lib.ptr(st["cond"][slot]), _lib.ptr(st["mask"][slot]), m.cls_token_num, slot, B,
                                               use_cfg, ws, ws_bytes, _lib.ptr(logits), stream), "lg_prefill_slot")
            return
        ws, ws_bytes = m._slot_prefix_scratch(use_cfg, P)
        # c2i: the prefill reads the class id from tok[slot] before a draw overwrites it (one stream)
        cond = _lib.ptr(st["cond"][slot]) if self.t2i else _lib.ptr(st["tok"][slot:slot + 1])
        mask = _lib.ptr(st["mask"][slot]) if self.t2i else None
        if self.t2i and st["has_neg"][slot]:
            _lib.check(lib.lg_prefill_slot_prefix_neg(handle, cond, mask, _lib.ptr(st["neg"][slot]), _lib.ptr(st["neg_mask"][slot]),
                                                      m.cls_token_num, _lib.ptr(st["out"][slot]), P, slot, B, use_cfg, ws, ws_bytes,
                                                      _lib.ptr(logits), stream), "lg_prefill_slot_prefix_neg")
        else:
            _lib.check(lib.lg_prefill_slot_prefix(handle, cond, mask, m.cls_token_num, _lib.ptr(st["out"][slot]), P, slot, B, use_cfg, ws,
                                                  ws_bytes, _lib.ptr(logits), stream), "lg_prefill_slot_prefix")

    def _device_join_t2i(self, st, params: SamplingParams, slot: int):
        """lg_prefill_slot of the condition and mask in st["cond"][slot], st["mask"][slot] (_device_prefill), then token 0 drawn from
        its logits (_draw: one image, the slot's seed, guidance, step 0) into st["out"][slot, 0] and st["tok"][slot]."""
        self._device_prefill(st, slot, 0, st["join_logits"])
        self._draw(st, params, st["join_logits"], slice(slot, slot + 1), st["step0"], st["out"][slot])

    def _device_join_prefix(self, st, params: SamplingParams, slot: int, P: int):
        """The join of a completion request with P given tokens, already in st["out"][slot, :P]: lg_prefill_slot_prefix of the slot's
        condition and the prefix (_device_prefill), then token P drawn from its logits (_draw: one image, the slot's seed, guidance,
        step P) into st["out"][slot, P] and st["tok"][slot]."""
        self._device_prefill(st, slot, P, st["join_logits"])
        st["join_step"].fill_(P)
        self._draw(st, params, st["join_logits"], slice(slot, slot + 1), st["join_step"], st["out"][slot])

    def _load_caption(self, st, i: int, r: _Request, c: int = 0):
        """A t2i request's condition c (0: its own; a composed request's c-th caption), its mask and, for c = 0, its negative to slot
        i's device rows (before its join). A condition slot's unconditional row keeps the null condition: it is never read."""
        cond, mask = (r.cond, r.mask) if c == 0 or r.conds is None else r.conds[c]
        neg = r.neg if c == 0 else None
        st["cond"][i].copy_(cond)
        st["mask"][i].copy_(mask)
        st["has_neg"][i] = neg is not None
        if neg is not None:
            st["neg"][i].copy_(neg)
        st["neg_mask"][i].copy_(mask if neg is None else r.neg_mask)

    # ------------------------------------------------------------------ composable guidance (SamplingParams.cond_weights)
    def _write_mix(self, st, joined):
        """The joining requests' rows of the gather table (st["mix_rows"] [B, 9], st["mix_w"] [B, 8]) and of st["lead"] [B], before
        their draws. Allocated, every row plain (-1) and every slot its own lead, when the first composed request joins; from then on
        every join rewrites its slots' rows: a plain slot -1, a condition slot -2, a lead slot [B + lead, its K slots, -1 ...] with the
        request's weights."""
        if "mix_rows" not in st and all(r.weights is None for _, r in joined):
            return
        B, dev, M = self.max_num_seqs, st["dev"], _lib.MAX_COMPOSE
        if "mix_rows" not in st:
            st.update(mix_rows=torch.full((B, 1 + M), -1, dtype=torch.int32, device=dev),
                      mix_w=torch.zeros(B, M, dtype=torch.float32, device=dev),
                      lead=torch.arange(B, dtype=torch.long, device=dev),
                      # a composed join: the [K, 2, V] logits of its K prefills and the gather table of its lead's draw over them
                      join_logits_k=torch.empty(M, 2, self.model.vocab_size, dtype=torch.float32, device=dev),
                      join_rows=torch.full((1, 1 + M), -1, dtype=torch.int32, device=dev),
                      join_w=torch.zeros(1, M, dtype=torch.float32, device=dev))
        idx, rows, ws = [], [], []
        for slots, r in joined:
            for k, s in enumerate(slots):
                row, w = [-1] * (1 + M), [0.0] * M
                if r.weights is not None and k % r.K == 0:
                    row[:1 + r.K] = [B + s] + slots[k:k + r.K]
                    w[:r.K] = r.weights
                elif r.weights is not None:
                    row[0] = -2
                idx.append(s), rows.append(row), ws.append(w)
        i = torch.tensor(idx, dtype=torch.long, device=dev)
        st["mix_rows"][i] = torch.tensor(rows, dtype=torch.int32, device=dev)
        st["mix_w"][i] = torch.tensor(ws, dtype=torch.float32, device=dev)
        st["lead"][i] = torch.tensor([self._lead[s] for s in idx], dtype=torch.long, device=dev)

    def _join_composed(self, st, params: SamplingParams, slots: List[int], r: _Request):
        """The join of a composed request (slots: sample j's condition i in slots[j K + i]). A c2i request without a prefix needs none:
        its K classes enter at position 0 and the step's decode draws token 0. Otherwise sample 0's K slots are prefilled alone
        (_device_prefill) into st["join_logits_k"] [K, 2, V], each condition slot's K / V is copied to the same condition's slot of every
        other sample, and token P of every sample is drawn once from those logits (lg_sample_rows_composed over rows u = 1, c_i = 2 (i - 1),
        with the lead's seed and image index); the lead's token then becomes its condition slots' next input."""
        K, n, P, M = r.K, r.n, _plen(r), _lib.MAX_COMPOSE
        if not self.t2i and P == 0:
            return
        dev, T, buf = st["dev"], self.model.cls_token_num, st["join_logits_k"]
        for i in range(K):
            self._device_prefill(st, slots[i], P, buf[i])
        if n > 1:
            for i in range(K):
                self._device_copy_kv(st, slots[i], [slots[j * K + i] for j in range(1, n)], T + P)
        st["join_rows"][0] = torch.tensor([1] + [2 * i for i in range(K)] + [-1] * (M - K), dtype=torch.int32, device=dev)
        st["join_w"][0] = torch.tensor(list(r.weights) + [0.0] * (M - K), dtype=torch.float32, device=dev)
        st["join_step"].fill_(P)
        for j in range(n):
            lead = slots[j * K]
            self._draw(st, params, buf, slice(lead, lead + 1), st["join_step"], st["out"][lead], mix=(st["join_rows"], st["join_w"], 2 * K))
            if K > 1:
                st["tok"][torch.tensor(slots[j * K + 1:(j + 1) * K], dtype=torch.long, device=dev)] = st["tok"][lead].clone()

    # ------------------------------------------------------------------ inpainting (given=, given_mask=)
    def _load_given(self, st, slots: List[int], r: _Request):
        """A joining request's given tokens to its slots' token rows st["out"] and given rows st["given"] (allocated, all -1, when the
        first request with given tokens joins; from then on every join rewrites its slots' given rows)."""
        if r.given is None and "given" not in st:
            return
        if "given" not in st:
            st["given"] = torch.full((self.max_num_seqs, st["S"]), -1, dtype=torch.int32, device=st["dev"])
        row = torch.full((st["S"],), -1, dtype=torch.int32) if r.given is None else r.given
        row = row.to(st["dev"])
        for s in slots:
            st["given"][s] = row
            if r.given is not None:
                st["out"][s] = row

    def _extends(self) -> List[tuple]:
        """(slot, a, K) of every running slot whose next token starts an interior given run: this step's decode row for it draws the
        given token a (the given select), and its extend follows the decode."""
        return [(i, self._depth[i], r.extends[self._depth[i]]) for i, r in enumerate(self._slots)
                if r is not None and self._depth[i] in r.extends]

    def _device_extend(self, st, params: SamplingParams, slot: int, a: int, K: int):
        """lg_extend_slot over the given run [a, a + K) of slot: tokens a - 1 .. a + K - 1 of st["out"][slot] at positions T + a - 1 ..,
        then token a + K drawn from its logits (_draw: the slot's seed, guidance and image index, step a + K) into st["out"][slot, a + K]
        and st["tok"][slot]."""
        B, m = self.max_num_seqs, self.model
        use_cfg = 1 if st["R"] == 2 * B else 0
        ws, ws_bytes = m._slot_extend_scratch(use_cfg, K)
        mask = _lib.ptr(st["mask"][slot]) if self.t2i else None
        neg_mask = _lib.ptr(st["neg_mask"][slot]) if self.t2i and use_cfg else None
        _lib.check(_lib.load().lg_extend_slot(m.engine(), _lib.ptr(st["out"][slot]), st["S"], a, K, slot, B, use_cfg, mask, neg_mask, ws,
                                              ws_bytes, _lib.ptr(st["join_logits"]), _lib.current_stream(st["dev"])), "lg_extend_slot")
        st["join_step"].fill_(a + K)
        self._draw(st, params, st["join_logits"], slice(slot, slot + 1), st["join_step"], st["out"][slot])

    def _run_extends(self, st, params: SamplingParams, ext: List[tuple]):
        """After a step's decode: every extend of `ext` ((slot, a, K), from _extends before the decode), then the slot's rows sit at
        position T + a + K with token a + K as input, and it has drawn a + K + 1 tokens."""
        B, R, T = self.max_num_seqs, st["R"], self.model.cls_token_num
        for i, a, K in ext:
            self._device_extend(st, params, i, a, K)
            st["pos"][[i, B + i] if R == 2 * B else [i]] = T + a + K
            if self.t2i:
                st["step"][i] = a + K + 1
            self._depth[i] = a + K + 1

    # ------------------------------------------------------------------ parallel sampling (SamplingParams.n)
    def _device_copy_kv(self, st, src: int, dsts: List[int], length: int):
        """lg_copy_slot_kv: positions [0, length) of slot src's K / V rows (and, under CFG, row B + src) to every slot in dsts."""
        B, use_cfg = self.max_num_seqs, 1 if st["R"] == 2 * self.max_num_seqs else 0
        arr = (ctypes.c_int32 * len(dsts))(*dsts)
        _lib.check(_lib.load().lg_copy_slot_kv(self.model.engine(), src, arr, len(dsts), B, use_cfg, length, _lib.current_stream(st["dev"])),
                   "lg_copy_slot_kv")

    def _device_join_draws(self, st, params: SamplingParams, slots: List[int], P: int):
        """Token P of every slot in `slots` drawn from the join's logits (st["join_logits"]) with the slot's seed, guidance and image
        index (_draw at step P) into st["out"][slot, P] and st["tok"][slot]."""
        st["join_step"].fill_(P)
        for i in slots:
            self._draw(st, params, st["join_logits"], slice(i, i + 1), st["join_step"], st["out"][i])

    def _fan_out(self, st, params: SamplingParams, slots: List[int], P: int):
        """After the join of a request with several samples prefilled its first slot: its K / V over [0, T + P) to the other slots, then
        their draws of token P from the same logits."""
        if len(slots) > 1:
            self._device_copy_kv(st, slots[0], slots[1:], self.model.cls_token_num + P)
            self._device_join_draws(st, params, slots[1:], P)

    def _sample_done(self, i: int, toks: List[int], lp: Optional[tuple] = None) -> Optional[_Request]:
        """Free slot i, whose sample finished with tokens toks (and logprob rows lp); returns its request when that was the request's
        last sample."""
        req = self._slots[i]
        for s in self._sample_slots(i)[1:]:   # a composed sample's condition slots leave with it
            self._slots[s], self._lead[s] = None, s
        self._slots[i] = None
        req.done[self._img[i]] = toks
        if lp is not None:
            req.done_lp[self._img[i]] = lp
        return req if len(req.done) == req.n else None

    def _free_rows(self, st, done: List[int]):
        """The slots of the finished samples whose lead slots are `done` (a composed sample's condition slots too) as a device index,
        for their rows to be reset; condition slots become their own leads again in st["lead"]."""
        members = [s for i in done for s in self._sample_slots(i)]
        idx = torch.tensor(members, dtype=torch.long, device=st["dev"])
        if len(members) > len(done):
            conds = torch.tensor([s for s in members if self._lead[s] != s], dtype=torch.long, device=st["dev"])
            st["lead"][conds] = conds
        return idx

    @staticmethod
    def _completions(req: _Request) -> List[CompletionOutput]:
        """The request's outputs: every image in index order, or with best_of the n with the largest cumulative logprob (descending,
        ties: the lower index first). With logprobs, one dict per token: None for a given prefix token, else the drawn token's Logprob
        and the N most likely kept tokens' (rank 1 .. N)."""
        sp, P = req.params, _plen(req)
        if not _wants_logprobs(sp):
            return [CompletionOutput(j, list(req.done[j])) for j in range(req.n)]
        outs = []
        for j in range(req.n):
            lp, rank, top_ids, top_lp = req.done_lp[j]
            toks = list(req.done[j])
            c = CompletionOutput(j, toks, cumulative_logprob=float(np.sum(lp[P:].astype(np.float64))))
            if sp.logprobs is not None:
                N = sp.logprobs
                lps, ranks, ids, tlps = lp.tolist(), rank.tolist(), top_ids[:, :N].tolist(), top_lp[:, :N].tolist()
                c.logprobs = [None] * P
                for k in range(P, len(toks)):
                    d = {toks[k]: Logprob(lps[k], ranks[k])}
                    for r, (t, x) in enumerate(zip(ids[k], tlps[k])):
                        if t >= 0:
                            d.setdefault(t, Logprob(x, r + 1))
                    c.logprobs.append(d)
            outs.append(c)
        if sp.best_of is not None:
            outs = sorted(outs, key=lambda c: (-c.cumulative_logprob, c.index))[:sp.n]
        return outs

    # ------------------------------------------------------------------ speculative Jacobi decoding (sjd_window)
    def _sjd_scratch(self, st):
        """(device pointer, bytes) of this LLM's per-slot SJD scratch: 256-byte aligned in st["sjd_ws"]."""
        buf = st["sjd_ws"]
        base = (buf.data_ptr() + 255) // 256 * 256
        return ctypes.c_void_p(base), buf.numel() - (base - buf.data_ptr())

    def _device_sjd_reset(self, st):
        """A new state's SJD scratch (lg_sjd_slots_workspace_bytes), then lg_sjd_slots_reset: every slot free. The slot state lives
        across steps, so the scratch belongs to this LLM's state, not to the model: another LLM on the same model cannot overwrite it."""
        B, use_cfg = self.max_num_seqs, 1 if st["R"] == 2 * self.max_num_seqs else 0
        lib, handle = _lib.load(), self.model.engine()
        need = ctypes.c_size_t()
        _lib.check(lib.lg_sjd_slots_workspace_bytes(handle, B, use_cfg, st["L"], ctypes.byref(need)), "lg_sjd_slots_workspace_bytes")
        st["sjd_ws"] = torch.empty(need.value + 256, dtype=torch.uint8, device=st["dev"])
        ws, ws_bytes = self._sjd_scratch(st)
        _lib.check(_lib.load().lg_sjd_slots_reset(self.model.engine(), B, use_cfg, st["L"], ws, ws_bytes, _lib.current_stream(st["dev"])),
                   "lg_sjd_slots_reset")

    def _device_sjd_start(self, st, slot: int, req: _Request):
        """lg_sjd_slot_start of slot, after its join drew token 0: the request's seed, guidance and pass counter 0; a sample j > 0 of a
        parallel-sampling request keys as image j (lg_sjd_slot_start_image)."""
        B, use_cfg = self.max_num_seqs, 1 if st["R"] == 2 * self.max_num_seqs else 0
        ws, ws_bytes = self._sjd_scratch(st)
        lib, args = _lib.load(), (self.model.engine(), slot, B, use_cfg, st["L"], st["S"], req.seed, req.cfg, req.interval)
        tail = (_lib.ptr(st["out"]), ws, ws_bytes, _lib.current_stream(st["dev"]))
        if self._img[slot] > 0:
            _lib.check(lib.lg_sjd_slot_start_image(*args, self._img[slot], *tail), "lg_sjd_slot_start_image")
        else:
            _lib.check(lib.lg_sjd_slot_start(*args, *tail), "lg_sjd_slot_start")

    def _device_sjd_pass(self, st, params: SamplingParams, dbg=None):
        """Enqueue pass st["passes"] (lg_sjd_pass_slots) over every slot; its final counts go to a pinned buffer behind an event.
        dbg: None or f32 [B, L, V] on the device, this pass's p rows."""
        B, dev = self.max_num_seqs, st["dev"]
        use_cfg = 1 if st["R"] == 2 * B else 0
        if st["events"] is None:
            st["nfin_host"] = torch.zeros(2, B, dtype=torch.int32).pin_memory()
            st["events"] = [torch.cuda.Event(), torch.cuda.Event()]
        j = st["passes"] & 1
        ws, ws_bytes = self._sjd_scratch(st)
        sc = self._sample_cfg(st, params, slice(0, B))
        mask = _lib.ptr(st["mask"]) if self.t2i else None
        neg_mask = _lib.ptr(st["neg_mask"]) if self.t2i and use_cfg else None
        _lib.check(_lib.load().lg_sjd_pass_slots(self.model.engine(), ctypes.byref(sc), mask, neg_mask, B, use_cfg, st["S"], st["L"], ws,
                                                 ws_bytes, _lib.ptr(st["out"]), _lib.ptr(st["nfin_host"][j]), _lib.ptr(dbg),
                                                 _lib.current_stream(dev)), "lg_sjd_pass_slots")
        st["events"][j].record(torch.cuda.current_stream(dev))

    def _sjd_nfin(self, st, p: int) -> List[int]:
        """Every slot's final count after pass p (the pass before the one last enqueued): waits for that pass only."""
        st["events"][p & 1].synchronize()
        return st["nfin_host"][p & 1].tolist()

    def _sjd_rows(self, st, done: List[int], p: int) -> List[List[int]]:
        """The token rows of the slots in `done`, final after pass p: copied on a side stream behind pass p's event, so that the host
        does not wait for the pass enqueued after it (that pass writes nothing of a frozen slot)."""
        dev = st["dev"]
        if st["copy_stream"] is None:
            st["copy_stream"] = torch.cuda.Stream(dev)
        side = st["copy_stream"]
        side.wait_event(st["events"][p & 1])
        with torch.cuda.stream(side):
            rows = st["out"][torch.tensor(done, dtype=torch.long, device=dev)].cpu().tolist()
        return rows

    def _step_sjd(self, st, params: SamplingParams) -> List[RequestOutput]:
        """step() with sjd_window: (1) admit waiting requests (their join draws token 0, then their slot starts), (2) enqueue one pass
        over every slot, (3) finish the requests whose final count reached max_tokens in the pass before it. The host never waits for
        the pass it just enqueued: a finished slot stays frozen until then, which changes no request's tokens."""
        B, S, dev = self.max_num_seqs, st["S"], st["dev"]
        joined = self._admit(params)
        if joined:
            flat = [(i, r) for slots, r in joined for i in slots]
            idx = self._write_guidance(st, flat)
            for slots, r in joined:
                i = slots[0]
                if self.t2i:
                    for s in slots:
                        self._load_caption(st, s, r)
                    self._device_join_t2i(st, params, i)
                else:   # one row with the class token (lg_prefill_slot_prefix, P = 0), token 0 drawn with step 0
                    st["tok"][i] = r.prompt_token_ids[0]
                    self._device_join_prefix(st, params, i, 0)
                self._fan_out(st, params, slots, 0)
                for s in slots:
                    self._device_sjd_start(st, s, r)
                    st["first_pass"][s] = st["passes"]
        done = []
        if self._running():
            self._device_sjd_pass(st, params)
            p = st["passes"]
            st["passes"] += 1
            self.sjd_passes += 1
            if p > 0:
                nfin = self._sjd_nfin(st, p - 1)
                done = [i for i in range(B) if self._slots[i] is not None and st["first_pass"][i] <= p - 1 and nfin[i] >= S]
                for i in done:
                    self.sjd_request_passes[self._slots[i].request_id] = p - st["first_pass"][i]
                self.sjd_tokens += len(done) * (S - 1)
        self.steps_run += 1
        return self._finish_c2i(st, done, self._sjd_rows(st, done, p - 1) if done else None)

    def _step_t2i(self, st, params: SamplingParams) -> List[RequestOutput]:
        """step() of a t2i LLM: decode the running slots, then admit waiting requests (their prefill draws token 0), then return the
        requests that reached max_tokens."""
        B, R, S, dev = self.max_num_seqs, st["R"], st["S"], st["dev"]
        T = self.model.cls_token_num
        # (1) one decode step for every slot; free slots run too (their rows are never read) so that the row count stays fixed; then the
        # extends of the slots whose decode row drew the first token of a given run
        if self._running():
            ext = self._extends()
            self._device_decode_t2i(st, params)
            st["pos"] += st["active"]
            st["step"] += st["active"][:B]
            for i in range(B):
                if self._slots[i] is not None:
                    self._depth[i] += 1
            self._run_extends(st, params, ext)
        # (2) admission: the conditions and masks go to their slots' rows, then each request is prefilled alone and draws token 0, or,
        # with P given tokens (written to its out row first), token P
        joined = self._admit(params)
        flat = [(i, r) for slots, r in joined for i in slots]
        for i, r in flat:
            self._depth[i] = _plen(r) + 1
        if joined:
            idx = self._write_guidance(st, flat)
            self._write_mix(st, joined)
            for slots, r in joined:
                i = slots[0]
                for k, s in enumerate(slots):
                    self._load_caption(st, s, r, k % r.K)
                self._load_given(st, slots, r)
                if r.prefix is not None:
                    for s in slots:
                        st["out"][s, :_plen(r)] = r.prefix.to(device=dev, dtype=torch.int32)
                if r.weights is not None:   # K prefills of sample 0, their fan-out and one draw per sample
                    self._join_composed(st, params, slots, r)
                    continue
                if r.prefix is None:
                    self._device_join_t2i(st, params, i)
                else:
                    self._device_join_prefix(st, params, i, _plen(r))
                self._fan_out(st, params, slots, _plen(r))
            P = torch.tensor([_plen(r) for _, r in flat], dtype=torch.int32, device=dev)
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["pos"][rows] = T + (torch.cat([P, P]) if R == 2 * B else P)
            st["active"][rows] = 1
            st["step"][idx] = P + 1
        self.steps_run += 1
        # (3) the finished requests (their last drawn token is drawn): the only device->host copy is their token rows
        done = [i for i in range(B) if self._slots[i] is not None and self._lead[i] == i and self._depth[i] >= self._slots[i].end]
        outs: List[RequestOutput] = []
        if done:
            idx = self._free_rows(st, done)
            toks, lps = self._host_rows(st, done)
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["active"][rows] = 0
            st["pos"][rows] = 0
            st["step"][idx] = 0                                # a free slot's draw goes to out[slot, 0], which its next request rewrites
            for i, t, lp in zip(done, toks, lps):
                req = self._sample_done(i, t, lp)
                if req is not None:
                    outs.append(RequestOutput(req.request_id, [], self._completions(req), True))
        return outs

    def _device_step(self, st, params: SamplingParams):
        """lg_decode_rows + a draw (_draw) on the slots' device state: logits of every row at its own position, then one draw per
        slot written to st["out"][slot, depth] and, in place, to st["tok"][slot] (the next step's input)."""
        B, R, dev = self.max_num_seqs, st["R"], st["dev"]
        lib, handle = _lib.load(), self.model.engine()
        use_cfg = 1 if R == 2 * B else 0
        stream = _lib.current_stream(dev)
        _lib.check(lib.lg_decode_rows(handle, _lib.ptr(st["tok"]), _lib.ptr(st["pos"]), B, use_cfg, _lib.ptr(st["logits"]), stream),
                   "lg_decode_rows")
        self._draw(st, params, st["logits"], slice(0, B), st["pos"], st["out"])

    @torch.no_grad()
    def step(self) -> List[RequestOutput]:
        """ONE engine iteration (llm_engine.py:511): admit waiting requests into free slots, decode one token for every running
        sequence (each at its own depth), sample, and return the requests that just finished (with their null-class twins)."""
        if not self.has_unfinished_requests():
            return []
        if self._running() == 0:
            self._params = self._waiting[0].params           # a new running set may change the sampling parameters
        params = self._params
        st = self._ensure_state(params)
        if self.sjd_window is not None:
            return self._step_sjd(st, params)
        if self.t2i:
            return self._step_t2i(st, params)
        B, R, S, dev = self.max_num_seqs, st["R"], st["S"], st["dev"]
        # (1) admission: requests that share the running set's sampling parameters join at position 0, mid-sequence of the others
        joined = self._admit(params)
        flat = [(i, r) for slots, r in joined for i in slots]
        for i, _ in flat:
            self._depth[i] = 0
        if joined:
            idx = self._write_guidance(st, flat)
            self._write_mix(st, joined)
            # every slot's class: a composed request's sample j takes class c_i in its condition i's slot
            st["tok"][idx] = torch.tensor([r.prompt_token_ids[k % r.K] for slots, r in joined for k in range(len(slots))], dtype=torch.int32,
                                          device=dev)
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["pos"][rows] = 0
            st["active"][rows] = 1
            for slots, r in joined:
                self._load_given(st, slots, r)
            # a completion request is prefilled through its P given tokens (written to its out rows first) and draws token P here; its
            # rows then sit at position 1 + P and this step's decode draws token P + 1
            for slots, r in joined:
                if r.prefix is not None:
                    P = _plen(r)
                    for i in slots:
                        st["out"][i, :P] = r.prefix.to(device=dev, dtype=torch.int32)
                    if r.weights is not None:
                        self._join_composed(st, params, slots, r)
                    else:
                        self._device_join_prefix(st, params, slots[0], P)
                        self._fan_out(st, params, slots, P)
                    for i in slots:
                        st["pos"][[i, B + i] if R == 2 * B else [i]] = self.model.cls_token_num + P
                        self._depth[i] = P + 1
        # a request whose join drew its last drawn token (P = max_tokens - 1, or a given tail after P) finishes now, before a decode could
        # write past its out row
        outs = self._finish_c2i(st, [i for i, r in flat if self._lead[i] == i and self._depth[i] >= r.end])
        # (2) one decode step for every slot, (3) per-request sampling; the sampled token becomes the slot's next input in place; then the
        # extends of the slots whose decode row drew the first token of a given run
        ext = []
        if self._running():
            ext = self._extends()
            self._device_step(st, params)
            st["pos"] += st["active"]
            st["tok"] *= st["active"][:B]                    # free slots keep a valid (class 0) input; their rows are never read
            self._run_extends(st, params, ext)
        self.steps_run += 1
        # (4) bookkeeping on the host (no EOS: depths are known without reading the device)
        done = []
        extended = {i for i, _, _ in ext}
        for i in range(B):
            if self._slots[i] is not None:
                if i not in extended:
                    self._depth[i] += 1
                if self._lead[i] == i and self._depth[i] >= self._slots[i].end:
                    done.append(i)
        return outs + self._finish_c2i(st, done)

    def _finish_c2i(self, st, done: List[int], toks: Optional[List[List[int]]] = None) -> List[RequestOutput]:
        """Free the c2i slots in `done` (or, with sjd_window, any slots) and return their requests' outputs (with their null-class
        twins'). toks: their token rows, already on the host, or None (copied here)."""
        B, R, dev = self.max_num_seqs, st["R"], st["dev"]
        outs: List[RequestOutput] = []
        if done:
            idx = self._free_rows(st, done)
            lps = [None] * len(done)
            if toks is None:                                  # the only device->host copy: token (and logprob) rows of finished requests
                toks, lps = self._host_rows(st, done)
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["active"][rows] = 0
            st["pos"][rows] = 0
            st["tok"][idx] = 0                                # a free slot sits at position 0 = the class branch: its input must be a valid
                                                              # class id, not the last sampled token (which indexed past the class table)
            for i, t, lp in zip(done, toks, lps):
                req = self._sample_done(i, t, lp)
                if req is None:
                    continue
                outs.append(RequestOutput(req.request_id, req.prompt_token_ids, self._completions(req), True))
                twin = self._twins.pop(req.request_id, None)
                if twin is not None:
                    outs.append(RequestOutput(twin.request_id, twin.prompt_token_ids, self._completions(req), True))
        return outs

    # ------------------------------------------------------------------ LLM.generate (llm.py:138-266)
    def _prefixes(self, prefixes, n: int, per: List[SamplingParams]) -> List[Optional[torch.Tensor]]:
        """LLM.generate's prefixes, one per request (or None), each checked as add_request checks it."""
        if prefixes is None:
            return [None] * n
        if len(prefixes) != n:
            raise ValueError(f"prefixes holds {len(prefixes)} entries for {n} requests (c2i with CFG: one per conditional prompt)")
        return [self._prefix(p, sp) for p, sp in zip(prefixes, per)]

    def _givens(self, givens, given_masks, n: int, per: List[SamplingParams], pfx) -> List[Optional[torch.Tensor]]:
        """LLM.generate's givens / given_masks, one per request (or None), each pair checked as add_request checks it."""
        if givens is None and given_masks is None:
            return [None] * n
        givens = [None] * n if givens is None else list(givens)
        given_masks = [None] * n if given_masks is None else list(given_masks)
        if len(givens) != n or len(given_masks) != n:
            raise ValueError(f"givens / given_masks hold {len(givens)} / {len(given_masks)} entries for {n} requests (c2i with CFG: one "
                             f"per conditional prompt)")
        return [self._given(g, m, sp, pf) for g, m, sp, pf in zip(givens, given_masks, per, pfx)]

    def generate(self, prompts=None, sampling_params=None, prompt_token_ids: Optional[List[List[int]]] = None,
                 use_tqdm: bool = False, prompt_embeds=None, prefixes=None, negative_prompt_embeds=None,
                 negative_prompts=None, givens=None, given_masks=None) -> List[RequestOutput]:
        """c2i: prompt_token_ids, one [class id] per request (with CFG followed by one [num_classes] twin each). t2i: prompt_embeds, one
        caption's T5 features per request (see add_request). prefixes: None, or one prefix (see add_request) or None per request; under
        c2i CFG one per conditional prompt, which its twin mirrors. negative_prompt_embeds (t2i, cfg_scale > 1): None, or one negative
        caption's features or None per request; negative_prompts: the same as strings (or None), with a text_encoder, encoded in one call
        with prompts. givens, given_masks: None, or one inpainting request's given tokens and mask (see add_request) or None per request;
        under c2i CFG one per conditional prompt, which its twin mirrors. A request whose SamplingParams has cond_weights takes K class
        ids, K captions' features or K caption strings in its entry (see add_request); every string of the call, negatives included, goes
        through one encoder call. Returns the RequestOutputs sorted by request id."""
        if negative_prompts is not None:
            if negative_prompt_embeds is not None:
                raise ValueError("pass negative_prompts or negative_prompt_embeds, not both")
            negative_prompts = [negative_prompts] if isinstance(negative_prompts, str) else list(negative_prompts)
            if not all(t is None or isinstance(t, str) for t in negative_prompts):
                raise ValueError("negative_prompts must hold caption strings or None")
        if prompts is not None or negative_prompts is not None:
            plist = [] if prompts is None else ([prompts] if isinstance(prompts, str) else list(prompts))
            if prompts is not None and prompt_embeds is not None:
                raise ValueError("pass caption strings (prompts) or their features (prompt_embeds), not both")
            nlist = [t for t in (negative_prompts or []) if t is not None]
            # a composed request's entry may be a list of its K captions: every string of the call goes through one encoder call
            sizes = [len(p) if isinstance(p, (list, tuple)) and self._composed(sampling_params, i) else None for i, p in enumerate(plist)]
            flat = [t for p, k in zip(plist, sizes) for t in (p if k is not None else [p])]
            feats = self._encode_prompts(flat + nlist) if prompts is not None or nlist else []
            if prompts is not None:
                it = iter(feats[:len(flat)])
                prompt_embeds = [next(it) if k is None else [next(it) for _ in range(k)] for k in sizes]
            if negative_prompts is not None:
                it = iter(feats[len(flat):])
                negative_prompt_embeds = [None if t is None else next(it) for t in negative_prompts]
        if self.t2i:
            if prompt_token_ids is not None or prompt_embeds is None:
                raise ValueError("a t2i LLM takes prompt_embeds (one caption's T5 features per request), not prompt_token_ids")
            n = len(prompt_embeds)
            if isinstance(sampling_params, list) and len(sampling_params) != n:
                raise ValueError("The lengths of prompts and sampling_params must be the same.")
            if negative_prompt_embeds is not None and len(negative_prompt_embeds) != n:
                raise ValueError(f"negative prompts hold {len(negative_prompt_embeds)} entries for {n} requests")
            per = sampling_params if isinstance(sampling_params, list) else [sampling_params or SamplingParams()] * n
            scales = [self._guidance(p)[0] for p in per]             # every guidance, caption, negative and prefix is checked before any
            captions = [self._captions(f, p) if p.cond_weights is not None else self._caption(f)   # is queued
                        for f, p in zip(prompt_embeds, per)]
            negs = [self._negative(f, s) for f, s in zip(negative_prompt_embeds or [None] * n, scales)]
            pfx = self._prefixes(prefixes, n, per)
            gvs = self._givens(givens, given_masks, n, per, pfx)
            for c, p, pf, ng, gv in zip(captions, per, pfx, negs, gvs):
                if p.cond_weights is not None:   # a composed request's K captions
                    self._enqueue_t2i(c[0], p, pf, ng, conds=c)
                elif gv is not None:
                    self._enqueue_t2i(c, p, pf, ng, gv)
                elif ng is None:
                    self._enqueue_t2i(c, p, pf)
                else:
                    self._enqueue_t2i(c, p, pf, ng)
            outputs = []
            while self.has_unfinished_requests():
                outputs.extend(o for o in self.step() if o.finished)
            return sorted(outputs, key=lambda o: int(o.request_id))
        if prompt_embeds is not None:
            raise ValueError("prompt_embeds apply to text-conditional (t2i) models")
        if negative_prompt_embeds is not None:
            raise ValueError("negative prompts apply to text-conditional (t2i) models")
        if prompt_token_ids is None:
            raise ValueError("Either prompts or prompt_token_ids must be provided.")
        n = len(prompt_token_ids)
        if isinstance(sampling_params, list) and len(sampling_params) != n:
            raise ValueError("The lengths of prompts and sampling_params must be the same.")
        per = sampling_params if isinstance(sampling_params, list) else [sampling_params or SamplingParams()] * n
        for p in per:
            self._guidance(p)
        half = n // 2
        paired = (self.cfg_scale > 1.0 and n % 2 == 0 and n > 0 and
                  all(list(p) == [self.num_classes] for p in prompt_token_ids[half:]) and
                  all(per[i] == per[i + half] for i in range(half)))
        if self.cfg_scale > 1.0 and not paired:
            raise ValueError("cfg_scale > 1 expects the serving protocol of serve/sample_c2i.py:35-37: the conditional prompts "
                             "followed by one [num_classes] prompt each")
        pfx = self._prefixes(prefixes, half if paired else n, per)
        gvs = self._givens(givens, given_masks, half if paired else n, per, pfx)
        for i in range(half if paired else n):   # a composed prompt's K class ids, before any request is queued
            if per[i].cond_weights is not None:
                self._class_ids(prompt_token_ids[i], per[i])
        ids = [self.add_request(prompt_token_ids[i], per[i], prefix=pfx[i]) if gvs[i] is None else
               self.add_request(prompt_token_ids[i], per[i], prefix=pfx[i], given=gvs[i], given_mask=gvs[i] >= 0)
               for i in range(half if paired else n)]
        if paired:
            for i in range(half):
                self.add_request(prompt_token_ids[half + i], per[half + i], twin_of=ids[i])
        outputs: List[RequestOutput] = []
        while self.has_unfinished_requests():
            outputs.extend(o for o in self.step() if o.finished)
        return sorted(outputs, key=lambda o: int(o.request_id))
