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

While requests are in flight the LLM owns the model's KV-cache workspace (a `generate()` call on the same model would reset it)."""
from __future__ import annotations

import itertools
from collections import deque
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import ctypes

import torch

from . import _lib


@dataclass(frozen=True)
class SamplingParams:
    """The vllm.SamplingParams fields the reference sets (serve/sample_c2i.py:47-49). top_k=-1 / 0 disables top-k."""
    temperature: float = 1.0
    top_p: float = 1.0
    top_k: int = -1
    max_tokens: int = 256


@dataclass
class CompletionOutput:
    index: int
    token_ids: List[int]
    finish_reason: str = "length"


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


class LLM:
    def __init__(self, gpt_model, cfg_scale: float = 1.0, num_classes: int = 1000, max_num_seqs: int = 64, seed: Optional[int] = None,
                 kv_cache_dtype: Optional[str] = None):
        """kv_cache_dtype: None keeps the model's KV-cache setting (Transformer.set_kv_cache, scales included); "auto" (the model
        dtype) or "fp8" (e4m3) sets it. Passing the dtype the model already has keeps its scales."""
        if gpt_model.model_type != "c2i":
            raise ValueError("serve.LLM handles class-conditional models (the reference's serve path is c2i only)")
        if kv_cache_dtype is not None and kv_cache_dtype != getattr(gpt_model, "_kv_cache", ("auto", None))[0]:
            gpt_model.set_kv_cache(kv_cache_dtype)
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
        self._params: Optional[SamplingParams] = None  # sampling parameters of the running set
        self._state = None                             # device tensors, allocated for (max_num_seqs, max_tokens)
        self.steps_run = 0

    # ------------------------------------------------------------------ engine-style surface (llm_engine.py)
    def add_request(self, prompt_token_ids: Sequence[int], sampling_params: Optional[SamplingParams] = None, twin_of=None) -> str:
        if len(prompt_token_ids) != 1 or not (0 <= int(prompt_token_ids[0]) <= self.num_classes):
            raise ValueError(f"a c2i prompt is one class id in [0, {self.num_classes}], got {list(prompt_token_ids)}")
        rid = str(next(self.request_counter))
        req = _Request(rid, [int(prompt_token_ids[0])], sampling_params or SamplingParams(), twin_of)
        if twin_of is None:
            self._waiting.append(req)
        else:
            self._twins[twin_of] = req
        return rid

    def _running(self) -> int:
        return sum(r is not None for r in self._slots)

    def has_unfinished_requests(self) -> bool:
        return bool(self._waiting) or self._running() > 0

    def get_num_unfinished_requests(self) -> int:
        return len(self._waiting) + self._running() + len(self._twins)

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
            out=torch.zeros(B, S, dtype=torch.int32, device=dev),
            logits=torch.empty(R, m.vocab_size, dtype=torch.float32, device=dev))
        return self._state

    def _device_step(self, st, params: SamplingParams):
        """lg_decode_rows + lg_sample_rows on the slots' device state: logits of every row at its own position, then one draw per
        slot written to st["out"][slot, depth] and, in place, to st["tok"][slot] (the next step's input)."""
        B, R, S, dev = self.max_num_seqs, st["R"], st["S"], st["dev"]
        lib, handle = _lib.load(), self.model.engine()
        use_cfg = 1 if R == 2 * B else 0
        stream = _lib.current_stream(dev)
        _lib.check(lib.lg_decode_rows(handle, _lib.ptr(st["tok"]), _lib.ptr(st["pos"]), B, use_cfg, _lib.ptr(st["logits"]), stream),
                   "lg_decode_rows")
        sc = _lib.SampleCfg(self.cfg_scale, -1, float(params.temperature), max(0, int(params.top_k)), float(params.top_p), 0, 0)
        dt = _lib.dtype_code(self.model.tok_embeddings.weight.dtype)   # 16-bit models round the head's logits to their dtype
        _lib.check(lib.lg_sample_rows(_lib.ptr(st["logits"]), B, self.model.vocab_size, use_cfg, dt, ctypes.byref(sc),
                                      _lib.ptr(st["seeds"]), _lib.ptr(st["pos"]), _lib.ptr(st["tok"]), _lib.ptr(st["out"]), S, stream),
                   "lg_sample_rows")

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
        B, R, S, dev = self.max_num_seqs, st["R"], st["S"], st["dev"]
        # (1) admission: requests that share the running set's sampling parameters join at position 0, mid-sequence of the others
        joined = []
        for i in range(B):
            if not self._waiting or self._waiting[0].params != params:
                break
            if self._slots[i] is None:
                req = self._waiting.popleft()
                self._slots[i], self._depth[i] = req, 0
                joined.append((i, req))
        if joined:
            idx = torch.tensor([i for i, _ in joined], dtype=torch.long, device=dev)
            st["tok"][idx] = torch.tensor([r.prompt_token_ids[0] for _, r in joined], dtype=torch.int32, device=dev)
            st["seeds"][idx] = torch.tensor([self._seed + int(r.request_id) for _, r in joined], dtype=torch.int64, device=dev)
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["pos"][rows] = 0
            st["active"][rows] = 1
        # (2) one decode step for every slot, (3) per-request sampling; the sampled token becomes the slot's next input in place
        self._device_step(st, params)
        st["pos"] += st["active"]
        st["tok"] *= st["active"][:B]                        # free slots keep a valid (class 0) input; their rows are never read
        self.steps_run += 1
        # (4) bookkeeping on the host (no EOS: depths are known without reading the device)
        done = []
        for i in range(B):
            if self._slots[i] is not None:
                self._depth[i] += 1
                if self._depth[i] >= S:
                    done.append(i)
        outs: List[RequestOutput] = []
        if done:
            idx = torch.tensor(done, dtype=torch.long, device=dev)
            toks = st["out"][idx].cpu().tolist()              # the only device->host copy: token rows of finished requests
            rows = torch.cat([idx, idx + B]) if R == 2 * B else idx
            st["active"][rows] = 0
            st["pos"][rows] = 0
            st["tok"][idx] = 0                                # a free slot sits at position 0 = the class branch: its input must be a valid
                                                              # class id, not the last sampled token (which indexed past the class table)
            for i, t in zip(done, toks):
                req = self._slots[i]
                self._slots[i] = None
                outs.append(RequestOutput(req.request_id, req.prompt_token_ids, [CompletionOutput(0, t)], True))
                twin = self._twins.pop(req.request_id, None)
                if twin is not None:
                    outs.append(RequestOutput(twin.request_id, twin.prompt_token_ids, [CompletionOutput(0, list(t))], True))
        return outs

    # ------------------------------------------------------------------ LLM.generate (llm.py:138-266)
    def generate(self, prompts=None, sampling_params=None, prompt_token_ids: Optional[List[List[int]]] = None,
                 use_tqdm: bool = False) -> List[RequestOutput]:
        if prompts is not None:
            raise ValueError("prompts must be None: the image models have no tokenizer (skip_tokenizer_init=True)")
        if prompt_token_ids is None:
            raise ValueError("Either prompts or prompt_token_ids must be provided.")
        n = len(prompt_token_ids)
        if isinstance(sampling_params, list) and len(sampling_params) != n:
            raise ValueError("The lengths of prompts and sampling_params must be the same.")
        per = sampling_params if isinstance(sampling_params, list) else [sampling_params or SamplingParams()] * n
        half = n // 2
        paired = (self.cfg_scale > 1.0 and n % 2 == 0 and n > 0 and
                  all(list(p) == [self.num_classes] for p in prompt_token_ids[half:]) and
                  all(per[i] == per[i + half] for i in range(half)))
        if self.cfg_scale > 1.0 and not paired:
            raise ValueError("cfg_scale > 1 expects the serving protocol of serve/sample_c2i.py:35-37: the conditional prompts "
                             "followed by one [num_classes] prompt each")
        ids = [self.add_request(prompt_token_ids[i], per[i]) for i in range(half if paired else n)]
        if paired:
            for i in range(half):
                self.add_request(prompt_token_ids[half + i], per[half + i], twin_of=ids[i])
        outputs: List[RequestOutput] = []
        while self.has_unfinished_requests():
            outputs.extend(o for o in self.step() if o.finished)
        return sorted(outputs, key=lambda o: int(o.request_id))
