"""GPU: engine calls on fenced scratch and fenced outputs, once on zeroed and once on poisoned memory: bit-identical, nothing written
outside.

Every device buffer a call is handed sits in a `Fenced` allocation: a 4 KiB front fence, exactly the bytes asked for from a 256-byte
aligned address, then a 64 KiB back fence, the fences holding fixed pseudo-random bytes. That covers the model's scratch
(`Transformer._device_buffer`: the workspace with its KV cache, the score, prefix, given, slot and SJD scratches), the VQ decoder's
scratch, and every CUDA tensor the package makes with torch.empty: the outputs (tokens, log-probabilities, logits, nll, pixels, T5
features), the T5 encoder's scratch and serve.LLM's per-slot SJD scratch. Each call runs twice, each time on a new engine and newly made
buffers: once zeroed, once poisoned by region class (lg_test_scratch_regions): 0xFF in float and 16-bit regions and in outputs (NaN in
fp32, bf16, fp16 and e4m3), the valid but wrong value 1 in int32 / uint64 state, NaN in the KV cache before the engine's first use (its
zero fill must clear it). A kernel that reads a byte nobody wrote, a memset that misses a region that is read, or an output element left
unwritten turns the second run's result into other bits; a write past a buffer changes a fence.

Covered: generate (c2i and t2i with a negative prompt; prefix in several prefill chunks; given with LEAD, EXTEND and TAIL segments;
return_logprobs; sjd_window; cond_weights), lg_prefill + lg_decode_step, the teacher-forced score (one chunk, several chunks; sequences of
11, 123 and 131 positions, which take the CUDA-core, the hd-64 tensor-core prefill and the windowed tensor-core attention, the last two
reading the never-written key rows past the sequence that the score's memset clears) on 2-layer GPT-B-shaped bf16 and fp16 models, a
head-dim-100 model, an fp8 KV cache, fp8 weights and two decode chains (R = 32); serve.LLM with plain, prefix, inpainting, n = 3 and
sjd_window requests; the T5 encoder at B * T not a multiple of 256; the VQ decoder (fp32 and uint8), its encoder, lg_pixels_to_u8 with a
resize to a width not a multiple of 4, and a small VQ decode on the scratch a larger one left behind. Draws are top-k or greedy: top-p
draws are not reproducible run to run (DESIGN §10). Not covered here: the KV rows outside those a slot call writes (lg_prefill_slot,
lg_extend_slot, the SJD slot calls)."""
import ctypes
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V = 4096
S = 12
FRONT, BACK = 4096, 65536
WS, SCORE, PREFIX, SLOT, SLOT_PREFIX, SLOT_EXTEND, GIVEN, SJD, SJD_SLOTS = range(9)
INT = 1
_real_empty = torch.empty


class Fenced:
    """One uint8 allocation: FRONT fence, a 256-byte aligned payload of exactly nbytes, a back fence of at least BACK bytes."""

    def __init__(self, nbytes, fill, int_regions=()):
        self.nbytes = nbytes
        total = FRONT + 256 + nbytes + BACK
        self.buf = _real_empty(total, dtype=torch.uint8, device="cuda")
        self.start = FRONT + (-(self.buf.data_ptr() + FRONT)) % 256
        g = torch.Generator(device="cuda").manual_seed(nbytes % (1 << 31))
        self.front = torch.randint(0, 256, (self.start,), generator=g, dtype=torch.uint8, device="cuda")
        self.back = torch.randint(0, 256, (total - self.start - nbytes,), generator=g, dtype=torch.uint8, device="cuda")
        self.buf[:self.start] = self.front
        self.buf[self.start + nbytes:] = self.back
        pay = self.payload()
        pay.fill_(0 if fill == "zero" else 0xFF)
        if fill != "zero":
            for off, n in int_regions:            # int32 / uint64 state: 1 in every int32
                pay[off:off + n].view(torch.int32).fill_(1)

    def payload(self):
        return self.buf[self.start:self.start + self.nbytes]

    def ptr(self):
        return self.buf.data_ptr() + self.start

    def check(self):
        e = self.start + self.nbytes
        assert torch.equal(self.buf[:self.start], self.front), "front fence written"
        bad = (self.buf[e:] != self.back).nonzero()
        assert bad.numel() == 0, f"back fence written at payload end + {int(bad[0])} (payload {self.nbytes} bytes)"


class Scratch:
    """Routes the model scratch and the package's CUDA torch.empty allocations through Fenced buffers in the current mode, and keeps
    every buffer for the fence check."""

    def __init__(self, monkeypatch):
        import importlib
        gpt, vq_model = (importlib.import_module(f"llamagen_b200.{n}") for n in ("gpt", "vq_model"))
        self.mode, self.all, self.given_chains = "zero", [], 1
        me = self

        def regions(model, layout):
            from llamagen_b200 import _lib
            lib, h, out = _lib.load(), model.engine(), []
            for kind, args, given in layout:
                a = np.asarray(args, np.int64)
                gp = None if given is None else ctypes.c_void_p(given.ctypes.data)
                n = lib.lg_test_scratch_regions(h, kind, ctypes.c_void_p(a.ctypes.data), len(a), gp, None, 0)
                assert n > 0, lib.lg_last_error()
                r = np.zeros((n, 4), np.int64)
                lib.lg_test_scratch_regions(h, kind, ctypes.c_void_p(a.ctypes.data), len(a), gp, ctypes.c_void_p(r.ctypes.data), n)
                out += [(int(o), int(b)) for o, b, c, _ in r if c == INT and b > 0]
            return out

        def fenced(nbytes, int_regions=()):
            f = Fenced(nbytes, me.mode, int_regions)
            me.all.append(f)
            return f

        def device_buffer(self, attr, nbytes, grow=False):
            store = self.__dict__.setdefault("_fenced", {})
            f = store.get(attr)
            if grow or f is None or f.nbytes < nbytes:
                layout = self.__dict__.pop("_fence_layout", {}).get(attr, [])
                store[attr] = None
                f = store[attr] = fenced(nbytes, regions(self, layout))
                setattr(self, attr, f.buf)
            return ctypes.c_void_p(f.ptr()), f.nbytes

        def stash(name, make):
            orig = getattr(gpt.Transformer, name)

            def wrapped(self, *a, **kw):
                self.__dict__.setdefault("_fence_layout", {}).update(make(self, *a, **kw))
                return orig(self, *a, **kw)
            monkeypatch.setattr(gpt.Transformer, name, wrapped)

        def given_layout(self, given, T, use_cfg):
            g = np.ascontiguousarray(given, np.int32)          # the windows of the chain count the call runs
            return {"_given_ws": [(GIVEN, [g.shape[0], g.shape[1], int(use_cfg), me.given_chains], g)]}

        monkeypatch.setattr(gpt.Transformer, "_device_buffer", device_buffer)
        stash("setup_caches", lambda self, max_batch_size, max_seq_length, dtype=None:
              {"_workspace": [(WS, [max_batch_size, gpt.find_multiple(max_seq_length, 8)], None)]})
        stash("_given_scratch", given_layout)
        stash("_slot_extend_scratch", lambda self, use_cfg, K: {"_slot_extend_ws": [(SLOT_EXTEND, [int(use_cfg), K], None)]})
        stash("_sjd_scratch", lambda self, B, use_cfg, L: {"_sjd_ws": [(SJD, [B, int(use_cfg), L], None)]})

        def vq_workspace(self, h, B, g, dev):
            from llamagen_b200 import _lib
            need = ctypes.c_size_t()
            _lib.check(_lib.load().lg_vq_workspace_bytes(h, B, g, ctypes.byref(need)), "lg_vq_workspace_bytes")
            f = self.__dict__.get("_fenced_ws")
            if f is None or f.nbytes < need.value:
                f = self.__dict__["_fenced_ws"] = fenced(need.value)
            return f.ptr(), need.value
        monkeypatch.setattr(vq_model.VQModel, "_workspace", vq_workspace)

        def empty(*size, dtype=None, device=None, **kw):
            shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else tuple(size)
            dtype = dtype or torch.get_default_dtype()
            n = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size() if shape else 0
            if device is None or torch.device(device).type != "cuda" or kw or n == 0:
                return _real_empty(*size, dtype=dtype, device=device, **kw)
            return fenced(n).payload().view(dtype).view(shape)
        proxy = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
        proxy.empty = empty
        for name in ("gpt", "generate", "serve", "t5", "vq_model", "postprocess"):
            monkeypatch.setattr(importlib.import_module(f"llamagen_b200.{name}"), "torch", proxy)

    def fresh(self, m):
        """A new engine and no scratch: the next call makes (and poisons) every buffer again."""
        if hasattr(m, "_drop_engine"):
            m._drop_engine()
            m._workspace, m._ws_shape = None, (0, 0)
        for attr in ("_fenced", "_fenced_ws", "_fence_layout"):
            m.__dict__.pop(attr, None)
        if "_ws" in m.__dict__:
            m._ws = None

    def run(self, mode, models, call):
        self.mode = mode
        for m in models:
            self.fresh(m)
        self.all = []
        out = _flat(call())
        torch.cuda.synchronize()
        for f in self.all:
            f.check()
        return out

    def twice(self, models, *calls):
        """Each call on new zeroed, then on new poisoned buffers: bit-identical results and intact fences."""
        for i, call in enumerate(calls):
            _same(self.run("zero", models, call), self.run("poison", models, call), f"call {i}")


def _same(xs, ys, what):
    assert len(xs) == len(ys)
    for a, b in zip(xs, ys):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b)), f"{what}: poisoned memory changed a result"


def _flat(x):
    if isinstance(x, torch.Tensor):
        return [x.detach().cpu().clone()]
    if isinstance(x, dict):
        return [t for k in sorted(x) for t in _flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _flat(v)]
    if x is None:
        return []
    return [torch.tensor(np.asarray(x, dtype=np.float64))]


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) if t.element_size() == 2 else t


@pytest.fixture
def scratch(monkeypatch):
    return Scratch(monkeypatch)


def _model(dtype=torch.bfloat16, kv="auto", weights="auto", dim=768, n_head=12, **kw):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(11)
    m = Transformer(ModelArgs(n_layer=2, n_head=n_head, dim=dim, block_size=256, vocab_size=V, **kw))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dtype).eval()
    m.set_kv_cache(kv)
    m.set_weight_dtype(weights)
    return m


T2I = dict(model_type="t2i", cls_token_num=16, caption_dim=256)
VARIANTS = {
    "bf16": dict(),
    "fp16": dict(dtype=torch.float16),
    "hd100": dict(dim=1600, n_head=16),
    "kv-fp8": dict(kv="fp8"),
    "w-fp8": dict(weights="fp8"),
}


def _given(B):
    g = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(5))
    mask = torch.zeros(B, S, dtype=torch.bool)
    mask[:, :3] = True        # LEAD
    mask[:, 6:8] = True       # EXTEND
    mask[:, -2:] = True       # TAIL
    return g, mask


def _score_cases(m, B, T, cond, gen, emb_masks=None):
    """Score calls over sequences of T + L - 1 positions for L in 11, 123 - T + 1 and 131 - T + 1 (lengths not a multiple of 8; 123
    and 131 take the tensor-core attentions, which read the never-written key rows past the sequence)."""
    calls = []
    for seq in (T + 10, 123, 131):
        L = seq - T + 1
        idx = torch.randint(0, V, (B, L - 1), generator=gen).cuda()
        tgt = torch.randint(0, V, (B, L), generator=gen).cuda()
        calls.append(lambda idx=idx, tgt=tgt: m(idx, cond, targets=tgt, emb_masks=emb_masks))
    return calls


@pytest.mark.parametrize("name", list(VARIANTS))
def test_c2i_generate_and_score_paths(scratch, monkeypatch, name):
    from llamagen_b200 import generate, gpt
    m = _model(**VARIANTS[name])
    B = 3
    cond = torch.tensor([1, 7, 42], device="cuda")
    kw = dict(cfg_scale=4.0, top_k=50, seed=9)
    g, mask = _given(B)
    prefix = g[:, :4].cuda()
    monkeypatch.setattr(gpt, "PREFIX_SCRATCH_CAP", 1)      # one image per prefill chunk
    gen = torch.Generator().manual_seed(3)
    idx = torch.randint(0, V, (B, 10), generator=gen).cuda()
    tgt = torch.randint(0, V, (B, 11), generator=gen).cuda()

    def prefill_decode():
        m.setup_caches(max_batch_size=2 * B, max_seq_length=16)
        rows = torch.cat([cond, torch.full_like(cond, 1000)])
        l0, _ = m(None, rows)
        l1, _ = m(l0.argmax(-1).reshape(-1, 1), None, input_pos=torch.tensor([1]))
        return l0, l1

    def several_chunks():
        monkeypatch.setattr(gpt, "SCORE_SCRATCH_CAP", 1)  # one image per chunk
        try:
            return m(idx, cond, targets=tgt)
        finally:
            monkeypatch.setattr(gpt, "SCORE_SCRATCH_CAP", 4 << 30)

    scratch.twice([m],
                  lambda: generate(m, cond, S, **kw),
                  lambda: generate(m, cond, S, prefix=prefix, **kw),
                  lambda: generate(m, cond, S, given=g.cuda(), given_mask=mask.cuda(), **kw),
                  lambda: generate(m, cond, S, return_logprobs=True, top_logprobs=3, **kw),
                  lambda: generate(m, cond, S, sjd_window=4, **kw),
                  lambda: generate(m, cond, S, cfg_scale=4.0, top_k=1, seed=2, sjd_window=16),
                  lambda: generate(m, torch.tensor([[1, 7], [42, 3], [5, 9]], device="cuda"), S, cond_weights=[2.5, 1.5], top_k=50,
                                   seed=9),
                  prefill_decode, several_chunks, *_score_cases(m, B, 1, cond, gen))


def test_t2i_negative_prompt_paths(scratch, monkeypatch):
    from llamagen_b200 import generate, gpt
    m = _model(**T2I)
    B, T, C = 2, T2I["cls_token_num"], T2I["caption_dim"]
    gen = torch.Generator().manual_seed(8)
    cond = torch.randn(B, T, C, generator=gen).to("cuda", torch.bfloat16)
    neg = torch.randn(1, T, C, generator=gen).to("cuda", torch.bfloat16)
    em = torch.ones(B, T, device="cuda")
    em[0, :5] = 0
    em[1, :11] = 0
    nem = torch.ones(1, T, device="cuda")
    nem[0, :9] = 0
    kw = dict(emb_masks=em, cfg_scale=4.0, top_k=50, seed=4, negative_cond=neg, negative_emb_masks=nem)
    g, mask = _given(B)
    monkeypatch.setattr(gpt, "PREFIX_SCRATCH_CAP", 1)
    scratch.twice([m],
                  lambda: generate(m, cond, S, **kw),
                  lambda: generate(m, cond, S, prefix=g[:, :3].cuda(), **kw),
                  lambda: generate(m, cond, S, given=g.cuda(), given_mask=mask.cuda(), **kw),
                  lambda: generate(m, cond, S, sjd_window=4, **kw),
                  lambda: generate(m, cond, S, return_logprobs=True, **kw),
                  *_score_cases(m, B, T, cond, gen, em))


def test_two_decode_chains(scratch, monkeypatch):
    from llamagen_b200 import _lib, generate, gpt
    monkeypatch.setenv("LG_SPLIT", "2")
    m = _model()
    B = 16                                                              # R = 32 rows under CFG: two chains of 16
    cond = torch.arange(B, device="cuda") * 37 % 1000
    g, mask = _given(B)
    monkeypatch.setattr(gpt, "PREFIX_SCRATCH_CAP", 1)
    scratch.given_chains = 2

    def prefix():
        out = generate(m, cond, S, cfg_scale=4.0, top_k=50, seed=1, prefix=g[:, :2].cuda())
        chains = ctypes.c_int(0)
        _lib.load().lg_test_prefix_chunks(m.engine(), ctypes.byref(chains))
        assert chains.value == 2
        return out

    scratch.twice([m],
                  lambda: generate(m, cond, S, cfg_scale=4.0, top_k=50, seed=1),
                  prefix,
                  lambda: generate(m, cond, S, cfg_scale=4.0, top_k=50, seed=1, given=g.cuda(), given_mask=mask.cuda()))


def test_serve_requests(scratch):
    from llamagen_b200 import serve
    m = _model()
    g, mask = _given(2)

    def run(sjd):
        llm = serve.LLM(m, cfg_scale=4.0, max_num_seqs=4, seed=3, sjd_window=sjd)
        sp = serve.SamplingParams(top_k=50, max_tokens=S)
        llm.add_request([5], sp)
        llm.add_request([9], sp)
        if sjd is None:                                                 # prefix and given requests do not take sjd_window
            llm.add_request([10], sp, prefix=g[0, :4].tolist())
            llm.add_request([11], sp, given=g[1], given_mask=mask[1])
            llm.add_request([13], serve.SamplingParams(top_k=50, max_tokens=S, n=3))
        res = []
        while llm.has_unfinished_requests():
            res += llm.step()
        return torch.tensor([t for _, outs in sorted((o.request_id, [c.token_ids for c in o.outputs]) for o in res)
                             for c in outs for t in c])
    scratch.twice([m], lambda: run(None), lambda: run(4))


def test_t5_encode(scratch):
    from llamagen_b200.t5 import T5Config, T5Encoder
    torch.manual_seed(2)
    enc = T5Encoder(T5Config(num_layers=2, d_model=128, d_kv=64, num_heads=2, d_ff=256, vocab_size=512))
    for k, p in enc.state_dict().items():
        p.copy_(1.0 + 0.1 * torch.randn_like(p) if k.endswith("layer_norm.weight") else 0.1 * torch.randn_like(p))
    enc = enc.to("cuda", torch.bfloat16)
    B, T = 3, 37                                                        # B * T = 111 rows: padding rows in the last 256-row chunk
    ids = torch.randint(0, 512, (B, T), generator=torch.Generator().manual_seed(1))
    mask = torch.ones(B, T, dtype=torch.long)
    mask[1, 20:] = 0
    mask[2, 1:] = 0
    scratch.twice([enc], lambda: enc.encode(ids, mask), lambda: enc.encode(ids[:1, :5], mask[:1, :5]))


def test_vq_paths_and_stale_scratch(scratch):
    from llamagen_b200 import VQ_models
    from llamagen_b200.postprocess import to_uint8_nhwc
    torch.manual_seed(0)
    vq = VQ_models["VQ-16"](codebook_size=1024, codebook_embed_dim=8).cuda().eval()
    codes = torch.randint(0, 1024, (4, 64), device="cuda")
    img = torch.rand(2, 3, 64, 64, device="cuda") * 2 - 1
    scratch.twice([vq],
                  lambda: vq.decode_code(codes, [4, 8, 8, 8]),
                  lambda: vq.decode_code_uint8(codes[:3], [3, 8, 8, 8]),
                  lambda: vq.encode(img, return_z=True),
                  lambda: to_uint8_nhwc(img, size=(37, 45)))
    # a small decode on the scratch a larger decode left behind equals the same decode on new poisoned scratch
    small = scratch.run("poison", [vq], lambda: vq.decode_code(codes[1:2], [1, 8, 8, 8]))
    stale = scratch.run("poison", [vq], lambda: (vq.decode_code(codes, [4, 8, 8, 8]), vq.decode_code(codes[1:2], [1, 8, 8, 8]))[1])
    _same(small, stale, "small decode after a large one")
