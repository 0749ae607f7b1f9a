"""GPU: the T5 encoder on the engine.

* t5_attn_tc_kernel (bf16) and t5_attn_kernel (fp32) one call at a time through lg_test_t5_attention against a float64 softmax of
  the operands as the kernel reads them, for T from 1 to 512: captions of valid length 1, T, T / 2 + 1 and one with holes, poison
  keys behind the mask with the highest scores and huge values, and a fully masked caption whose output must stay finite.
* Needles: one head per relative-distance pair (7/8, 11/12, 15/16, 31/32, 63/64, 127/128, 128/129, both directions) whose only
  non-zero values sit at those two distances from one query, with the two buckets' biases +8 and -8, so a wrong bucket on either side
  of the boundary moves that query's output by a large fraction of its own bound scale.
* The gated-GELU epilogue (lg_test_linear epi 6) bit-equal (>= 99.9 %, else one ulp) to an fp32 restatement on the kernel's own
  split-K sum in bf16; within a few fp32 ulps in fp32.
* Weights written in place (load_state_dict) are what the next encode uses.
* The whole encoder against transformers (tests/golden/t5_tiny.pt), and at flan-t5-xl shape (random weights) against the oracle.
* Batch independence: a caption's features are bit-identical across B and under permutations of the batch.
* serve.LLM(text_encoder=...).generate(prompts=...) gives the tokens of generate(prompt_embeds=<the encoder's features>).
* python -m llamagen_b200.sample.extract_t5_feature on a saved random-weight T5 directory with a sentencepiece tokenizer trained in
  the test, in both modes; the feature-file writer with a stub tokenizer."""
import ctypes
import math

import numpy as np
import pytest
import torch

from llamagen_b200 import _lib
from llamagen_b200.t5 import T5Config, T5Encoder, bucket_table
from oracle.t5_oracle import t5_encoder_oracle
from util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
TDT = {"bf16": torch.bfloat16, "f32": torch.float32}
CODE = {"bf16": _lib.LG_DTYPE_BF16, "f32": _lib.LG_DTYPE_F32}


# ------------------------------------------------------------------------------------------------ attention, one call at a time
def _attn_case(T, H, seed, dt):
    g = torch.Generator().manual_seed(seed)
    B, I = 5, H * 64
    q = 0.05 * torch.randn(B, T, H, 64, generator=g)
    k = torch.randn(B, T, H, 64, generator=g)
    v = torch.randn(B, T, H, 64, generator=g)
    lens = [1, T, max(1, T // 2 + 1), T, 0]                              # caption 4: no valid key at all (finite output only)
    mask = torch.zeros(B, T, dtype=torch.int32)
    for b, n in enumerate(lens):
        mask[b, :n] = 1
    mask[3] = (torch.rand(T, generator=g) < 0.7).to(torch.int32)     # holes anywhere
    mask[3, 0] = 1
    # poison: every masked key would win the softmax by far and carries huge values
    poison = mask == 0
    k[poison] = 40.0 * q.mean(dim=(1,))[:, None].expand(B, T, H, 64)[poison].sign()
    v[poison] = 1e3
    bias = 4.0 * torch.randn(32, H, generator=g)
    qkv = torch.stack([q, k, v], dim=2).reshape(B * T, 3 * I).to(TDT[dt])
    return qkv, mask, bias.to(TDT[dt]), bucket_table(T)


def _attn_ref(qkv, mask, bias, buckets, B, T, H):
    x = qkv.double().reshape(B, T, 3, H, 64)
    q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)   # [B, H, T, 64]
    i = torch.arange(T)
    rel = buckets.long()[(i[None, :] - i[:, None]) + T - 1]                                          # [T, T]
    s = q @ k.transpose(-1, -2) + bias.double()[rel].permute(2, 0, 1)[None]
    s = s.masked_fill(mask[:, None, None, :] == 0, -math.inf)
    p = torch.softmax(s, dim=-1)
    o = p @ v
    pabs = p @ v.abs()
    kv = k.abs() * (mask[:, None, :, None] != 0)                                                    # valid keys only
    sabs = (q.abs() @ kv.transpose(-1, -2)).amax(dim=-1, keepdim=True)
    return o.transpose(1, 2).reshape(B * T, H * 64), pabs.transpose(1, 2).reshape(B * T, H * 64), \
        sabs.expand(B, H, T, 64).transpose(1, 2).reshape(B * T, H * 64)


@pytest.mark.parametrize("dt", ["bf16", "f32"])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 120, 128, 129, 257, 512])
def test_attention_against_float64(dt, T):
    H, B = 2, 5
    qkv, mask, bias, buckets = _attn_case(T, H, 100 + T, dt)
    _check_attention(dt, B, T, H, qkv, mask, bias, buckets)


NEEDLES = [(7, 8), (11, 12), (15, 16), (31, 32), (63, 64), (127, 128), (128, 129)]


@pytest.mark.parametrize("dt", ["bf16", "f32"])
@pytest.mark.parametrize("T", [260, 512])
def test_attention_needles_at_bucket_boundaries(dt, T):
    """Head c holds one (d_lo, d_hi, direction) case: query i0 = T // 2, keys i0 + s * d_lo and i0 + s * d_hi carry the head's only
    non-zero values, the bucket of s * d_lo has bias +8 and that of s * d_hi -8 (0 elsewhere; where both distances share a bucket it is
    +8). A bucket misplaced on either side of the boundary changes the needles' weights by e^16 and query i0's output by O(|v|)."""
    cases = [(lo, hi, sgn) for lo, hi in NEEDLES for sgn in (1, -1)]
    H, B, i0 = len(cases), 1, T // 2
    g = torch.Generator().manual_seed(T)
    q = 0.05 * torch.randn(B, T, H, 64, generator=g)
    k = 0.05 * torch.randn(B, T, H, 64, generator=g)
    v = torch.zeros(B, T, H, 64)
    buckets = bucket_table(T)
    bias = torch.zeros(32, H)
    for c, (lo, hi, sgn) in enumerate(cases):
        blo, bhi = int(buckets[sgn * lo + T - 1]), int(buckets[sgn * hi + T - 1])
        bias[bhi, c] = -8.0
        bias[blo, c] = 8.0
        v[0, i0 + sgn * lo, c] = torch.randn(64, generator=g)
        v[0, i0 + sgn * hi, c] = torch.randn(64, generator=g)
    mask = torch.ones(B, T, dtype=torch.int32)
    qkv = torch.stack([q, k, v], dim=2).reshape(B * T, 3 * H * 64).to(TDT[dt])
    got = _check_attention(dt, B, T, H, qkv, mask, bias.to(TDT[dt]), buckets)
    # the checks above hold row i0 to the float64 reference; a misplaced boundary would move it by this much
    ref, _, _ = _attn_ref(qkv, mask, bias.to(TDT[dt]), buckets, B, T, H)
    row = ref[i0].reshape(H, 64)
    assert (row.abs().amax(dim=1) > 1e-3).all(), row.abs().amax(dim=1)
    assert got.shape == ref.shape


def _check_attention(dt, B, T, H, qkv, mask, bias, buckets):
    lib = _lib.load()
    out = torch.full((B * T, H * 64), float("nan"), dtype=TDT[dt], device=DEV)
    path = ctypes.c_int(-1)
    dq, dm, db, dw = qkv.to(DEV), mask.to(DEV), buckets.to(DEV), bias.to(DEV)   # alive until the kernel has run
    _lib.check(lib.lg_test_t5_attention(CODE[dt], B, T, H, _lib.ptr(dq), _lib.ptr(dm), _lib.ptr(db), _lib.ptr(dw), 32, _lib.ptr(out),
                                        ctypes.byref(path), None), "lg_test_t5_attention")
    torch.cuda.synchronize()
    assert path.value == (1 if dt == "bf16" else 0)
    got = out.double().cpu()
    assert torch.isfinite(got).all()
    ref, pabs, sabs = _attn_ref(qkv, mask, bias, buckets, B, T, H)
    rows = (mask.sum(dim=1) > 0).repeat_interleave(T)
    # fp32 scores (64 products) shift every weight by at most exp(64 * 2^-23 * sum|q||k|) - 1, the fp32 sums over T keys add
    # T * 2^-24 relative each; bf16 rounds every P (2^-9 relative, numerator and denominator) and the output (2^-9 of |o|)
    e_s = 64 * 2.0 ** -23 * sabs + T * 2.0 ** -23 + 2.0 ** -20
    if dt == "bf16":
        E = (2 * 2.0 ** -9 + 2 * e_s) * pabs + 2.0 ** -9 * ref.abs() + 1e-6
    else:
        E = 2 * e_s * pabs + 1e-6
    err = (got - ref).abs()
    bad = (err > E) & rows[:, None]
    assert not bad.any(), (T, dt, err[rows].max().item(), (err / E)[rows].max().item())
    return got


# ------------------------------------------------------------------------------------------------ gated-GELU epilogue
@pytest.mark.parametrize("dt, M, N, K", [("bf16", 64, 384, 128), ("bf16", 300, 5120, 2048), ("bf16", 5, 1024, 256), ("f32", 40, 384, 256)])
def test_gelu_mul_epilogue_bit_exact(dt, M, N, K):
    lib = _lib.load()
    g = torch.Generator().manual_seed(M + N)
    t = TDT[dt]
    x = torch.randn(M, K, generator=g).to(t).to(DEV)
    wa = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(t).to(DEV)
    wb = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(t).to(DEV)
    out = torch.empty(M, N, dtype=t, device=DEV)
    acc = torch.empty(M, 2 * N, dtype=torch.float32, device=DEV)
    scratch = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    path = (ctypes.c_int * 4)()
    _lib.check(lib.lg_test_linear(CODE[dt], M, N, K, _lib.ptr(x), None, 1e-6, _lib.ptr(wa), _lib.ptr(wb), 6, None, None, _lib.ptr(out),
                                  None, _lib.ptr(acc), 0, _lib.ptr(scratch), scratch.numel(), path, None), "lg_test_linear")
    torch.cuda.synchronize()
    a, b = acc[:, :N].to(t).float(), acc[:, N:].to(t).float()
    gl = (0.5 * a * (1.0 + torch.tanh(0.7978845608028654 * (a + 0.044715 * a * a * a)))).to(t).float()
    want = (gl * b).to(t)
    if t == torch.bfloat16:
        same = (out == want).float().mean().item()
        assert same >= 0.999, same
        ulp = (out.view(torch.int16).int() - want.view(torch.int16).int()).abs().max().item()
        assert ulp <= 1, ulp
    else:
        # fp32 keeps the last bits that the kernel's contracted multiply-adds and tanhf change against torch's separate roundings
        # (amplified by the cancellation in 1 + tanh for negative inputs): held to a few fp32 ulps of the operands' scale
        err = (out - want).abs()
        assert (err <= 2.0 ** -20 * (a.abs() + 1) * b.abs()).all(), err.max().item()
    ref64 = x.double() @ torch.cat([wa, wb]).double().t()
    assert (acc.double() - ref64).abs().max().item() <= 1e-2 * ref64.abs().max().item() + 1e-3


# ------------------------------------------------------------------------------------------------ whole encoder
OCFG = dict(num_layers=2, num_heads=2, d_kv=64, num_buckets=32, max_distance=128, eps=1e-6)
TINY = dict(num_layers=2, d_model=128, d_kv=64, num_heads=2, d_ff=384, vocab_size=256)


def _encoder(cfg: dict, sd, dtype, max_length=120, tokenizer=None):
    enc = T5Encoder(T5Config(**cfg), max_length=max_length, tokenizer=tokenizer)
    enc.load_state_dict(sd)
    return enc.to(device=DEV, dtype=dtype).eval()


def test_encoder_against_transformers_golden():
    gd = load_golden("t5_tiny.pt")
    ids, mask = gd["ids"].to(DEV), gd["mask"].to(DEV)
    e32 = _encoder(TINY, gd["state_dict"], torch.float32).encode(ids, mask).cpu()
    err32 = (e32 - gd["hidden_fp32"]).abs().max().item()
    assert err32 <= 1e-4, err32
    e16 = _encoder(TINY, gd["state_dict"], torch.bfloat16).encode(ids, mask).float().cpu()
    spread = (gd["hidden_bf16"].float() - gd["hidden_fp32"]).abs()
    err = (e16 - gd["hidden_fp32"]).abs()
    print(f"[t5 golden] fp32 max {err32:.2e}; bf16 max {err.max():.4f} mean {err.mean():.5f}, "
          f"transformers bf16 spread max {spread.max():.4f} mean {spread.mean():.5f}")
    assert err.max() <= 1.5 * spread.max() + 0.02 and err.mean() <= 1.5 * spread.mean() + 1e-3


FLAN = dict(d_model=2048, d_kv=64, num_heads=32, d_ff=5120, vocab_size=32128)


def _random_sd(cfg, seed):
    enc = T5Encoder(T5Config(**cfg))
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in enc.state_dict().items():
        r = torch.randn(v.shape, generator=g)
        if k.endswith("layer_norm.weight"):
            sd[k] = 1.0 + 0.1 * r
        elif "relative_attention_bias" in k or k == "shared.weight":
            sd[k] = r
        else:
            sd[k] = r / math.sqrt(v.shape[1])
    return sd


def _ids(B, T, V, seed, lens=None):
    g = torch.Generator().manual_seed(seed)
    lens = lens or torch.randint(1, T + 1, (B,), generator=g).tolist()
    mask = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None]).to(torch.int64)
    return torch.randint(0, V, (B, T), generator=g) * mask, mask


@pytest.mark.parametrize("layers, B", [(2, 8), (24, 2)])
def test_flan_t5_xl_shape_bf16_against_fp32_oracle(layers, B):
    cfg = dict(FLAN, num_layers=layers)
    sd = {k: v.to(torch.bfloat16) for k, v in _random_sd(cfg, 7).items()}     # the bf16-rounded weights both sides use
    T = 120
    ids, mask = _ids(B, T, cfg["vocab_size"], 3, lens=[T, 1] + [17 * (i + 1) for i in range(B - 2)])
    enc = _encoder(cfg, sd, torch.bfloat16)
    got = enc.encode(ids.to(DEV), mask.to(DEV)).float()
    ocfg = dict(num_layers=layers, num_heads=32, d_kv=64, num_buckets=32, max_distance=128, eps=1e-6)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = t5_encoder_oracle(sdd, ocfg, ids.to(DEV), mask.to(DEV), torch.float32)
        o16 = t5_encoder_oracle(sdd, ocfg, ids.to(DEV), mask.to(DEV), torch.bfloat16).float()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    spread, err = (o16 - ref).abs(), (got - ref).abs()
    dev_b, cpu_b = bucket_table(512, device=DEV).cpu(), bucket_table(512)
    print(f"[t5 flan-xl {layers}L B={B}] bf16 max {err.max():.4f} mean {err.mean():.5f}; oracle bf16 spread max {spread.max():.4f} "
          f"mean {spread.mean():.5f}; CUDA vs CPU bucket table: {int((dev_b != cpu_b).sum())} of 1023 entries differ")
    assert torch.isfinite(got).all()
    assert err.max() <= 1.5 * spread.max() + 0.02 and err.mean() <= 1.5 * spread.mean() + 1e-3


def test_flan_t5_xl_shape_fp32_against_transformers():
    transformers = pytest.importorskip("transformers")
    cfg = dict(FLAN, num_layers=2)
    sd = _random_sd(cfg, 8)
    hf = transformers.T5EncoderModel(transformers.T5Config(num_layers=2, feed_forward_proj="gated-gelu", dropout_rate=0.0, **FLAN)).eval()
    hf.load_state_dict(sd, strict=False)
    ids, mask = _ids(4, 120, FLAN["vocab_size"], 4)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref = hf.to(DEV)(input_ids=ids.to(DEV), attention_mask=mask.to(DEV)).last_hidden_state
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    got = _encoder(cfg, sd, torch.float32).encode(ids.to(DEV), mask.to(DEV))
    assert (got - ref).abs().max().item() <= 1e-4


def test_in_place_weight_writes_are_used():
    """The engine borrows the parameters: after load_state_dict (an in-place copy into the same storage) the next encode uses the new
    weights, equal to an encoder built from them."""
    gd = load_golden("t5_tiny.pt")
    ids, mask = gd["ids"].to(DEV), gd["mask"].to(DEV)
    enc = _encoder(TINY, gd["state_dict"], torch.bfloat16)
    first = enc.encode(ids, mask)
    other = _random_sd(TINY, 17)
    ptrs = [t.data_ptr() for t in enc.state_dict().values()]
    enc.load_state_dict(other)
    assert ptrs == [t.data_ptr() for t in enc.state_dict().values()]
    again = enc.encode(ids, mask)
    fresh = _encoder(TINY, other, torch.bfloat16).encode(ids, mask)
    assert torch.equal(again, fresh) and not torch.equal(again, first)


def test_batch_independence():
    cfg = dict(FLAN, num_layers=2)
    sd = {k: v.to(torch.bfloat16) for k, v in _random_sd(cfg, 9).items()}
    enc = _encoder(cfg, sd, torch.bfloat16)
    ids, mask = _ids(16, 120, cfg["vocab_size"], 5)
    ids, mask = ids.to(DEV), mask.to(DEV)
    full = enc.encode(ids, mask)
    for bs in (1, 2, 5):
        for s in range(0, 16, bs):
            part = enc.encode(ids[s: s + bs], mask[s: s + bs])
            assert torch.equal(part, full[s: s + bs]), (bs, s)
    perm = torch.randperm(16, generator=torch.Generator().manual_seed(0)).to(DEV)
    assert torch.equal(enc.encode(ids[perm], mask[perm]), full[perm])


# ------------------------------------------------------------------------------------------------ serving and the CLI writer
class _StubTokenizer:
    """Word ids from a fixed hash, eos 1, padded / truncated to max_length: the call signature of a HuggingFace tokenizer."""

    def __call__(self, prompts, max_length, padding, truncation, return_attention_mask, add_special_tokens, return_tensors):
        ids = torch.zeros(len(prompts), max_length, dtype=torch.long)
        mask = torch.zeros(len(prompts), max_length, dtype=torch.long)
        for i, p in enumerate(prompts):
            toks = ([2 + sum(map(ord, w)) % 250 for w in p.split()] + [1])[:max_length]
            ids[i, : len(toks)] = torch.tensor(toks)
            mask[i, : len(toks)] = 1
        return {"input_ids": ids, "attention_mask": mask}


PROMPTS = ["a red cube on a table", "two cats", "a very long caption about a small house by the sea at night with stars", "sun"]


@pytest.mark.parametrize("cfg_scale, prefix", [(1.0, False), (4.0, False), (4.0, True)])
def test_serve_prompts_equal_prompt_embeds(cfg_scale, prefix):
    from llamagen_b200.gpt import ModelArgs, Transformer
    from llamagen_b200.serve import LLM, SamplingParams
    gd = load_golden("t5_tiny.pt")
    enc = _encoder(TINY, gd["state_dict"], torch.bfloat16, max_length=12, tokenizer=_StubTokenizer())
    torch.manual_seed(5)
    gpt = Transformer(ModelArgs(n_layer=2, n_head=2, dim=128, vocab_size=256, block_size=16, cls_token_num=12, model_type="t2i",
                                caption_dim=128))
    gpt.output.weight.data.normal_(std=0.02)
    gpt = gpt.to(device=DEV, dtype=torch.bfloat16).eval()
    sp = SamplingParams(temperature=1.0, top_k=0, max_tokens=16)
    pf = [torch.tensor([3, 4, 5]), None, torch.tensor([7]), None] if prefix else None
    embs, m = enc(PROMPTS)
    feats = [embs[i][m[i] != 0] for i in range(len(PROMPTS))]
    a = LLM(gpt, cfg_scale=cfg_scale, max_num_seqs=3, seed=11, text_encoder=enc).generate(prompts=PROMPTS, sampling_params=sp, prefixes=pf)
    b = LLM(gpt, cfg_scale=cfg_scale, max_num_seqs=3, seed=11).generate(prompt_embeds=feats, sampling_params=sp, prefixes=pf)
    assert [o.outputs[0].token_ids for o in a] == [o.outputs[0].token_ids for o in b]
    # add_request(prompt=...) joining mid-sequence
    llm, ref = LLM(gpt, cfg_scale=cfg_scale, max_num_seqs=3, seed=11, text_encoder=enc), LLM(gpt, cfg_scale=cfg_scale, max_num_seqs=3, seed=11)
    outs = {}
    for k, (l, kw) in enumerate([(llm, [dict(prompt=p) for p in PROMPTS]), (ref, [dict(prompt_embeds=f) for f in feats])]):
        l.add_request(sampling_params=sp, **kw[0])
        got = []
        for _ in range(3):
            got += l.step()
        for x in kw[1:]:
            l.add_request(sampling_params=sp, **x)
        while l.has_unfinished_requests():
            got += l.step()
        outs[k] = sorted((int(o.request_id), o.outputs[0].token_ids) for o in got if o.finished)
    assert outs[0] == outs[1] and len(outs[0]) == len(PROMPTS)


def test_extract_feature_writer(tmp_path):
    from llamagen_b200.cond import load_t5_feature_files
    from llamagen_b200.sample.extract_t5_feature import write_features
    gd = load_golden("t5_tiny.pt")
    enc = _encoder(TINY, gd["state_dict"], torch.bfloat16, max_length=20, tokenizer=_StubTokenizer())
    write_features(enc, [(p, "part0", i) for i, p in enumerate(PROMPTS)], str(tmp_path), batch_size=3)
    write_features(enc, [(p, None, i) for i, p in enumerate(PROMPTS)], str(tmp_path / "csv"), batch_size=2)
    embs, mask = enc(PROMPTS)
    for sub in ("part0", "csv"):
        files = [str(tmp_path / sub / f"{i}.npy") for i in range(len(PROMPTS))]
        for i, f in enumerate(files):
            x = np.load(f)
            n = int(mask[i].sum())
            assert x.dtype == np.float32 and x.shape == (1, n, 128)
            assert torch.equal(torch.from_numpy(x[0]), embs[i, :n].float().cpu())
        e2, m2 = load_t5_feature_files(files, max_len=20, dim=128)
        assert torch.equal(m2.long(), mask.cpu())


def test_extract_t5_feature_cli(tmp_path):
    """The CLI end to end on a saved random-weight T5 directory (the tiny golden weights, safetensors + config.json) with a sentencepiece
    tokenizer trained here and saved through T5Tokenizer: jsonl mode and --prompt-csv mode; the files equal T5Encoder's valid rows."""
    spm = pytest.importorskip("sentencepiece")
    transformers = pytest.importorskip("transformers")
    import json
    from safetensors.torch import save_file
    from llamagen_b200.cond import load_t5_feature_files
    from llamagen_b200.sample.extract_t5_feature import main
    caps = ["a red cube on a table. it is small", "two cats sleeping on a sofa", "a small house by the sea at night",
            "the sun over green hills", "a dog runs in the park"]
    model = tmp_path / "ckpt" / "t5-tiny"
    model.mkdir(parents=True)
    spm.SentencePieceTrainer.train(sentence_iterator=iter(caps * 20), model_prefix=str(tmp_path / "sp"), vocab_size=48,
                                   model_type="unigram", pad_id=0, eos_id=1, unk_id=2, bos_id=-1, hard_vocab_limit=False)
    transformers.T5Tokenizer(vocab_file=str(tmp_path / "sp.model"), extra_ids=0).save_pretrained(str(model))
    gd = load_golden("t5_tiny.pt")
    save_file({k: v.contiguous() for k, v in gd["state_dict"].items()}, str(model / "model.safetensors"))
    (model / "config.json").write_text(json.dumps(dict(TINY, relative_attention_num_buckets=32, layer_norm_epsilon=1e-6,
                                                       feed_forward_proj="gated-gelu")))
    data = tmp_path / "data"
    data.mkdir()
    for name, rows in (("part_a.jsonl", caps[:3]), ("part_b.jsonl", caps[3:])):
        (data / name).write_text("".join(json.dumps({"text": [c, "llava " + c]}) + "\n" for c in rows))
    (tmp_path / "prompts.tsv").write_text("Prompt\n" + "\n".join(caps) + "\n")
    common = ["--t5-model-path", str(tmp_path / "ckpt"), "--t5-model-type", "t5-tiny", "--precision", "bf16", "--max-length", "16",
              "--batch-size", "2"]
    main(["--data-path", str(data), "--t5-path", str(tmp_path / "feat"), "--data-start", "0", "--data-end", "1", "--trunc-caption"]
         + common)
    main(["--prompt-csv", str(tmp_path / "prompts.tsv"), "--t5-path", str(tmp_path / "csv")] + common)
    enc = T5Encoder.from_pretrained(str(model), dtype=torch.bfloat16, device=DEV, max_length=16)
    for texts, files in ((([c.split(".")[0] for c in caps]), [str(tmp_path / "feat" / d / f"{i}.npy") for d, n in (("part_a", 3), ("part_b", 2))
                                                             for i in range(n)]),
                         (caps, [str(tmp_path / "csv" / f"{i}.npy") for i in range(len(caps))])):
        embs, mask = enc(texts)
        got, got_mask = load_t5_feature_files(files, max_len=16, dim=128)
        assert torch.equal(got_mask.long(), mask.cpu())
        assert torch.equal(got, (embs.float() * mask[:, :, None]).cpu())
