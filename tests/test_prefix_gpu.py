"""GPU: image completion, generate(..., prefix=tokens) / lg_generate_prefix, and attn_causal_tc_kernel on fp8 caches.

* Kernel, one call at a time: lg_test_attention runs kernel 2 on fp8 caches against the float64 reference of the decoded codes,
  with test_attention_gpu's inputs (wide scores, needles, poison) and its bound; needles sit at 16-row box, 32-key box, 64-key
  block, ring and diagonal edges; scales 2^-8, 1 and 2^7; the t2i emb-mask; Tq 129, 257, 1143; R * Tq > 65535.
* fp32 exact mode on the tiny golden models: greedy tokens bit-exact against the prefix oracle, logits at steps >= P to 1e-4.
* 16-bit models at full layer width (GPT-L c2i under CFG, a GPT-3B-shaped hd 100 model, GPT-XL t2i with emb-masks, also with an
  fp8 KV cache): the prefix run's logits at steps >= P against the same model's fp32 twin teacher-forced on the prefix run's own
  tokens, within 1.5 x the spread between the 16-bit and the fp32 teacher-forced runs, and arg-max agreement where the fp32 top-2
  gap exceeds twice that bound.
* Cache contents after the prefill, chains (LG_SPLIT 1 vs 2, bit-identical), a capped scratch that forces >= 3 chunks, and the
  sampling keys: each token k >= P redrawn by lg_sample from the run's own dumped row k with step k."""
import ctypes
import zlib

import pytest
import torch

import test_attention_gpu as ta
from kv_fp8_oracle import KvFp8Oracle
from oracle import GPTOracle, sample_oracle
from prefix_oracle import prefix_oracle
from util import build_gpt, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------ kernel 2, fp8
def _kernel_cases():
    cs, i = [], 0
    for dt in ("bf16", "f16"):
        for hd, hdp in ((64, 64), (128, 128), (100, 112)):
            for Tq in (129, 257):
                sc = ta.FP8_SCALES[i % 3]
                i += 1
                mask = ("ragged", 3, 120) if Tq == 257 else None
                cs.append(ta.Case(f"causal_fp8_{dt}_{hd}_{hdp}_tq{Tq}", dt, "fp8", hd, 6 if mask else 3, 2, Tq + 7, (2, 2, 0), hdp=hdp,
                                  Tq=Tq, pos=("scalar", 0), mask=mask, scales=sc))
    # R * Tq = 58 * 1143 > 65535: beyond attention_kernel's grid
    cs.append(ta.Case("causal_fp8_bf16_64_tq1143_rows", "bf16", "fp8", 64, 58, 1, 1150, (2, 2, 0), Tq=1143, pos=("scalar", 0),
                      scales=ta.FP8_SCALES[0], needles=False))
    cs.append(ta.Case("causal_fp8_f16_112_tq1143_mask", "f16", "fp8", 100, 6, 2, 1150, (2, 2, 0), hdp=112, Tq=1143,
                      pos=("scalar", 0), mask=("ragged", 3, 120), scales=ta.FP8_SCALES[2]))
    return cs


KCASES = {c.id: c for c in _kernel_cases()}


def test_kernel_cases_cover_the_matrix():
    cs = list(KCASES.values())
    assert {s for c in cs for s in c.scales} == {2.0 ** -8, 1.0, 2.0 ** 7}
    assert {(c.dt, c.hd) for c in cs} >= {(dt, hd) for dt in ("bf16", "f16") for hd in (64, 128, 100)}
    assert {c.Tq for c in cs} == {129, 257, 1143} and any(c.R * c.Tq > 65535 for c in cs) and any(c.mask for c in cs)


@pytest.mark.parametrize("cid", list(KCASES))
def test_causal_fp8_call(cid):
    c = KCASES[cid]
    seed = zlib.crc32(cid.encode())
    worst = ta._one(c, "wide", None, seed)[2]
    needles = [("abs", j) for j in (0, 15, 16, 31, 32, 33, 63, 64, 127, 128, 191, 192)] + [("rel", d) for d in (0, 1, 15, 16, 64)]
    if c.mask:
        needles += [("abs", 119), ("abs", 120)]
    if not c.needles:
        needles = [("abs", 0), ("abs", 64), ("rel", 0)]
    for i, nd in enumerate(needles):
        worst = max(worst, ta._one(c, "needle", nd, seed + 1 + i)[2])
    if c.hdp > c.hd:
        a = ta._one(c, "needle", ("rel", 1), seed + 99, pad="zero")[0]
        b = ta._one(c, "needle", ("rel", 1), seed + 99, pad="garbage")[0]
        assert torch.equal(a, b), f"{cid}: dims {c.hd}..{c.hdp - 1} of the cache rows change the output"
    print(f"[{cid}] max |out - ref| / absO {worst:.3g}")


# ------------------------------------------------------------------------------------------------------------ end to end
def _gen(model, cond, S, em=None, **kw):
    from llamagen_b200 import generate
    out = generate(model, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), return_logits=True, **kw)
    torch.cuda.synchronize()
    return out[0].cpu(), out[1].cpu()


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
def test_fp32_exact_against_prefix_oracle(name, cfg_scale):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    S, toks = g["S"], g[f"tokens_cfg{cfg_scale}"]
    for P in (1, 7, S - 1):
        pf = toks[:, :P].clone()
        pf[:, 0] = (pf[:, 0] + 3) % m.vocab_size          # a prefix the model would not have sampled
        out, logits = _gen(m, g["cond"], S, g["emb_masks"], cfg_scale=cfg_scale, sample_logits=False, prefix=pf)
        want, wl = prefix_oracle(GPTOracle(g["state_dict"], g["cfg"]), g["cond"], pf, S, emb_masks=g["emb_masks"], cfg_scale=cfg_scale,
                                 sample_logits=False)
        assert torch.equal(out[:, :P], pf.to(torch.int32))
        assert torch.equal(out, want.cpu()), f"{name} P={P}: greedy tokens differ from the prefix oracle"
        assert (logits[:P] == 0).all()
        assert (logits[P:] - wl[P:].cpu()).abs().max().item() <= 1e-4


def _model(dt, kv="auto", **cfg):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(1234)
    m = Transformer(ModelArgs(**cfg))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dt).eval()
    m.set_kv_cache(kv)
    return m


GPT_L = dict(n_layer=4, n_head=16, dim=1024, vocab_size=16384, block_size=256, num_classes=1000)
GPT_3B = dict(n_layer=2, n_head=32, dim=3200, vocab_size=16384, block_size=256, num_classes=1000)
GPT_XL_T2I = dict(n_layer=3, n_head=20, dim=1280, vocab_size=16384, block_size=256, cls_token_num=120, model_type="t2i",
                  caption_dim=2048)
FLOORS = {torch.bfloat16: 0.02, torch.float16: 0.0025}     # the dtype floors of the fp8-KV parity protocol (test_kv_fp8_gpu)


def _parity(m, cond, S, P, em=None, cfg_scale=4.0):
    """The 16-bit parity protocol for a prefix run. ref32: the fp32 prefix oracle's greedy stream from prefix pf (KvFp8Oracle, the
    fp8-cache semantics, when the model keeps an fp8 cache); ref16: the same oracle in the model dtype teacher-forced on ref32's
    stream. The engine's generate(prefix=pf) is greedy too, so up to each image's first token that differs from ref32 it is fed
    exactly ref32's stream: on those rows (k >= P, the row of the first difference included) its logits must lie within
    1.5 x ref16's own spread from ref32 plus the dtype floor, with the same arg-max wherever ref32's top-2 gap exceeds twice that."""
    dt = m.tok_embeddings.weight.dtype
    cfg = oracle_cfg(m)
    fp8 = m._kv_cache[0] == "fp8"
    make = (lambda sd: KvFp8Oracle(sd, cfg)) if fp8 else (lambda sd: GPTOracle(sd, cfg))
    sd16 = {k: v.detach() for k, v in m.state_dict().items()}
    sd32 = {k: v.float() for k, v in sd16.items()}
    g = torch.Generator().manual_seed(P)
    pf = torch.randint(0, m.vocab_size, (cond.shape[0], P), generator=g)
    c = cond.cuda()
    em_d = None if em is None else em.cuda()
    kw = dict(emb_masks=em_d, cfg_scale=cfg_scale, sample_logits=False)
    ref_t, ref_l = prefix_oracle(make(sd32), c.float() if c.is_floating_point() else c, pf.cuda(), S, **kw)
    _, h_l = prefix_oracle(make(sd16), c.to(dt) if c.is_floating_point() else c, pf.cuda(), S, teacher=ref_t, **kw)
    ref_t, ref_l, h_l = ref_t.cpu(), ref_l.cpu(), h_l.cpu()
    tol = 1.5 * (h_l[P:] - ref_l[P:]).abs().max().item() + FLOORS[dt]
    out, lg = _gen(m, cond, S, em, cfg_scale=cfg_scale, sample_logits=False, prefix=pf)
    assert torch.equal(out[:, :P], pf.to(torch.int32)) and (lg[:P] == 0).all()
    rows = 0
    for b in range(cond.shape[0]):
        d = (out[b, P:] != ref_t[b, P:]).nonzero()
        last = P + int(d[0]) if len(d) else S - 1          # rows P .. last were fed ref32's tokens
        e, r = lg[P:last + 1, b], ref_l[P:last + 1, b]
        err = (e - r).abs().max().item()
        assert err <= tol, f"P={P} image {b}: |engine - ref32| {err:.4g} > bound {tol:.4g}"
        sure = top2_gap(r) > 2 * tol
        assert torch.equal(e.argmax(-1)[sure], r.argmax(-1)[sure])
        rows += last + 1 - P
    return rows, tol


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("kv", ["auto", "fp8"])
def test_gpt_l_c2i_cfg(dt, kv):
    m = _model(dt, kv, **GPT_L)
    cond = torch.tensor([207, 360, 387, 974])
    for P in (1, 64, 127, 128, 200):
        print(dt, kv, P, _parity(m, cond, 256, P))


def test_gpt_3b_shape_hd100():
    m = _model(torch.bfloat16, "auto", **GPT_3B)
    for kv in ("auto", "fp8"):
        m.set_kv_cache(kv)
        for P in (64, 130):
            print(kv, P, _parity(m, torch.tensor([1, 2]), 256, P))


@pytest.mark.parametrize("kv", ["auto", "fp8"])
def test_gpt_xl_t2i_emb_masks(kv):
    m = _model(torch.bfloat16, kv, **GPT_XL_T2I)
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(3, 120, 2048, generator=g) * 0.5
    em = torch.stack([(torch.arange(120) >= p).float() for p in (40, 0, 100)])
    for P in (8, 64, 200):
        print(kv, P, _parity(m, cond, 256, P, em=em, cfg_scale=7.5))


def _cache_bytes(m, layers):
    """Layer 0's K and V of the full workspace as raw bytes [rows, H, max_seq, hdp * esz] (the workspace starts with the caches)."""
    rows, max_seq = m._ws_shape
    c = m.config
    hd = c.dim // c.n_head
    esz = 1 if m._kv_cache[0] == "fp8" else 2
    n = rows * c.n_head * max_seq * hd * esz
    base = (m._workspace.data_ptr() + 255) // 256 * 256 - m._workspace.data_ptr()
    ws = m._workspace[base:]
    kbytes = n * layers
    k = ws[:n].view(rows, c.n_head, max_seq, hd * esz)
    v = ws[(kbytes + 255) // 256 * 256:][:n].view(rows, c.n_head, max_seq, hd * esz)
    return k.clone(), v.clone()


@pytest.mark.parametrize("kv", ["auto", "fp8"])
def test_cache_contents_after_prefill(kv):
    cfg = dict(GPT_L, n_layer=2)
    P, S = 150, 256
    cond = torch.tensor([3, 4])
    pf = torch.randint(0, 16384, (2, P), generator=torch.Generator().manual_seed(3))
    a = _model(torch.bfloat16, kv, **cfg)
    _gen(a, cond, P + 1, cfg_scale=4.0, sample_logits=False, prefix=pf)
    ka, va = _cache_bytes(a, 2)
    b = _model(torch.bfloat16, kv, **cfg)
    teacher = torch.cat([pf, torch.zeros(2, 1, dtype=pf.dtype)], 1)
    _gen(b, cond, P + 1, cfg_scale=4.0, sample_logits=False, teacher=teacher)
    kb, vb = _cache_bytes(b, 2)
    T = 1
    assert ka[:, :, T + P:].eq(0).all() and va[:, :, T + P:].eq(0).all(), "positions >= T + P written before decoding"
    for x, y in ((ka, kb), (va, vb)):
        x, y = x[:, :, :T + P], y[:, :, :T + P]
        if kv == "fp8":
            xv = x.view(torch.float8_e4m3fn).float()
            yv = y.view(torch.float8_e4m3fn).float()
            tol = 0.13 * yv.abs() + 2.0 ** -9          # one e4m3 step of the stored value (3 mantissa bits)
        else:
            xv = x.reshape(*x.shape[:-1], -1).view(torch.bfloat16).float()
            yv = y.reshape(*y.shape[:-1], -1).view(torch.bfloat16).float()
            tol = 2.0 ** -7 * yv.abs() + 1e-6          # one bf16 ulp: the batched and the decode GEMMs sum in other orders
        assert ((xv - yv).abs() <= tol).float().mean().item() >= 0.999
        assert (xv - yv).abs().max().item() <= 4 * tol.max().item()


def test_chains_are_bit_identical(monkeypatch):
    """LG_SPLIT=1 and 2 at B = 64 under CFG (two chains of 64 rows): the prefill runs the same chunks in both, so tokens and logits are
    bit-identical, as lg_generate's are."""
    from llamagen_b200 import _lib, generate
    lib = _lib.load()
    B, P = 64, 100
    cond = torch.arange(B)
    pf = torch.randint(0, 16384, (B, P), generator=torch.Generator().manual_seed(9))
    res, plain = [], []
    for split in ("1", "2"):
        monkeypatch.setenv("LG_SPLIT", split)
        m = _model(torch.bfloat16, "auto", **dict(GPT_L, n_layer=2))
        plain.append(generate(m, cond.cuda(), 256, cfg_scale=4.0, seed=11, top_k=100).cpu())
        res.append(_gen(m, cond, 256, cfg_scale=4.0, seed=11, prefix=pf, top_k=100))
        chains = ctypes.c_int(0)
        chunks = lib.lg_test_prefix_chunks(m.engine(), ctypes.byref(chains))
        assert (chains.value, chunks) == (int(split), 4), (split, chains.value, chunks)   # 2 blocks of 32 images per half
    assert torch.equal(plain[0], plain[1]), "lg_generate itself differs between one and two chains here"
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_chunks_match_one_chunk(monkeypatch):
    """B = 9 (no two-chain split): the whole half in one chunk, then a scratch capped at 3 rows: 3 chunks per half."""
    from llamagen_b200 import _lib, gpt
    B, P = 9, 130
    cond = torch.arange(B)
    pf = torch.randint(0, 16384, (B, P), generator=torch.Generator().manual_seed(4))
    m = _model(torch.bfloat16, "auto", **dict(GPT_L, n_layer=2))
    one = _gen(m, cond, 256, cfg_scale=4.0, sample_logits=False, prefix=pf)
    lib = _lib.load()
    assert lib.lg_test_prefix_chunks(m.engine(), None) == 2    # the conditional and the unconditional rows
    need = ctypes.c_size_t()
    _lib.check(lib.lg_prefix_workspace_bytes(m.engine(), 3, 1 + P, ctypes.byref(need)))
    monkeypatch.setattr(gpt, "PREFIX_SCRATCH_CAP", need.value)
    m._prefix_ws = None
    many = _gen(m, cond, 256, cfg_scale=4.0, sample_logits=False, prefix=pf)
    assert lib.lg_test_prefix_chunks(m.engine(), None) == 2 * 3
    # greedy: identical up to each image's first disagreement, which must sit at a near tie of the one-chunk run's row
    top = torch.topk(one[1], 2, -1).values
    for i in range(B):
        d = (one[0][i, P:] != many[0][i, P:]).nonzero()
        if len(d):
            k = P + int(d[0])
            assert float(top[k, i, 0] - top[k, i, 1]) <= 0.5, f"image {i}: token {k} differs away from a tie"
    # other chunk sizes run other GEMM plans (split-K), so the bf16 roundings differ: a few ulps at logit scale ~2
    assert (one[1][P] - many[1][P]).abs().max().item() <= 0.25


def test_sampling_keys_are_lg_generate_keys():
    from llamagen_b200 import _lib
    m = _model(torch.bfloat16, "auto", **dict(GPT_L, n_layer=2))
    B, S, P, seed = 4, 256, 100, 77
    pf = torch.randint(0, 16384, (B, P), generator=torch.Generator().manual_seed(2))
    out, lg = _gen(m, torch.tensor([1, 2, 3, 4]), S, cfg_scale=4.0, seed=seed, top_k=1000, top_p=0.95, temperature=1.0, prefix=pf)
    lib = _lib.load()
    sc = _lib.SampleCfg(1.0, -1, 1.0, 1000, 0.95, 0, seed)
    rows = lg.cuda()
    idx = torch.empty(B, dtype=torch.int32, device="cuda")
    for k in range(P, S):
        _lib.check(lib.lg_sample(_lib.ptr(rows[k].contiguous()), B, m.vocab_size, 0, _lib.LG_DTYPE_F32, ctypes.byref(sc), k,
                                 _lib.ptr(idx), None, _lib.current_stream("cuda")), "lg_sample")
        assert torch.equal(idx.cpu(), out[:, k]), f"token {k} is not lg_generate's draw for index {k}"


def test_token_p_distribution_chi2():
    """The distribution token P is drawn from, after the prefill: 256 images with one class and one prefix per call, 40 seeds, on the
    tiny c2i model in fp32 under CFG with top-k 20, against the prefix oracle's mixed row P passed through the oracle's filter."""
    g = load_golden("gpt_c2i.pt")
    m = build_gpt(g["cfg"], g["state_dict"], torch.float32)
    B, P, S, n_rounds = 256, 5, 6, 40
    pf = g["tokens_cfg4.0"][:1, :P].repeat(B, 1)
    cond = torch.full((B,), int(g["cond"][0]))
    _, wl = prefix_oracle(GPTOracle(g["state_dict"], g["cfg"]), cond[:1], pf[:1], S, cfg_scale=4.0, sample_logits=False)
    _, rprobs = sample_oracle(wl[P], temperature=1.0, top_k=20, top_p=1.0, sample_logits=False)
    V = m.vocab_size
    counts = torch.zeros(V)
    from llamagen_b200 import generate
    for r in range(n_rounds):
        out = generate(m, cond.cuda(), S, cfg_scale=4.0, temperature=1.0, top_k=20, top_p=1.0, seed=1000 + r, prefix=pf).cpu()
        assert torch.equal(out[:, :P], pf.to(torch.int32))
        counts += torch.bincount(out[:, P].long(), minlength=V).float()
    n = B * n_rounds
    exp = rprobs[0] * n
    keep = exp > 0
    assert counts[~keep].sum() == 0, "sampled a filtered token"
    chi2 = (((counts - exp) ** 2)[keep] / exp[keep]).sum().item()
    dof = int(keep.sum()) - 1
    assert chi2 < dof + 6 * (2 * dof) ** 0.5, (chi2, dof)      # ~6 sigma, as test_sampling_gpu's check


def test_sample_c2i_cli_prefix_image(tmp_path, monkeypatch):
    """sample_c2i --prefix-image <png> --prefix-rows 4: the PNG is written, and the first 4 * g tokens of every image are the codes
    VQModel.encode gives for the centre-cropped image."""
    import numpy as np
    from PIL import Image
    from llamagen_b200.sample import sample_c2i
    from llamagen_b200.sample.vq_demo import center_crop
    monkeypatch.chdir(tmp_path)
    rng = np.random.default_rng(0)
    img = (rng.random((300, 280, 3)) * 255).astype(np.uint8)
    img[:150] //= 3                                            # some structure: a darker top half
    Image.fromarray(img).save(tmp_path / "in.png")
    seen = {}
    real_generate, real_load_vq = sample_c2i.generate, sample_c2i.load_vq

    def gen(*a, **kw):
        seen["prefix"] = kw.get("prefix")
        seen["out"] = real_generate(*a, **kw)
        return seen["out"]

    def load_vq(*a, **kw):
        seen["vq"] = real_load_vq(*a, **kw)
        return seen["vq"]
    monkeypatch.setattr(sample_c2i, "generate", gen)
    monkeypatch.setattr(sample_c2i, "load_vq", load_vq)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--image-size", "256", "--cfg-scale", "4.0", "--top-k", "2000",
                                                 "--seed", "1", "--class-labels", "1", "2", "3",
                                                 "--prefix-image", str(tmp_path / "in.png"), "--prefix-rows", "4"])
    sample_c2i.main(args)
    out_png = Image.open(tmp_path / "sample_c2i.png")
    assert out_png.size[0] > 256 and out_png.size[1] >= 256
    g = 16
    x = center_crop(Image.open(tmp_path / "in.png").convert("RGB"), 256)
    xt = torch.from_numpy(2.0 * (np.array(x) / 255.0) - 1.0).permute(2, 0, 1)[None].float().cuda()
    _, _, [_, _, codes] = seen["vq"].encode(xt)
    codes = codes.reshape(-1)[: 4 * g].cpu()
    out = seen["out"].cpu()
    assert out.shape == (3, g * g)
    for b in range(3):
        assert torch.equal(out[b, : 4 * g].long(), codes), f"image {b}: the first 4 rows are not the encoded codes"
    assert seen["prefix"].shape == (3, 4 * g)
