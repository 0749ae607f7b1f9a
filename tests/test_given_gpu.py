"""GPU: inpainting, generate(..., given=tokens, given_mask=mask) / lg_generate_given, and the sample kernel's given select.

* Bit identity with the existing paths: an all-False mask is generate(seed=s), and a mask of the first P columns is
  generate(prefix=given[:, :P], seed=s), for c2i and t2i, fp32 / bf16 / fp16, with and without CFG, at B = 1 and at B = 64 (two
  decode chains on the 16-bit c2i models, on the given path too). Given tokens are kept everywhere.
* fp32 greedy tokens equal the given oracle's exactly: a box hole and per-image masks on the golden models (one with a negative
  prompt), and runs of 64, 96 and 128 given tokens (windows of 2 or 3 chunks, one ending in a one-row chunk) on a 16 x 16 grid.
* bf16 greedy with a box hole: every drawn token is the arg-max of score()'s teacher-forced logits of the final sequence, within 4
  bf16 ulps (test_serve_sjd_gpu's bound); per-image masks too, where a decode step's fused tail feeds the given tokens.
* fp8 KV cache and fp8 weights: an all-False mask is generate() under the same settings; one seed gives one result.
* The sample kernel: given all -1 draws what lg_sample_rows draws; a given token goes to out_seq and next_tokens."""
import ctypes

import pytest
import torch

from given_oracle import given_oracle
from oracle import GPTOracle
from util import build_gpt, load_golden, oracle_cfg

pytestmark = pytest.mark.gpu


def _model(dt, kv="auto", w8="auto", t2i=False, **kw):
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(4321)
    cfg = dict(n_layer=2, n_head=4, dim=256, vocab_size=4096, block_size=256, num_classes=1000)
    if t2i:
        cfg.update(cls_token_num=16, model_type="t2i", caption_dim=2048)
    cfg.update(kw)
    m = Transformer(ModelArgs(**cfg))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dt).eval()
    m.set_kv_cache(kv)
    m.set_weight_dtype(w8)
    return m


def _cond(m, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    if m.model_type == "c2i":
        return torch.randint(0, 1000, (B,), generator=g).cuda(), None
    T, C = m.cls_token_num, m.config.caption_dim
    cond = (0.5 * torch.randn(B, T, C, generator=g)).to(device="cuda", dtype=m.tok_embeddings.weight.dtype)
    em = torch.ones(B, T)
    for b in range(B):
        em[b, : b % 5] = 0                                  # left padding
    return cond, em.cuda()


def _box(grid, top, left, bottom, right):
    m = torch.ones(grid, grid, dtype=torch.bool)
    m[top:bottom, left:right] = False
    return m.reshape(-1)


def _run(m, cond, em, S, **kw):
    from llamagen_b200 import generate
    out = generate(m, cond, S, em, **kw)
    torch.cuda.synchronize()
    return out.cpu()


DTYPES = [torch.float32, torch.bfloat16, torch.float16]


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
@pytest.mark.parametrize("dt", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
@pytest.mark.parametrize("B", [1, 64])
def test_bit_identity_with_plain_and_prefix(kind, dt, cfg_scale, B, monkeypatch):
    from llamagen_b200 import _lib
    monkeypatch.delenv("LG_SPLIT", raising=False)
    m = _model(dt, t2i=kind == "t2i")
    S, P = 256, 100
    cond, em = _cond(m, B)
    given = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(B))
    kw = dict(cfg_scale=cfg_scale, top_k=100, seed=5, cfg_interval=150 if cfg_scale > 1 else -1)
    plain = _run(m, cond, em, S, **kw)
    none = _run(m, cond, em, S, given=given, given_mask=torch.zeros(S, dtype=torch.bool), **kw)
    assert torch.equal(none, plain), "an all-False mask differs from generate()"
    lib = _lib.load()
    chains = []

    def ran():   # the decode chains of the model's last prefill of a leading run
        n = ctypes.c_int(0)
        lib.lg_test_prefix_chunks(m.engine(), ctypes.byref(n))
        chains.append(n.value)

    pre = _run(m, cond, em, S, prefix=given[:, :P], **kw)
    ran()
    if B > 1:   # fewer rows than the workspace holds run one chain: the counter now reads 1 whatever the two calls below run
        _run(m, cond[: B // 2], None if em is None else em[: B // 2], S, prefix=given[: B // 2, :P], **kw)
        ran()
    lead = torch.zeros(1, S, dtype=torch.bool)
    lead[:, :P] = True
    got = _run(m, cond, em, S, given=given, given_mask=lead, **kw)
    ran()
    assert torch.equal(got, pre), "a leading mask differs from generate(prefix=)"
    assert torch.equal(got[:, :P], given[:, :P].to(torch.int32))
    assert chains[-1] == chains[0], f"the given call ran {chains[-1]} chains, generate(prefix=) {chains[0]}"
    if B == 64 and dt != torch.float32 and kind == "c2i":
        assert chains == [2, 1, 2], f"B = 64 was meant to run two decode chains on both paths, ran {chains}"


def _golden(name):
    g = load_golden(name)
    return g, build_gpt(g["cfg"], g["state_dict"], torch.float32)


def _exact(m, sd, cond, gv, mask, S, cfg_scale, em=None, neg=None, nm=None):
    """fp32 greedy generate(given=) of model m against the given oracle on its state_dict sd; the given tokens are kept."""
    kw = dict(cfg_scale=cfg_scale, sample_logits=False)
    extra = {} if neg is None else dict(negative_cond=neg, negative_emb_masks=nm)
    out = _run(m, cond, em, S, given=gv, given_mask=mask, **kw, **extra)
    orc = GPTOracle({k: v.cuda() for k, v in sd.items()}, oracle_cfg(m))
    want, wl = given_oracle(orc, cond.cuda(), gv.cuda(), mask.expand(gv.shape).cuda(), S,
                            emb_masks=None if em is None else em.cuda(), negative=None if neg is None else neg.cuda(),
                            negative_emb_masks=None if nm is None else nm.cuda(), **kw)
    mk = mask.expand(gv.shape)
    assert torch.equal(out[mk], gv[mk].to(torch.int32))
    return out, want.cpu(), wl.cpu()


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
@pytest.mark.parametrize("cfg_scale", [1.0, 4.0])
def test_fp32_exact_against_given_oracle(name, cfg_scale):
    g, m = _golden(name)
    S = g["S"]
    cond, em = g["cond"], g["emb_masks"]
    B = cond.shape[0]
    gv = (g[f"tokens_cfg{cfg_scale}"].long() + 3) % m.vocab_size      # tokens the model would not have drawn
    masks = {"box": _box(4, 1, 1, 3, 3).view(1, S).expand(B, S),
             "per_image": torch.rand(B, S, generator=torch.Generator().manual_seed(7)) < 0.5,
             "runs_of_one": (torch.arange(S) % 2 == 1).view(1, S).expand(B, S)}
    masks["per_image"][:, 0] = False
    for key, mask in masks.items():
        out, want, _ = _exact(m, g["state_dict"], cond, gv, mask, S, cfg_scale, em=em)
        assert torch.equal(out, want), f"{name} {key}: greedy tokens differ from the given oracle"


def test_fp32_exact_with_a_negative_prompt():
    g, m = _golden("gpt_t2i.pt")
    S, cond, em = g["S"], g["cond"], g["emb_masks"]
    B, T, C = cond.shape
    neg = 0.5 * torch.randn(1, T, C, generator=torch.Generator().manual_seed(2))
    nm = torch.ones(1, T)
    nm[:, :30] = 0
    gv = (g["tokens_cfg4.0"].long() + 5) % m.vocab_size
    for mask in (_box(4, 1, 0, 3, 2).view(1, S).expand(B, S), torch.rand(B, S, generator=torch.Generator().manual_seed(1)) < 0.4):
        out, want, _ = _exact(m, g["state_dict"], cond, gv, mask, S, 4.0, em=em, neg=neg, nm=nm)
        assert torch.equal(out, want)


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_fp32_long_runs_in_window_chunks(kind):
    """fp32 greedy tokens equal the oracle's exactly on a 16 x 16 grid for runs longer than one window chunk: 64 given tokens (a window
    of 65 rows: chunks of 64 + 1, the last on the one-row per-row-position attention), 96 (64 + 33) and 128 (64 + 64 + 1), and a box
    hole with per-image extras."""
    m = _model(torch.float32, t2i=kind == "t2i", dim=128, n_head=2, vocab_size=512)
    S, B = 256, 3
    cond, em = _cond(m, B, seed=3)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    gv = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(8))
    masks = {}
    for a, n in ((40, 64), (48, 96), (20, 128)):
        masks[f"run of {n}"] = torch.zeros(B, S, dtype=torch.bool)
        masks[f"run of {n}"][:, a:a + n] = True
    hole = _box(16, 4, 4, 12, 12).view(1, S).expand(B, S).clone()
    hole[1, 100:110] = True
    masks["hole"] = hole
    for where, mask in masks.items():
        out, want, _ = _exact(m, sd, cond.cpu(), gv, mask, S, 4.0, em=None if em is None else em.cpu())
        assert torch.equal(out, want), f"{kind} {where}: greedy tokens differ from the given oracle"


def _argmax_of_score(m, cond, em, toks, mask, cfg_scale):
    from llamagen_b200 import score
    _, logits = score(m, cond, toks.cuda().long(), emb_masks=em, cfg_scale=cfg_scale, return_logits=True)
    logits = logits.float()
    drawn = ~mask.expand(toks.shape).cuda()
    picked = logits.gather(-1, toks.cuda().long()[..., None])[..., 0]
    top = logits.max(-1).values
    _, e = torch.frexp(top.abs())
    margin = 4 * torch.ldexp(torch.ones_like(top), e - 8)     # 4 bf16 ulps at the row's largest logit, as test_serve_sjd_gpu
    gap = (top - picked)[drawn]
    assert (gap <= margin[drawn]).all(), (gap.max().item(), margin.min().item())


@pytest.mark.parametrize("kind", ["c2i", "t2i"])
def test_bf16_greedy_box_hole_is_argmax_of_score(kind):
    m = _model(torch.bfloat16, t2i=kind == "t2i", dim=512, n_head=8, n_layer=4)
    S, B = 256, 4
    cond, em = _cond(m, B, seed=1)
    gv = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(6))
    hole = _box(16, 4, 4, 12, 12).view(1, S)
    per = hole.expand(B, S).clone()
    per[0, 120:124] = True                                  # given to one image inside the hole: decode steps take it
    per[2, 150] = True
    for mask in (hole, per):
        out = _run(m, cond, em, S, given=gv, given_mask=mask, cfg_scale=4.0, sample_logits=False)
        mk = mask.expand(B, S)
        assert torch.equal(out[mk], gv[mk].to(torch.int32))
        _argmax_of_score(m, cond, em, out, mask, 4.0)


@pytest.mark.parametrize("kv, w8", [("fp8", "auto"), ("auto", "fp8"), ("fp8", "fp8")])
def test_fp8_storage(kv, w8):
    m = _model(torch.bfloat16, kv=kv, w8=w8, dim=512, n_head=8)
    S, B = 256, 8
    cond, _ = _cond(m, B)
    gv = torch.randint(0, m.vocab_size, (B, S), generator=torch.Generator().manual_seed(2))
    kw = dict(cfg_scale=4.0, top_k=200, seed=3)
    plain = _run(m, cond, None, S, **kw)
    assert torch.equal(_run(m, cond, None, S, given=gv, given_mask=torch.zeros(S, dtype=torch.bool), **kw), plain)
    hole = _box(16, 2, 3, 9, 14)
    a = _run(m, cond, None, S, given=gv, given_mask=hole, **kw)
    b = _run(m, cond, None, S, given=gv, given_mask=hole, **kw)
    assert torch.equal(a, b)
    assert torch.equal(a[:, hole], gv[:, hole].to(torch.int32))


@pytest.mark.parametrize("rd", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("greedy", [0, 1])
@pytest.mark.parametrize("B", [1, 8, 64])
def test_sample_kernel_given_select(rd, greedy, B):
    from llamagen_b200 import _lib
    lib = _lib.load()
    RD = {"f32": _lib.LG_DTYPE_F32, "bf16": _lib.LG_DTYPE_BF16, "f16": _lib.LG_DTYPE_F16}[rd]
    V, S = 4096, 40
    g = torch.Generator().manual_seed(B + greedy)
    logits = (3 * torch.randn(2 * B, V, generator=g)).cuda()
    seeds = torch.randint(0, 2 ** 62, (B,), generator=g).cuda()
    steps = torch.randint(0, S, (B,), generator=g).to(torch.int32).cuda()
    sc = _lib.SampleCfg(4.0, -1, 1.0, 300, 0.9, greedy, 0)
    st = _lib.current_stream("cuda")

    def draw(given):
        seq = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
        idx = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        nxt = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        if given is None:
            _lib.check(lib.lg_sample_rows(_lib.ptr(logits), B, V, 1, RD, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps), _lib.ptr(idx),
                                          _lib.ptr(seq), S, st), "lg_sample_rows")
        else:
            _lib.check(lib.lg_test_sample_given(_lib.ptr(logits), B, V, 1, RD, ctypes.byref(sc), _lib.ptr(seeds), _lib.ptr(steps),
                                                _lib.ptr(given), _lib.ptr(idx), _lib.ptr(seq), S, _lib.ptr(nxt), st), "lg_test_sample_given")
        torch.cuda.synchronize()
        return seq.cpu(), idx.cpu(), nxt.cpu()

    ref_seq, ref_idx, _ = draw(None)
    seq, idx, nxt = draw(torch.full((B, S), -1, dtype=torch.int32, device="cuda"))
    assert torch.equal(seq, ref_seq) and torch.equal(idx, ref_idx) and torch.equal(nxt, ref_idx)
    given = torch.full((B, S), -1, dtype=torch.int32)
    forced = torch.arange(B) % 3 == 0
    rows = torch.arange(B)
    st_cpu = steps.cpu().long()
    vals = (ref_idx + 11) % V
    given[rows[forced], st_cpu[forced]] = vals[forced]
    given[rows[~forced], (st_cpu[~forced] + 1) % S] = 5           # given at another step: not read
    seq, idx, nxt = draw(given.cuda())
    want = torch.where(forced, vals, ref_idx)
    assert torch.equal(idx, want) and torch.equal(nxt, want)
    assert torch.equal(seq[rows, st_cpu], want)
    other = torch.ones(B, S, dtype=torch.bool)
    other[rows, st_cpu] = False
    assert (seq[other] == -7).all()
