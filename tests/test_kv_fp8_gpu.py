"""GPU: the fp8 (e4m3) KV cache (`Transformer.set_kv_cache("fp8")`, samplers' --kv-cache-dtype fp8) through the fused TMA decode
attention, its deep / NST-3/4 rings, the QKV epilogue writer and the CUDA-core attention.

Parity protocol (like the fp16 tests): the engine is teacher-forced on the greedy stream of the fp32 oracle WITH an fp8 cache
(ref32); the model-dtype oracle with an fp8 cache (ref16) has exactly the engine's semantics, and the engine must stay within
1.5x ref16's own spread from ref32 (max and mean) plus the dtype's floor; arg-max and tokens must agree wherever ref32's top-1 /
top-2 gap exceeds twice that bound."""
import os

import pytest
import torch

from kv_fp8_oracle import KvFp8Oracle, e4m3_bytes
from util import build_gpt, cpu_state, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

FLOORS = {torch.bfloat16: (0.02, 0.005), torch.float16: (0.0025, 0.000625)}


def _gen(model, cond, S, em, **kw):
    from llamagen_b200 import generate
    toks, logits = generate(model, cond.cuda(), S, emb_masks=None if em is None else em.cuda(), sample_logits=False,
                            return_logits=True, **kw)
    torch.cuda.synchronize()
    return toks.cpu(), logits.cpu()


def _fp8_parity(m, cond, S, em=None, scales=None):
    """Returns (engine logits, max bound, teacher stream, ref16 oracle after its run)."""
    cfg = oracle_cfg(m)
    dt = m.tok_embeddings.weight.dtype
    cond32 = cond if cond.dtype == torch.long else cond.float()
    ref_t, ref_l = KvFp8Oracle(cpu_state(m, torch.float32), cfg, scales).generate(cond32, S, emb_masks=em, cfg_scale=4.0,
                                                                                   sample_logits=False)
    o16 = KvFp8Oracle(cpu_state(m), cfg, scales)
    _, h_l = o16.generate(cond, S, emb_masks=em, cfg_scale=4.0, sample_logits=False, teacher=ref_t)
    fmax, fmean = FLOORS[dt]
    tol_max = 1.5 * (h_l - ref_l).abs().max().item() + fmax
    tol_mean = 1.5 * (h_l - ref_l).abs().mean().item() + fmean
    m.set_kv_cache("fp8", scales)
    toks, logits = _gen(m, cond, S, em, cfg_scale=4.0, teacher=ref_t.clone())
    for other in (ref_l, h_l):
        err = (logits - other).abs()
        assert err.max().item() <= tol_max, (err.max().item(), tol_max)
        assert err.mean().item() <= tol_mean, (err.mean().item(), tol_mean)
    decisive = top2_gap(ref_l) > 2 * tol_max
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    assert torch.equal(toks.t()[decisive], ref_t.t()[decisive])
    return logits, tol_max, ref_t, o16


def _registry_model(name, dtype, seed, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(seed)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dtype).eval()


def _ordinal(b):
    b = b.to(torch.int32)
    mag = b & 0x7F
    return torch.where(b & 0x80 != 0, -mag, mag)


@pytest.fixture
def one_chain(monkeypatch):
    """The byte checks read layer 0 as one [rows, H, maxS, hdp] block: that is the layout of a single decode chain (with n chains,
    chain g keeps all its layers in the g-th n-th of the region)."""
    monkeypatch.setenv("LG_SPLIT", "1")


def _check_cache_bytes(m, o16, scales=None):
    """Layer 0's K and V bytes read straight from the workspace (DESIGN §3 layout at the 256-byte aligned base) against the
    ref16 oracle's e4m3 bytes: <= 0.1 % of the written prefix may differ, each by exactly one code; the rest is zero."""
    assert os.environ.get("LG_SPLIT") == "1", "single-chain layout only: use the one_chain fixture"
    c = m.config
    L, H, hd = c.n_layer, c.n_head, c.dim // c.n_head
    rows, maxS = m._ws_shape
    hdp = 112 if hd == 100 else hd
    ws = m._workspace
    off = (ws.data_ptr() + 255) // 256 * 256 - ws.data_ptr()
    layer = rows * H * maxS * hdp
    kv_region = (L * layer + 255) // 256 * 256
    ks, vs = (1.0, 1.0) if scales is None else scales[0]
    n_written = o16.max_seq
    saturated = 0
    for which, base, s, ref in (("k", off, ks, o16.k[0].tensor), ("v", off + kv_region, vs, o16.v[0].tensor)):
        got = ws[base: base + layer].view(rows, H, maxS, hdp).cpu()
        R = ref.shape[0]
        npos = int((ref.abs().sum(dim=(0, 1, 3)) != 0).nonzero().max().item()) + 1
        want = e4m3_bytes(ref[:, :, :npos], s)
        mine = got[:R, :, :npos, :hd]
        diff = mine != want
        assert diff.float().mean().item() <= 1e-3, (which, diff.float().mean().item())
        assert ((_ordinal(mine) - _ordinal(want)).abs() <= 1).all(), which
        assert got[:, :, npos:].eq(0).all() and got[R:].eq(0).all(), which
        if hdp > hd:
            assert got[..., hd:].eq(0).all(), which
        sat = (want == 0x7E) | (want == 0xFE)
        assert torch.equal(mine[sat], want[sat]), which
        saturated += int(sat.sum())
        assert npos <= n_written
    return saturated


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_fp8_tiny_goldens_teacher_forced(name, dtype, one_chain):
    g = load_golden(name)
    m = build_gpt(g["cfg"], g["state_dict"], dtype)
    cond = g["cond"] if name == "gpt_c2i.pt" else g["cond"].to(dtype)
    _, _, _, o16 = _fp8_parity(m, cond, g["S"], g["emb_masks"])
    _check_cache_bytes(m, o16)


@pytest.mark.parametrize("B,dtype", [(1, torch.bfloat16), (9, torch.bfloat16), (40, torch.bfloat16), (9, torch.float16)])
def test_gpt_l_fp8_teacher_forced(B, dtype, one_chain):
    """B = 1: small-row path with the deep ring of the fused attention; B = 9 / 40: the 2-stage fused kernel."""
    m = _registry_model("GPT-L", dtype, 1, block_size=256, vocab_size=16384)
    torch.manual_seed(B)
    _, _, _, o16 = _fp8_parity(m, torch.randint(0, 1000, (B,)), 6)
    _check_cache_bytes(m, o16)


def test_gpt_3b_head_dim_100_fp8(one_chain):
    """hd 100: 112-byte fp8 rows on the TMA kernel."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(3)
    m = Transformer(ModelArgs(n_layer=4, n_head=32, dim=3200, block_size=576, vocab_size=16384))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=torch.bfloat16).eval()
    _, _, _, o16 = _fp8_parity(m, torch.tensor([1, 2, 3]), 5)
    _check_cache_bytes(m, o16)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_t2i_fp8_masked_prefill_tensor_core_attention(dtype, monkeypatch, one_chain):
    """t2i, 120-token condition with emb_masks at B = 8: the fp8 condition prefill runs on attn_prefill_tc_kernel. The same run
    with LG_ATTN_PREFILL_TC=0 (CUDA-core attention) is within the bound; in bf16 it is not bit-identical, which shows the two runs
    took different kernels (the dispatch does not depend on the 16-bit type; in fp16 both kernels give the same logits on this
    model). The cache bytes the prefill read are checked against the oracle's."""
    g = load_golden("gpt_t2i.pt")
    B = 8
    torch.manual_seed(4)
    em = torch.zeros(B, 120)
    for b, n in enumerate((5, 61, 120, 17, 90, 1, 33, 100)):
        em[b, -n:] = 1
    cond = (torch.randn(B, 120, 64) * em[:, :, None]).to(dtype)
    m = build_gpt(g["cfg"], g["state_dict"], dtype)
    tc, tol, ref_t, o16 = _fp8_parity(m, cond, 5, em)
    _check_cache_bytes(m, o16)
    monkeypatch.setenv("LG_ATTN_PREFILL_TC", "0")
    m = build_gpt(g["cfg"], g["state_dict"], dtype)
    core, _, _, _ = _fp8_parity(m, cond, 5, em)
    assert (tc - core).abs().max().item() <= tol
    if dtype == torch.bfloat16:
        assert not torch.equal(tc, core)            # only the prefill attention differs between the two runs


def test_fp8_per_layer_scales(one_chain):
    """Non-unit power-of-two scales, K 2^(l mod 3 - 1) and V 2^(1 - l mod 3), against the oracle with the same scales."""
    m = _registry_model("GPT-B", torch.bfloat16, 2, block_size=256, vocab_size=16384)
    scales = [[2.0 ** (l % 3 - 1), 2.0 ** (1 - l % 3)] for l in range(m.n_layer)]
    logits, tol, _, o16 = _fp8_parity(m, torch.tensor([5, 6, 7]), 6, scales=scales)
    _check_cache_bytes(m, o16, scales)
    unit, _, _, _ = _fp8_parity(m, torch.tensor([5, 6, 7]), 6)
    assert not torch.equal(logits, unit)          # the scales change what is stored


def test_fp8_saturates_like_the_oracle(one_chain):
    """Layer 0's key rows of wqkv scaled up so that |k| > 448: the cache holds 0x7E / 0xFE exactly where the oracle saturates."""
    g = load_golden("gpt_c2i.pt")
    sd = dict(g["state_dict"])
    D = g["cfg"]["dim"]
    w = sd["layers.0.attention.wqkv.weight"].clone()
    w[D:2 * D] *= 3000.0
    sd["layers.0.attention.wqkv.weight"] = w
    m = build_gpt(g["cfg"], sd, torch.bfloat16)
    cfg = oracle_cfg(m)
    ref_t, _ = KvFp8Oracle(cpu_state(m, torch.float32), cfg).generate(g["cond"], 6, cfg_scale=4.0, sample_logits=False)
    o16 = KvFp8Oracle(cpu_state(m), cfg)
    o16.generate(g["cond"], 6, cfg_scale=4.0, sample_logits=False, teacher=ref_t)
    m.set_kv_cache("fp8")
    _gen(m, g["cond"], 6, None, cfg_scale=4.0, teacher=ref_t.clone())
    assert _check_cache_bytes(m, o16) > 0


def test_fp8_changes_logits_and_shrinks_workspace():
    g = load_golden("gpt_c2i.pt")
    m = build_gpt(g["cfg"], g["state_dict"], torch.bfloat16)
    _, auto = _gen(m, g["cond"], 8, None, cfg_scale=4.0)
    ws16 = m._workspace.numel()
    m.set_kv_cache("fp8")
    _, f8 = _gen(m, g["cond"], 8, None, cfg_scale=4.0)
    ws8 = m._workspace.numel()
    c = m.config
    rows, maxS = m._ws_shape
    kv16 = 2 * c.n_layer * rows * c.n_head * maxS * (c.dim // c.n_head) * 2
    assert abs((ws16 - ws8) - kv16 // 2) <= 512, (ws16, ws8, kv16)
    assert not torch.equal(auto, f8)
    m.set_kv_cache("auto")
    _, back = _gen(m, g["cond"], 8, None, cfg_scale=4.0)
    assert torch.equal(back, auto)


def _run_env(monkeypatch, env, build, cond, S, teacher):
    for k in ("LG_ATTN_TMA", "LG_NO_GRAPH", "LG_SPLIT", "LG_FUSE_TAIL", "LG_ATTN_NST"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = build()
    m.set_kv_cache("fp8")
    forced = _gen(m, cond, S, None, cfg_scale=4.0, teacher=teacher)
    from llamagen_b200 import generate
    sampled = generate(m, cond.cuda(), S, cfg_scale=4.0, temperature=1.0, top_k=50, top_p=1.0, sample_logits=True, seed=5).cpu()
    return forced[0], forced[1], sampled


def test_fp8_paths_agree(monkeypatch):
    """CUDA-core attention within the bound of the default; the ring-depth, chain-count, tail and graph switches bit-identical to it."""
    S, B = 8, 24
    cond = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(3))

    def build():
        return _registry_model("GPT-B", torch.bfloat16, 7, block_size=256, vocab_size=16384)

    m = build()
    _, tol, _, _ = _fp8_parity(m, cond, S)
    del m
    teacher = torch.randint(0, 16384, (B, S), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
    base = _run_env(monkeypatch, {"LG_SPLIT": "1"}, build, cond, S, teacher)
    _, logits, _ = _run_env(monkeypatch, {"LG_ATTN_TMA": "0", "LG_SPLIT": "1"}, build, cond, S, teacher)
    assert (logits - base[1]).abs().max().item() <= tol
    for env in ({"LG_ATTN_NST": "3", "LG_SPLIT": "1"}, {"LG_SPLIT": "2"}, {"LG_FUSE_TAIL": "0", "LG_SPLIT": "1"},
                {"LG_NO_GRAPH": "1", "LG_FUSE_TAIL": "0", "LG_SPLIT": "1"}):
        other = _run_env(monkeypatch, env, build, cond, S, teacher)
        for i in range(3):
            assert torch.equal(other[i], base[i]), (env, i)


def test_serve_llm_fp8_matches_generate():
    from llamagen_b200 import GPT_models, generate
    from llamagen_b200.serve import LLM, SamplingParams
    torch.manual_seed(0)
    gpt = GPT_models["GPT-B"](vocab_size=16384, block_size=64, num_classes=1000, cls_token_num=1, model_type="c2i")
    gpt = gpt.to("cuda", torch.bfloat16).eval()
    gpt.output.weight.data.normal_(std=0.02)
    S, slots = 64, 4
    sp = SamplingParams(temperature=1.0, top_p=1.0, top_k=2000, max_tokens=S)
    llm = LLM(gpt, cfg_scale=4.0, num_classes=1000, max_num_seqs=slots, seed=11, kv_cache_dtype="fp8")
    assert gpt._kv_cache[0] == "fp8"
    labels = [207, 360, 387, 974, 88]
    outs = []
    for c in labels:
        llm.add_request([c], sp)
    while llm.has_unfinished_requests():
        outs += llm.step()
    got = {int(o.request_id): o.outputs[0].token_ids for o in outs}
    for rid, c in enumerate(labels):
        ref = generate(gpt, torch.full((slots,), c, device="cuda"), S, cfg_scale=4.0, temperature=1.0, top_k=2000, top_p=1.0, seed=11 + rid)
        assert ref[0].cpu().tolist() == got[rid], rid


def test_sample_c2i_cli_fp8(tmp_path, monkeypatch):
    from llamagen_b200.sample import sample_c2i
    monkeypatch.chdir(tmp_path)
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--image-size", "256", "--cfg-scale", "4.0",
                                                 "--top-k", "2000", "--seed", "1", "--kv-cache-dtype", "fp8"])
    sample_c2i.main(args)
    from PIL import Image
    img = Image.open(tmp_path / "sample_c2i.png")
    assert img.size == (4 * 256 + 5 * 2, 2 * 256 + 3 * 2)
