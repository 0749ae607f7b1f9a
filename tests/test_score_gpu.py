"""GPU: teacher-forced scoring (lg_score, Transformer.forward(idx, cond_idx, targets), llamagen_b200.score) against the golden
logits the reference produced, the scoring oracle (tests/score_oracle.py), the decode path, and the long causal tensor-core attention
(attn_causal_tc_kernel, path id 2) against float64 through lg_test_attention."""
import json
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import GPTOracle
from score_oracle import score_oracle
from test_attention_gpu import Case, _one
from util import build_gpt, cpu_state, load_golden, oracle_cfg, top2_gap

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-4


def _golden_model(name, dtype=torch.float32):
    g = load_golden(name)
    return g, build_gpt(g["cfg"], g["state_dict"], dtype)


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_forward_teacher_forced_fp32_golden(name):
    g, m = _golden_model(name)
    toks = g["tokens_cfg1.0"]
    em = g["emb_masks"].cuda() if g["emb_masks"] is not None else None
    logits, loss = m(idx=toks[:, :-1].cuda(), cond_idx=g["cond"].cuda(), targets=toks.cuda(), emb_masks=em)
    ref = g["logits_cfg1.0"].transpose(0, 1)
    assert logits.shape == ref.shape
    assert (logits.cpu() - ref).abs().max().item() <= FP32_TOL
    want = F.cross_entropy(ref.reshape(-1, ref.shape[-1]), toks.reshape(-1).long())
    assert abs(loss.item() - want.item()) <= 1e-5
    valid = torch.tensor([1.0, 0.0, 1.0])
    _, vloss = m(idx=toks[:, :-1].cuda(), cond_idx=g["cond"].cuda(), targets=toks.cuda(), emb_masks=em, valid=valid.cuda())
    per = F.cross_entropy(ref.reshape(-1, ref.shape[-1]), toks.reshape(-1).long(), reduction="none").view(3, -1)
    assert abs(vloss.item() - per[[0, 2]].mean().item()) <= 1e-5
    if name == "gpt_t2i.pt":                            # the dataset's attention mask gives the same result
        from llamagen_b200.gpt import t2i_attn_mask
        T, S = g["emb_masks"].shape[1], toks.shape[1]
        mask = t2i_attn_mask(g["emb_masks"], T + S - 1)[:, None].cuda()
        l2, loss2 = m(idx=toks[:, :-1].cuda(), cond_idx=g["cond"].cuda(), targets=toks.cuda(), mask=mask)
        assert torch.equal(l2, logits) and torch.equal(loss2, loss)
        bad = mask.clone()
        bad[0, 0, -1, -1] = False
        with pytest.raises(ValueError):
            m(idx=toks[:, :-1].cuda(), cond_idx=g["cond"].cuda(), targets=toks.cuda(), mask=bad)


@pytest.mark.parametrize("name", ["gpt_c2i.pt", "gpt_t2i.pt"])
def test_score_cfg_fp32_golden(name):
    from llamagen_b200 import score
    g, m = _golden_model(name)
    toks = g["tokens_cfg4.0"]
    em = g["emb_masks"].cuda() if g["emb_masks"] is not None else None
    nll, logits = score(m, g["cond"].cuda(), toks.cuda(), emb_masks=em, cfg_scale=4.0, return_logits=True)
    ref = g["logits_cfg4.0"].transpose(0, 1)
    assert (logits.cpu() - ref).abs().max().item() <= FP32_TOL
    want = F.cross_entropy(ref.reshape(-1, ref.shape[-1]), toks.reshape(-1).long(), reduction="none").view(toks.shape)
    assert (nll.cpu() - want).abs().max().item() <= 1e-4
    # S = 1: the condition alone
    n1 = score(m, g["cond"].cuda(), toks[:, :1].cuda(), emb_masks=em, cfg_scale=4.0)
    assert (n1.cpu() - want[:, :1]).abs().max().item() <= 1e-4


def _registry_model(name, dtype, seed, **kw):
    from llamagen_b200 import GPT_models
    torch.manual_seed(seed)
    m = GPT_models[name](**kw)
    m.output.weight.data.normal_(std=0.02)
    return m.to(device="cuda", dtype=dtype).eval()


def _parity_16(m, cond, toks, cfg_scale):
    """The calibrated-spread protocol of test_gpt_gpu._bf16_parity on scored logits: the engine may deviate from the fp32 oracle
    (same 16-bit weights) and from the like-dtype oracle by 1.5x the oracles' own 16-bit-vs-fp32 spread; arg-max agrees wherever
    the fp32 oracle's top-2 gap exceeds twice that bound. The oracles run on the GPU."""
    from llamagen_b200 import score
    cfg = oracle_cfg(m)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    ref_l, _ = score_oracle(GPTOracle({k: v.float() for k, v in sd.items()}, cfg), cond.cuda(), toks.cuda(), cfg_scale=cfg_scale)
    low_l, _ = score_oracle(GPTOracle(sd, cfg), cond.cuda(), toks.cuda(), cfg_scale=cfg_scale)
    spread_max = (low_l - ref_l).abs().max().item()
    spread_mean = (low_l - ref_l).abs().mean().item()
    tol_max, tol_mean = 1.5 * spread_max + 0.02, 1.5 * spread_mean + 0.005
    nll, logits = score(m, cond.cuda(), toks.cuda(), cfg_scale=cfg_scale, return_logits=True)
    for other in (ref_l, low_l):
        err = (logits - other).abs()
        assert err.max().item() <= tol_max, (err.max().item(), tol_max)
        assert err.mean().item() <= tol_mean, (err.mean().item(), tol_mean)
    decisive = top2_gap(ref_l) > 2 * tol_max
    assert torch.equal(logits.argmax(-1)[decisive], ref_l.argmax(-1)[decisive])
    want = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), toks.cuda().reshape(-1).long(), reduction="none")
    assert torch.allclose(nll.reshape(-1), want, atol=1e-4, rtol=1e-5)
    return spread_max


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_gpt_l_16bit_all_positions(dtype):
    """GPT-L c2i, B = 8, all 256 positions (seq 256: attn_causal_tc_kernel, hd 64), with and without CFG."""
    m = _registry_model("GPT-L", dtype, 11, block_size=256, vocab_size=16384)
    torch.manual_seed(5)
    cond, toks = torch.randint(0, 1000, (8,)), torch.randint(0, 16384, (8, 256))
    _parity_16(m, cond, toks, 1.0)
    _parity_16(m, cond, toks, 4.0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_gpt_3b_head_dim_100(dtype):
    """4 layers of the GPT-3B shape: head_dim 100 in 112-wide K / V rows, seq 576 + 1 - 1 on attn_causal_tc_kernel."""
    from llamagen_b200.gpt import ModelArgs, Transformer
    torch.manual_seed(3)
    m = Transformer(ModelArgs(n_layer=4, n_head=32, dim=3200, block_size=576, vocab_size=16384))
    m.output.weight.data.normal_(std=0.02)
    m = m.to(device="cuda", dtype=dtype).eval()
    toks = torch.randint(0, 16384, (3, 576))
    _parity_16(m, torch.tensor([1, 2, 3]), toks, 4.0)


def test_score_matches_teacher_forced_decode():
    """cfg 4.0, bf16: the one-pass logits equal generate(teacher=tokens)'s per-step logits within the bf16 protocol bound."""
    from llamagen_b200 import generate, score
    m = _registry_model("GPT-B", torch.bfloat16, 2, block_size=256, vocab_size=16384)
    torch.manual_seed(9)
    cond, toks = torch.randint(0, 1000, (4,)), torch.randint(0, 16384, (4, 40))
    spread = _parity_16(m, cond, toks, 4.0)
    _, dec = generate(m, cond.cuda(), 40, cfg_scale=4.0, sample_logits=False, return_logits=True, teacher=toks.cuda())
    _, logits = score(m, cond.cuda(), toks.cuda(), cfg_scale=4.0, return_logits=True)
    assert (logits - dec.transpose(0, 1)).abs().max().item() <= 3.0 * spread + 0.04


def test_scoring_leaves_generation_state_alone():
    from llamagen_b200 import generate, score
    m = _registry_model("GPT-B", torch.bfloat16, 4, block_size=256, vocab_size=16384)
    cond = torch.tensor([1, 7, 42, 999], device="cuda")
    a = generate(m, cond, 64, cfg_scale=4.0, seed=123)
    toks = torch.randint(0, 16384, (4, 256), device="cuda")
    n0 = score(m, cond, toks, cfg_scale=4.0)
    b = generate(m, cond, 64, cfg_scale=4.0, seed=123)
    assert torch.equal(a, b)
    m.set_kv_cache("fp8")
    n1 = score(m, cond, toks, cfg_scale=4.0)
    assert torch.equal(n0, n1), "scoring keeps K / V in the model dtype whatever the decode cache stores"


def test_chunked_scratch_matches_one_chunk(monkeypatch):
    """A scratch for one image at a time (three chunks) agrees with the whole batch in one chunk."""
    import llamagen_b200.gpt as gpt_mod
    from llamagen_b200 import score
    g, m = _golden_model("gpt_t2i.pt")
    toks = g["tokens_cfg4.0"].cuda()
    em = g["emb_masks"].cuda()
    n_all, l_all = score(m, g["cond"].cuda(), toks, emb_masks=em, cfg_scale=4.0, return_logits=True)
    monkeypatch.setattr(gpt_mod, "SCORE_SCRATCH_CAP", 1)
    m._score_ws = None
    n_one, l_one = score(m, g["cond"].cuda(), toks, emb_masks=em, cfg_scale=4.0, return_logits=True)
    assert m._score_ws.numel() < 2 * 1024 * 1024 * 8
    assert (l_all - l_one).abs().max().item() <= 1e-5 and (n_all - n_one).abs().max().item() <= 1e-5
    mb = build_gpt(g["cfg"], g["state_dict"], torch.bfloat16)
    monkeypatch.setattr(gpt_mod, "SCORE_SCRATCH_CAP", 4 << 30)
    a = score(mb, g["cond"].cuda(), toks, emb_masks=em, cfg_scale=4.0)
    monkeypatch.setattr(gpt_mod, "SCORE_SCRATCH_CAP", 1)
    mb._score_ws = None
    b = score(mb, g["cond"].cuda(), toks, emb_masks=em, cfg_scale=4.0)
    assert (a - b).abs().max().item() <= 1e-2


def test_score_cli_matches_score(tmp_path, capsys):
    from llamagen_b200 import score
    from llamagen_b200.sample.score_c2i import main
    m = _registry_model("GPT-B", torch.bfloat16, 6, block_size=256, vocab_size=1024, num_classes=10)
    ckpt = tmp_path / "gpt.pt"
    torch.save({"model": {k: v.cpu() for k, v in m.state_dict().items()}}, ckpt)
    codes, labels = tmp_path / "c" / "imagenet256_codes", tmp_path / "c" / "imagenet256_labels"
    codes.mkdir(parents=True)
    labels.mkdir(parents=True)
    rng = np.random.default_rng(1)
    toks, ys = [], []
    for i in range(5):
        x = rng.integers(0, 1024, size=(1, 2, 256), dtype=np.int64)
        np.save(codes / f"{i}.npy", x)
        np.save(labels / f"{i}.npy", np.array([i * 3 % 10]))
        toks.append(torch.from_numpy(x[0, 0]))
        ys.append(i * 3 % 10)
    main(["--code-path", str(tmp_path / "c"), "--gpt-model", "GPT-B", "--gpt-ckpt", str(ckpt), "--codebook-size", "1024",
          "--num-classes", "10", "--batch-size", "2"])
    out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    nll = score(m, torch.tensor(ys, device="cuda"), torch.stack(toks).cuda())
    assert out["images"] == 5 and out["tokens"] == 5 * 256
    assert abs(out["mean_nll"] - nll.double().mean().item()) <= 1e-5 * max(1.0, abs(out["mean_nll"]))


# ------------------------------------------------------------------------------------------- attn_causal_tc_kernel (path 2)
def _causal_cases():
    cs = []
    for dt in ("bf16", "f16"):
        for hd, hdp in ((64, 64), (128, 128), (100, 112)):
            for Tq in (129, 256, 257, 577, 1143):
                if hd == 100 and Tq not in (129, 577):
                    continue
                cs.append(Case(f"causal{Tq}_{dt}_{hd}", dt, "auto", hd, 2, 2, Tq + 7, (2, 2, 0), hdp=hdp, Tq=Tq, pos=("scalar", 0),
                               needles=Tq <= 257))
            cs.append(Case(f"causal_mask_{dt}_{hd}", dt, "auto", hd, 6, 2, 263, (2, 2, 0), hdp=hdp, Tq=256, pos=("scalar", 0),
                           mask=("ragged", 3, 120)))
        cs.append(Case(f"causal_mask_slab_{dt}", dt, "auto", 64, 4, 2, 1143, (2, 2, 0), Tq=1143, pos=("scalar", 0),
                       mask=("ragged", 2, 120), inp="slab", needles=False))
    cs.append(Case("causal_rows_over_65535_bf16", "bf16", "auto", 64, 58, 1, 1143, (2, 2, 0), Tq=1143, pos=("scalar", 0),
                   needles=False))
    return cs


CAUSAL = {c.id: c for c in _causal_cases()}


@pytest.mark.parametrize("cid", list(CAUSAL))
def test_causal_attention_call(cid):
    c = CAUSAL[cid]
    seed = zlib.crc32(cid.encode())
    worst = _one(c, "wide", None, seed)[2]
    needles = [("abs", j) for j in (0, 63, 64, 65, 127, 128, 129)] + [("rel", d) for d in (0, 1, 64)] if c.needles else [("rel", 0)]
    if c.mask:
        needles += [("abs", 119), ("abs", 120)]
    for i, nd in enumerate(needles):
        worst = max(worst, _one(c, "needle", nd, seed + 1 + i)[2])
    if c.hdp > c.hd:
        a = _one(c, "needle", ("rel", 1), seed + 99, pad="zero")[0]
        b = _one(c, "needle", ("rel", 1), seed + 99, pad="garbage")[0]
        assert torch.equal(a, b)
    print(f"[{cid}] max |out - ref| / absO {worst:.3g}")
