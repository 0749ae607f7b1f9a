"""CPU: the fp16 oracle against the reference's fp16 outputs (tests/golden/reference_fp16.pt, written by
tests/golden/make_reference_fp16.py), and the fp16 plumbing of the C-ABI and the samplers that runs without a GPU."""
import ctypes
import os
import re

import torch

from oracle import GPTOracle
from util import load_golden, seeded_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(case):
    sd = {k: v.to(torch.float16) for k, v in seeded_state_dict(case["shapes"], case["seed"]).items()}
    return GPTOracle(sd, case["cfg"])


def test_fp16_oracle_reproduces_reference_greedy_tokens():
    g = load_golden("reference_fp16.pt")
    for model_type in ("c2i", "t2i"):
        case = g[model_type]
        toks, _ = _oracle(case).generate(case["cond"], 16, emb_masks=case["emb_masks"], cfg_scale=3.0, sample_logits=False)
        assert torch.equal(toks.to(case["tokens"].dtype), case["tokens"]), model_type


def test_fp16_oracle_reproduces_reference_prefill_logits():
    g = load_golden("reference_fp16.pt")
    for model_type in ("c2i", "t2i"):
        case = g[model_type]
        orc = _oracle(case)
        B, T = case["cond"].shape[0], case["cfg"]["cls_token_num"]
        orc.setup(B, T + 16)
        with torch.no_grad():
            logits = orc.forward(None, case["cond"], torch.arange(0, T))
        assert torch.equal(logits, case["prefill_logits"]), model_type


def test_f16_dtype_code_matches_header():
    from llamagen_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "llamagen_b200.h")).read()
    assert re.search(r"LG_DTYPE_F16\s*=\s*2\b", hdr)
    assert _lib.LG_DTYPE_F16 == 2
    assert _lib.dtype_code(torch.float16) == _lib.LG_DTYPE_F16
    assert _lib.dtype_code(torch.bfloat16) == _lib.LG_DTYPE_BF16 and _lib.dtype_code(torch.float32) == _lib.LG_DTYPE_F32
    try:
        _lib.dtype_code(torch.float64)
    except _lib.LgError:
        pass
    else:
        raise AssertionError("float64 must be rejected")


def test_engine_create_accepts_f16_and_rejects_unknown_dtype():
    from llamagen_b200 import _lib
    lib = _lib.load()
    cfg = _lib.ModelCfg(2, 2, 128, 256, 512, 1, 16, 10, 64, _lib.LG_MODEL_C2I, _lib.LG_DTYPE_F16, 1e-5)
    h = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == 0
    try:
        assert lib.lg_engine_finalize(h) < 0
        assert b"missing weight" in lib.lg_last_error()
    finally:
        lib.lg_engine_destroy(h)
    cfg.dtype = 3
    h2 = ctypes.c_void_p()
    assert lib.lg_engine_create(ctypes.byref(cfg), 0, ctypes.byref(h2)) < 0
    assert b"unsupported dtype" in lib.lg_last_error()


def test_load_gpt_fp16_on_cpu():
    from llamagen_b200.sample import sample_c2i
    from llamagen_b200.sample.common import load_gpt
    args = sample_c2i.build_parser().parse_args(["--gpt-model", "GPT-B", "--precision", "fp16"])
    m = load_gpt(args, "cpu", 16)
    assert m.tok_embeddings.weight.dtype == torch.float16
