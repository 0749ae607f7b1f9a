"""CPU: the oracle against outputs of the reference LlamaGen code recorded in tests/golden/reference_api.pt
(tests/golden/make_reference_api.py): greedy generate() tokens, the 2-D RoPE table, the model registries, VQ
decode / encode of a tiny model, and the sample scripts' center crop."""
import pytest
import torch

from oracle import GPTOracle, VQOracle, rope_table_2d_oracle
from util import load_golden, seeded_state_dict


@pytest.fixture(scope="module")
def ref():
    return load_golden("reference_api.pt")


@pytest.mark.parametrize("model_type,cls", [("c2i", 1), ("t2i", 120)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_generate_matches_live_reference(ref, model_type, cls, dtype):
    case = ref["generate"][f"{model_type}_{str(dtype)[6:]}"]
    assert case["cfg"]["cls_token_num"] == cls
    sd = {k: v.to(dtype) for k, v in seeded_state_dict(case["shapes"], case["seed"]).items()}
    toks, _ = GPTOracle(sd, case["cfg"]).generate(case["cond"], 16, emb_masks=case["emb_masks"], cfg_scale=3.0, sample_logits=False)
    assert torch.equal(case["tokens"], toks)


def test_rope_table_matches_live_reference(ref):
    from llamagen_b200.gpt import rope_table_2d
    for (grid, hd, cls), table in ref["rope"].items():
        assert torch.equal(table, rope_table_2d_oracle(grid, hd, 10000, cls))
        assert torch.equal(table, rope_table_2d(grid, hd, 10000, cls))


def test_registry_matches_live_reference(ref):
    """Same keys, same parameter names and shapes as the reference registries (drop-in boundary §8b)."""
    from llamagen_b200 import GPT_models
    assert set(ref["gpt_names"]) == set(GPT_models)
    for kw in (dict(model_type="c2i", cls_token_num=1, block_size=256), dict(model_type="t2i", cls_token_num=120, block_size=256)):
        b = GPT_models["GPT-B"](**kw).state_dict()
        assert ref["gpt_registry"][kw["model_type"]] == {k: tuple(v.shape) for k, v in b.items()}


def test_vq_registry_matches_live_reference(ref):
    from llamagen_b200 import VQ_models
    assert set(ref["vq_registry"]) == set(VQ_models)
    for name, shapes in ref["vq_registry"].items():
        b = VQ_models[name](codebook_size=16384, codebook_embed_dim=8).state_dict()
        assert shapes == {k: tuple(v.shape) for k, v in b.items()}


def test_vq_decode_matches_live_reference(ref):
    case = ref["vq_decode"]
    sd = seeded_state_dict(case["shapes"], case["seed"], fan_in=True)
    assert torch.equal(case["pixels"], VQOracle(sd, ch_mult=(1, 2, 2)).decode_code(case["codes"], [1, 8, 3, 3]))


def test_vq_encode_matches_live_reference(ref):
    case = ref["vq_encode"]
    sd = seeded_state_dict(case["shapes"], case["seed"], fan_in=True)
    q, idx = VQOracle(sd, ch_mult=(1, 2, 2)).encode(case["x"])
    assert torch.equal(idx, case["indices"]) and torch.equal(q, case["quant"])


def test_center_crop_matches_live_reference(ref):
    import hashlib

    import numpy as np
    from PIL import Image
    from llamagen_b200.sample.vq_demo import center_crop
    rng = np.random.default_rng(1)
    for shape in [(300, 420), (1100, 900), (256, 256), (513, 2000)]:
        im = Image.fromarray(rng.integers(0, 255, (*shape, 3), dtype=np.uint8))
        for s in (256, 384):
            a = np.array(center_crop(im, s))
            assert (a.shape, hashlib.sha256(a.tobytes()).hexdigest()) == ref["center_crop"][(shape, s)]
