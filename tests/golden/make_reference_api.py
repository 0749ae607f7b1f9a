"""Record what the live-reference tests (tests/test_oracle_vs_reference.py, the CLI flag test) compare against, by running the
reference LlamaGen checkout given as the first argument:  python tests/golden/make_reference_api.py <llamagen checkout>
Weights come from tests/util.py:seeded_state_dict, so the tests rebuild the same models without the reference."""
import os, re, sys, json
import torch
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.dirname(HERE))
from util import seeded_state_dict
from autoregressive.models.generate import generate
from autoregressive.models.gpt import ModelArgs, Transformer, precompute_freqs_cis_2d, GPT_models as RefGPT
from tokenizer.tokenizer_image.vq_model import VQ_models as RefVQ
out = {"generate": {}, "rope": {}, "cli_flags": {}, "gpt_registry": {}, "vq_registry": {}}
for model_type, cls in (("c2i", 1), ("t2i", 120)):
    for dtype in (torch.float32, torch.bfloat16):
        torch.manual_seed(11)
        cfg = dict(n_layer=2, n_head=2, dim=128, vocab_size=256, block_size=16, cls_token_num=cls, model_type=model_type,
                   num_classes=7, caption_dim=64, norm_eps=1e-5, rope_base=10000)
        m = Transformer(ModelArgs(**cfg)).eval()
        shapes = {k: list(v.shape) for k, v in m.state_dict().items() if v.is_floating_point() and not k.startswith("freqs")}
        sd = seeded_state_dict(shapes, 11)
        m.load_state_dict(sd, strict=False)
        m = m.to(dtype)
        B = 2
        if model_type == "c2i":
            cond, em = torch.tensor([3, 6]), None
        else:
            em = torch.zeros(B, cls); em[0, -5:] = 1; em[1, -77:] = 1
            cond = (torch.randn(B, cls, 64) * em[:, :, None]).to(dtype)
        ref = generate(m, cond, 16, emb_masks=em, cfg_scale=3.0, temperature=1.0, top_k=0, top_p=1.0, sample_logits=False)
        out["generate"][f"{model_type}_{str(dtype)[6:]}"] = dict(cfg=cfg, shapes=shapes, seed=11, cond=cond, emb_masks=em, tokens=ref)
for grid, hd, cls in ((16, 64, 1), (24, 100, 1), (32, 64, 120)):
    out["rope"][(grid, hd, cls)] = precompute_freqs_cis_2d(grid, hd, 10000, cls)
for script in ("sample_c2i", "sample_t2i", "sample_c2i_ddp"):
    out["cli_flags"][script] = sorted(set(re.findall(r'add_argument\(\s*"(--[a-z0-9\-]+)"', open(os.path.join(sys.argv[1], "autoregressive", "sample", f"{script}.py")).read())))
for kw in (dict(model_type="c2i", cls_token_num=1, block_size=256), dict(model_type="t2i", cls_token_num=120, block_size=256)):
    out["gpt_registry"][kw["model_type"]] = {k: tuple(v.shape) for k, v in RefGPT["GPT-B"](**kw).state_dict().items()}
out["gpt_names"] = sorted(RefGPT)
for name in RefVQ:
    out["vq_registry"][name] = {k: tuple(v.shape) for k, v in RefVQ[name](codebook_size=16384, codebook_embed_dim=8).state_dict().items()}
import hashlib
import numpy as np
import torch.nn as nn
from PIL import Image
from dataset.augmentation import center_crop_arr
from tokenizer.tokenizer_image.vq_model import Decoder, Encoder, VectorQuantizer


def float_shapes(sd):
    return {k: list(v.shape) for k, v in sd.items() if v.is_floating_point()}


# VQ decode: Decoder + post_quant_conv + codebook lookup composed as VQModel.decode_code does
torch.manual_seed(5)
dec = Decoder(z_channels=32, ch=32, ch_mult=(1, 2, 2)).eval()
quant = VectorQuantizer(128, 8, 0.25, 0.0, True, True).eval()
pqc = nn.Conv2d(8, 32, 1).eval()
sd = {"decoder." + k: v for k, v in dec.state_dict().items()}
sd.update({"quantize.embedding.weight": quant.embedding.weight.data, "post_quant_conv.weight": pqc.weight.data,
           "post_quant_conv.bias": pqc.bias.data})
shapes = float_shapes(sd)
w = seeded_state_dict(shapes, 5, fan_in=True)
dec.load_state_dict({k[len("decoder."):]: v for k, v in w.items() if k.startswith("decoder.")}, strict=False)
quant.embedding.weight.data.copy_(w["quantize.embedding.weight"])
pqc.weight.data.copy_(w["post_quant_conv.weight"]); pqc.bias.data.copy_(w["post_quant_conv.bias"])
codes = torch.randint(0, 128, (1, 9))
with torch.no_grad():
    pix = dec(pqc(quant.get_codebook_entry(codes, [1, 8, 3, 3], True)))
out["vq_decode"] = dict(shapes=shapes, seed=5, codes=codes, pixels=pix.clone())

# VQ encode: Encoder + quant_conv + VectorQuantizer composed as VQModel.encode does
torch.manual_seed(6)
enc = Encoder(ch=32, ch_mult=(1, 2, 2), z_channels=32).eval()
quant = VectorQuantizer(128, 8, 0.25, 0.0, True, True).eval()
qc = nn.Conv2d(32, 8, 1).eval()
sd = {"encoder." + k: v for k, v in enc.state_dict().items()}
sd.update({"quantize.embedding.weight": quant.embedding.weight.data, "quant_conv.weight": qc.weight.data,
           "quant_conv.bias": qc.bias.data})
shapes = float_shapes(sd)
w = seeded_state_dict(shapes, 6, fan_in=True)
enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=False)
quant.embedding.weight.data.copy_(w["quantize.embedding.weight"])
qc.weight.data.copy_(w["quant_conv.weight"]); qc.bias.data.copy_(w["quant_conv.bias"])
x = torch.rand(1, 3, 24, 16) * 2 - 1
with torch.no_grad():
    zq, _, info = quant(qc(enc(x)))
out["vq_encode"] = dict(shapes=shapes, seed=6, x=x, quant=zq.clone(), indices=info[2].clone())

# center_crop_arr (dataset/augmentation.py) on seeded random images: sha256 of each crop's bytes
rng = np.random.default_rng(1)
crops = {}
for shape in [(300, 420), (1100, 900), (256, 256), (513, 2000)]:
    im = Image.fromarray(rng.integers(0, 255, (*shape, 3), dtype=np.uint8))
    for s in (256, 384):
        a = np.array(center_crop_arr(im, s))
        crops[(shape, s)] = (a.shape, hashlib.sha256(a.tobytes()).hexdigest())
out["center_crop"] = crops

torch.save(out, os.path.join(HERE, "reference_api.pt"))
print(os.path.getsize(os.path.join(HERE, "reference_api.pt")))
