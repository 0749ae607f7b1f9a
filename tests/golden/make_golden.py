"""Generate golden vectors by RUNNING THE REFERENCE (a LlamaGen checkout) on tiny seeded models.

Run:  python tests/golden/make_golden.py <llamagen checkout>
Outputs (committed, small):
  tests/golden/gpt_c2i.pt  gpt_t2i.pt   : state_dict + inputs + reference generate() greedy tokens and logits
  tests/golden/vq_tiny.pt               : state_dict + codes + reference decode_code pixels + argmin indices
  tests/golden/vq_enc_tiny.pt           : encoder state_dict + image + reference z / quant / indices (VQModel.encode)
  tests/golden/sampling.pt              : logits + reference top_k_top_p_filtering / sample outputs
Every tensor here is an output of the unmodified reference code; nothing is copied from its source.
"""
import os
import sys

import torch

sys.path.insert(0, sys.argv[1])
HERE = os.path.dirname(os.path.abspath(__file__))

from autoregressive.models.generate import generate, sample, top_k_top_p_filtering  # noqa: E402
from autoregressive.models.gpt import ModelArgs, Transformer  # noqa: E402
from tokenizer.tokenizer_image.vq_model import ModelArgs as VQArgs  # noqa: E402
from tokenizer.tokenizer_image.vq_model import VQModel  # noqa: E402


def ref_step_logits(model, cond, S, emb_masks, cfg_scale, tokens):
    """Teacher-forced per-step mixed logits from the reference model (fp32): replays generate()'s model
    calls with hooks-free plain forward calls on the same caches."""
    import autoregressive.models.generate as G
    logs = []
    orig = G.sample

    def spy(logits, **kw):
        logs.append(logits[:, -1, :].clone())
        return orig(logits, **kw)

    G.sample = spy
    try:
        out = generate(model, cond, S, emb_masks=emb_masks, cfg_scale=cfg_scale, temperature=1.0, top_k=0,
                       top_p=1.0, sample_logits=False)
    finally:
        G.sample = orig
    assert torch.equal(out, tokens)
    return torch.stack(logs)


def gpt_case(model_type, seed):
    torch.manual_seed(seed)
    cls = 1 if model_type == "c2i" else 120
    cfg = dict(n_layer=2, n_head=2, dim=128, vocab_size=512, block_size=16, cls_token_num=cls, model_type=model_type,
               num_classes=10, caption_dim=64, norm_eps=1e-5, rope_base=10000)
    model = Transformer(ModelArgs(**cfg)).eval()
    model.output.weight.data.normal_(std=0.02)          # SURVEY G1: the stock init zeroes the head
    B, S = 3, 16
    if model_type == "c2i":
        cond, em = torch.tensor([1, 5, 9]), None
    else:
        em = torch.zeros(B, cls)
        for b, n in enumerate([7, 30, 120]):
            em[b, -n:] = 1
        cond = torch.randn(B, cls, 64) * em[:, :, None]
    case = dict(cfg=cfg, state_dict={k: v.clone() for k, v in model.state_dict().items()}, cond=cond, emb_masks=em, S=S)
    for cfg_scale in (1.0, 4.0):
        toks = generate(model, cond, S, emb_masks=em, cfg_scale=cfg_scale, temperature=1.0, top_k=0, top_p=1.0,
                        sample_logits=False)
        case[f"tokens_cfg{cfg_scale}"] = toks.clone()
        case[f"logits_cfg{cfg_scale}"] = ref_step_logits(model, cond, S, em, cfg_scale, toks)
    # cfg_interval variant (generate.py:113-114)
    case["tokens_cfg4.0_int3"] = generate(model, cond, S, emb_masks=em, cfg_scale=4.0, cfg_interval=3, temperature=1.0,
                                          top_k=0, top_p=1.0, sample_logits=False).clone()
    return case


def vq_case(seed):
    """Tiny decoder (ch=32, ch_mult=(1,2), z_channels=32) assembled from the reference's own classes exactly as
    VQModel.decode_code composes them (vq_model.py:47-55); VQModel itself hard-codes ch=128 (35 MB of weights)."""
    import torch.nn as nn
    from tokenizer.tokenizer_image.vq_model import Decoder, VectorQuantizer
    torch.manual_seed(seed)
    dec = Decoder(z_channels=32, ch=32, ch_mult=(1, 2)).eval()
    quant = VectorQuantizer(64, 8, 0.25, 0.0, True, True).eval()
    pqc = nn.Conv2d(8, 32, 1).eval()
    sd = {"decoder." + k: v.clone() for k, v in dec.state_dict().items()}
    sd["quantize.embedding.weight"] = quant.embedding.weight.data.clone()
    sd["post_quant_conv.weight"] = pqc.weight.data.clone()
    sd["post_quant_conv.bias"] = pqc.bias.data.clone()
    codes = torch.randint(0, 64, (2, 16))
    with torch.no_grad():
        pix = dec(pqc(quant.get_codebook_entry(codes, [2, 8, 4, 4], True)))
        z = torch.randn(2, 8, 4, 4)
        idx = quant(z)[2][2]
    return dict(ch=32, z_channels=32, ch_mult=[1, 2], state_dict=sd, codes=codes, pixels=pix.clone(), z=z,
                argmin=idx.clone())


def vq_enc_case(seed):
    """Tiny encoder (ch=32, ch_mult=(1,2), z_channels=32) + quant_conv + quantizer composed as VQModel.encode does
    (vq_model.py:41-45)."""
    import torch.nn as nn
    from tokenizer.tokenizer_image.vq_model import Encoder, VectorQuantizer
    torch.manual_seed(seed)
    enc = Encoder(ch=32, ch_mult=(1, 2), z_channels=32).eval()
    quant = VectorQuantizer(64, 8, 0.25, 0.0, True, True).eval()
    qc = nn.Conv2d(32, 8, 1).eval()
    sd = {"encoder." + k: v.clone() for k, v in enc.state_dict().items()}
    sd["quantize.embedding.weight"] = quant.embedding.weight.data.clone()
    sd["quant_conv.weight"] = qc.weight.data.clone()
    sd["quant_conv.bias"] = qc.bias.data.clone()
    x = torch.rand(2, 3, 16, 16) * 2 - 1
    with torch.no_grad():
        z = qc(enc(x))
        zq, _, info = quant(z)
    return dict(ch=32, z_channels=32, ch_mult=[1, 2], state_dict=sd, x=x, z=z.clone(), quant=zq.clone(),
                indices=info[2].clone())


def save_golden(case, name, part_bytes=900 * 1024):
    """torch.save `case` as HERE/name; a state_dict that would push the file past 1 MB goes to name.sd<i>.pt parts of at
    most `part_bytes` tensor bytes each (tests/util.py:load_golden joins them)."""
    stem = os.path.join(HERE, name[:-3])
    sd = case.get("state_dict")
    if sd is not None and sum(t.numel() * t.element_size() for t in sd.values()) > part_bytes:
        parts, cur, size = [], {}, 0
        for k, t in sd.items():
            nb = t.numel() * t.element_size()
            if cur and size + nb > part_bytes:
                parts.append(cur)
                cur, size = {}, 0
            cur[k] = t
            size += nb
        parts.append(cur)
        for i, part in enumerate(parts):
            torch.save(part, f"{stem}.sd{i}.pt")
        case = dict(case, state_dict=None, state_dict_parts=len(parts))
    torch.save(case, stem + ".pt")


def sampling_case(seed):
    torch.manual_seed(seed)
    V = 1024
    logits = torch.randn(4, V) * 2.5
    logits[1, 10] = logits[1, 20] = logits[1].topk(5).values[-1]      # tie at the k=5 boundary (SURVEY G8)
    out = dict(logits=logits)
    for k, p in ((0, 1.0), (5, 1.0), (50, 1.0), (V, 1.0), (0, 0.9), (100, 0.5), (1, 1.0)):
        out[f"filtered_k{k}_p{p}"] = top_k_top_p_filtering(logits.clone(), top_k=k, top_p=p)
        idx, probs = sample(logits[:, None, :].clone(), temperature=0.7, top_k=k, top_p=p, sample_logits=False)
        out[f"greedy_k{k}_p{p}"] = idx.clone()
        out[f"probs_k{k}_p{p}"] = probs.clone()
    return out


if __name__ == "__main__":
    save_golden(gpt_case("c2i", 0), "gpt_c2i.pt")
    save_golden(gpt_case("t2i", 1), "gpt_t2i.pt")
    save_golden(vq_case(2), "vq_tiny.pt")
    save_golden(sampling_case(3), "sampling.pt")
    save_golden(vq_enc_case(4), "vq_enc_tiny.pt")
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".pt"):
            print(f, os.path.getsize(os.path.join(HERE, f)) // 1024, "KiB")
