"""Record the reference's fp16 sampling outputs that tests/test_fp16_reference.py compares the fp16 oracle against, by running
the reference LlamaGen checkout given as the first argument:  python tests/golden/make_reference_fp16.py <llamagen checkout>
Same tiny c2i / t2i models and seeded weights as make_reference_api.py, cast to fp16 (the samplers' --precision fp16):
greedy generate() tokens at cfg 3.0, and the prefill logits m(None, cond, input_pos) of the condition rows."""
import os, sys
import torch
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.dirname(HERE))
from util import seeded_state_dict
from autoregressive.models.generate import generate
from autoregressive.models.gpt import ModelArgs, Transformer
out = {}
for model_type, cls in (("c2i", 1), ("t2i", 120)):
    torch.manual_seed(11)
    cfg = dict(n_layer=2, n_head=2, dim=128, vocab_size=256, block_size=16, cls_token_num=cls, model_type=model_type,
               num_classes=7, caption_dim=64, norm_eps=1e-5, rope_base=10000)
    m = Transformer(ModelArgs(**cfg)).eval()
    shapes = {k: list(v.shape) for k, v in m.state_dict().items() if v.is_floating_point() and not k.startswith("freqs")}
    m.load_state_dict(seeded_state_dict(shapes, 11), strict=False)
    m = m.to(torch.float16)
    B = 2
    if model_type == "c2i":
        cond, em = torch.tensor([3, 6]), None
    else:
        em = torch.zeros(B, cls); em[0, -5:] = 1; em[1, -77:] = 1
        cond = (torch.randn(B, cls, 64) * em[:, :, None]).to(torch.float16)
    with torch.no_grad():
        tokens = generate(m, cond, 16, emb_masks=em, cfg_scale=3.0, temperature=1.0, top_k=0, top_p=1.0, sample_logits=False)
        T = 1 if model_type == "c2i" else cls
        m.setup_caches(max_batch_size=B, max_seq_length=T + 16, dtype=torch.float16)
        prefill, _ = m(None, cond, input_pos=torch.arange(0, T))
    out[model_type] = dict(cfg=cfg, shapes=shapes, seed=11, cond=cond, emb_masks=em, tokens=tokens,
                           prefill_logits=prefill.float().contiguous())
torch.save(out, os.path.join(HERE, "reference_fp16.pt"))
