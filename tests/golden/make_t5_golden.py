"""Record what tests/test_t5.py and tests/test_t5_gpu.py compare the T5 encoder against, on a machine with `transformers`:
    python tests/golden/make_t5_golden.py
A seeded tiny T5EncoderModel (gated-gelu, 2 layers, 2 heads x d_kv 64, d_model 128, d_ff 384, vocab 256; weights from
tests/util.py:seeded_state_dict) encodes B = 3 captions of T = 160 tokens with valid lengths 1, 57 and 160 (so relative distances
past max_distance 128 occur), in fp32 and bf16 on the CPU. Also stored: transformers' bucket of every relative position
-511..511 (the table of any T <= 512 is its middle 2T - 1 entries)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from util import seeded_state_dict  # noqa: E402
from transformers import T5Config, T5EncoderModel  # noqa: E402
from transformers.models.t5.modeling_t5 import T5Attention  # noqa: E402

CFG = dict(vocab_size=256, d_model=128, d_kv=64, d_ff=384, num_layers=2, num_heads=2, feed_forward_proj="gated-gelu",
           relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6, dropout_rate=0.0)
SEED, B, T, LENS = 23, 3, 160, (1, 57, 160)

model = T5EncoderModel(T5Config(**CFG)).eval()
shapes = {k: list(v.shape) for k, v in model.state_dict().items() if k != "encoder.embed_tokens.weight"}
sd = seeded_state_dict(shapes, SEED)
missing, unexpected = model.load_state_dict(sd, strict=False)
assert not unexpected and set(missing) <= {"encoder.embed_tokens.weight"}, (missing, unexpected)
g = torch.Generator().manual_seed(SEED)
ids = torch.randint(0, CFG["vocab_size"], (B, T), generator=g)
mask = (torch.arange(T)[None, :] < torch.tensor(LENS)[:, None]).long()
ids = ids * mask   # padding id 0, as the tokenizer pads
out = {}
with torch.no_grad():
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        out[name] = model.to(dt)(input_ids=ids, attention_mask=mask).last_hidden_state.float()
rel = torch.arange(-511, 512)
buckets = T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=32, max_distance=128).to(torch.int32)
keys = sorted(sd)
parts = [keys[i::3] for i in range(3)]
for i, ks in enumerate(parts):
    torch.save({k: sd[k] for k in ks}, os.path.join(HERE, f"t5_tiny.sd{i}.pt"))
torch.save(dict(cfg=CFG, seed=SEED, ids=ids, mask=mask, hidden_fp32=out["fp32"], hidden_bf16=out["bf16"].to(torch.bfloat16),
                buckets=buckets, state_dict_parts=len(parts)), os.path.join(HERE, "t5_tiny.pt"))
print({k: v.shape for k, v in out.items()})
