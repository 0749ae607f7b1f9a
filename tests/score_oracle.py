"""Teacher-forced scoring oracle (TEST INFRASTRUCTURE ONLY): GPTOracle.forward over the condition, then ONE multi-token forward of
the token embeddings at positions T .. T + S - 2 through the same KV cache (the inference branch of gpt.py:341-368 with the causal
mask rows of those positions), CFG-mixed as generate.py:79-82. Logits [B, S, V] of positions T - 1 .. T + S - 2."""
import torch
import torch.nn.functional as F

from oracle import GPTOracle, cfg_mix_oracle


@torch.no_grad()
def score_oracle(orc: GPTOracle, cond, tokens, emb_masks=None, cfg_scale=1.0):
    """tokens [B, S] (int). Returns (logits fp32 [B, S, V], nll fp32 [B, S])."""
    c = orc.cfg
    B, S = tokens.shape
    use_cfg = cfg_scale > 1.0
    if c.model_type == "c2i":
        T = 1
        cond_all = torch.cat([cond, torch.ones_like(cond) * c.num_classes]) if use_cfg else cond
    else:
        T = cond.shape[1]
        null = torch.zeros_like(cond) + orc.sd["cls_embedding.uncond_embedding"]
        cond_all = torch.cat([cond, null]) if use_cfg else cond
    rows = 2 * B if use_cfg else B
    orc.setup(rows, T + S)
    if emb_masks is not None:
        orc.apply_emb_masks(torch.cat([emb_masks, emb_masks]) if use_cfg else emb_masks, T)
    orc.math_sdp = False
    out = [orc.forward(None, cond_all, torch.arange(0, T, device=orc.device))[:, -1:]]
    if S > 1:
        idx = tokens[:, :-1].to(orc.device).long()
        idx = torch.cat([idx, idx]) if use_cfg else idx
        out.append(orc.forward(idx, None, torch.arange(T, T + S - 1, device=orc.device)))
    logits = torch.cat(out, dim=1)
    if use_cfg:
        logits = cfg_mix_oracle(logits, cfg_scale)
    nll = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), tokens.reshape(-1).long().to(logits.device),
                          reduction="none").view(B, S)
    return logits, nll
