"""Negative-prompt oracle (TEST INFRASTRUCTURE ONLY): the semantics of `generate(..., negative_cond=, negative_emb_masks=)`.

GPTOracle.generate (generate.py:126-176) with one substitution: the unconditional rows take the negative's features instead of
`zeros_like(cond) + uncond_embedding`, and the emb-mask of those rows is the negative's, `cat([emb_masks, negative_emb_masks])`
(a missing mask counts as all ones). The forward, the CFG mix, cfg_interval and the sampling are GPTOracle's."""
import torch

from oracle import GPTOracle, cfg_mix_oracle, sample_oracle


@torch.no_grad()
def negative_oracle(orc: GPTOracle, cond, negative, max_new_tokens, emb_masks=None, negative_emb_masks=None, cfg_scale=4.0,
                    cfg_interval=-1, temperature=1.0, top_k=0, top_p=1.0, sample_logits=True, teacher=None, generator=None):
    """cond [B, T, C], negative [1 or B, T, C] (prepared as cond is). Returns (tokens int32 [B, S], mixed logits fp32 [S, B, V])."""
    assert orc.cfg.model_type == "t2i" and cfg_scale > 1.0
    B, T = cond.shape[0], cond.shape[1]
    neg = negative.to(cond.device, cond.dtype).expand(B, *cond.shape[1:])
    ones = torch.ones(B, T, device=cond.device)
    em = ones if emb_masks is None else emb_masks.to(cond.device).float()
    nm = ones if negative_emb_masks is None else negative_emb_masks.to(cond.device).float().expand(B, T)
    orc.setup(2 * B, T + max_new_tokens)
    orc.apply_emb_masks(torch.cat([em, nm]), T)
    sk = dict(temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits, generator=generator)
    orc.math_sdp = False
    logits = orc.forward(None, torch.cat([cond, neg]), torch.arange(0, T, device=orc.device))
    orc.math_sdp = True
    toks, mixed_all = [], []
    pos = torch.tensor([T], device=orc.device, dtype=torch.int)
    for i in range(max_new_tokens):
        cfg_flag = not (cfg_interval > -1 and i - 1 > cfg_interval)       # generate.py:113-114: step i >= 1 decodes after index i - 1
        mixed = cfg_mix_oracle(logits, cfg_scale) if cfg_flag else logits[: logits.shape[0] // 2]
        mixed_all.append(mixed[:, -1].clone())
        nxt = sample_oracle(mixed[:, -1], **sk)[0]
        toks.append(nxt)
        if i == max_new_tokens - 1:
            break
        cur = nxt if teacher is None else teacher[:, i:i + 1].to(nxt.dtype)
        logits = orc.forward(torch.cat([cur, cur]).view(-1, 1), None, pos)
        pos += 1
    return torch.cat(toks, dim=1).to(torch.int32), torch.stack(mixed_all)
