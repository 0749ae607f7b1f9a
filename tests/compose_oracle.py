"""Composable-guidance oracle (TEST INFRASTRUCTURE ONLY): the semantics of `generate(..., cond_weights=)`.

GPTOracle's forward and sampling with K conditions per image. Image j runs K conditional rows (its conditions) and ONE unconditional
row (the null condition, or the image's negative), and every token is drawn from

    x = u + d,   d = w_1 (c_1 - u) + w_2 (c_2 - u) + ... + w_K (c_K - u)   (left to right, in the logits' dtype)

The unconditional row attends with the emb-mask of condition 1, or with the negative's mask. cfg_interval (K = 1 only) drops the mix
as GPTOracle.generate does, leaving c_1. The drawn token feeds all K + 1 rows of its image."""
import torch

from oracle import GPTOracle, sample_oracle


def compose_mix_oracle(c, u, w):
    """c [B, K, V], u [B, V], w [B, K] -> x [B, V]: u + sum_i w_i (c_i - u), accumulated left to right."""
    d = (c[:, 0] - u) * w[:, :1]
    for i in range(1, c.shape[1]):
        d = d + (c[:, i] - u) * w[:, i:i + 1]
    return u + d


@torch.no_grad()
def compose_oracle(orc: GPTOracle, cond, weights, max_new_tokens, emb_masks=None, negative=None, negative_emb_masks=None, prefix=None,
                   cfg_interval=-1, temperature=1.0, top_k=0, top_p=1.0, sample_logits=True, generator=None):
    """cond: c2i int [B, K] class ids, t2i [B, K, T, C]; weights [K] or [B, K]; emb_masks [B, K, T] or None; negative [1 or B, T, C] and
    negative_emb_masks [1 or B, T] (t2i); prefix [B, P]: tokens 0 .. P - 1 of every image (given, fed before the first draw). Returns
    (tokens int32 [B, S], mixed logits [S, B, V]; rows k < P of a prefix are zero)."""
    c2i = orc.cfg.model_type == "c2i"
    B, K = cond.shape[0], cond.shape[1]
    assert K == 1 or cfg_interval == -1
    dev = orc.device
    T = 1 if c2i else cond.shape[2]
    R = B * K
    if c2i:
        rows = torch.cat([cond.reshape(R), torch.full((B,), orc.cfg.num_classes, dtype=cond.dtype)]).to(dev)
    else:
        null = torch.zeros_like(cond[:, 0]) + orc.sd["cls_embedding.uncond_embedding"].to(cond.dtype)
        un = null if negative is None else negative.to(cond.dtype).expand(B, T, cond.shape[3])
        rows = torch.cat([cond.reshape(R, T, cond.shape[3]), un]).to(dev)
    if not c2i and (emb_masks is not None or negative is not None):
        ones = torch.ones(B, K, T)
        em = ones if emb_masks is None else emb_masks.float()
        um = em[:, 0] if negative_emb_masks is None else negative_emb_masks.float().expand(B, T)
        if negative is not None and negative_emb_masks is None:
            um = torch.ones(B, T)
        masks = torch.cat([em.reshape(R, T), um]).to(dev)
    else:
        masks = None
    w = torch.as_tensor(weights).to(dev).expand(B, K)
    P = 0 if prefix is None else prefix.shape[1]
    orc.setup(R + B, T + max_new_tokens)
    if masks is not None:
        orc.apply_emb_masks(masks, T)
    sk = dict(temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits, generator=generator)

    def feed(tok):   # image j's token to its K conditional rows and its unconditional row
        return torch.cat([tok.repeat_interleave(K, 0), tok]).view(-1, 1)

    orc.math_sdp = False
    logits = orc.forward(None, rows, torch.arange(0, T, device=dev))
    orc.math_sdp = True
    pos = torch.tensor([T], device=dev, dtype=torch.int)
    toks, mixed_all = [], []
    for k in range(max_new_tokens):
        if k < P:
            tok = prefix[:, k:k + 1].to(dev).long()
            toks.append(tok)
            mixed_all.append(torch.zeros(B, logits.shape[-1], dtype=logits.dtype, device=dev))
        else:
            last = logits[:, -1]
            c, u = last[:R].view(B, K, -1), last[R:]
            mix = not (cfg_interval > -1 and k - 1 > cfg_interval)          # generate.py:113-114 by token index
            mixed = compose_mix_oracle(c, u, w.to(last.dtype)) if mix else c[:, 0]
            mixed_all.append(mixed.clone())
            tok = sample_oracle(mixed, **sk)[0]
            toks.append(tok)
        if k == max_new_tokens - 1:
            break
        logits = orc.forward(feed(tok), None, pos)
        pos += 1
    return torch.cat(toks, dim=1).to(torch.int32), torch.stack(mixed_all)
