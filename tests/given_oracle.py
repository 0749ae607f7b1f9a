"""Inpainting oracle (TEST INFRASTRUCTURE ONLY): the semantics of `generate(..., given=tokens, given_mask=mask)`.

It extends prefix_oracle's semantics to any mask: GPTOracle.forward runs the condition and the leading run of tokens given to every
image at positions 0 .. T + P - 1 in ONE call, then the oracle goes position by position: at token k >= P, image b takes given[b, k]
where mask[b, k] is True and otherwise draws from the CFG-mixed logits (cfg_interval by token index), and the token is fed at
position T + k. Masks may differ per image. A negative prompt replaces the null condition of the unconditional rows, with its
emb-mask, as negative_oracle does."""
import torch

from oracle import GPTOracle, cfg_mix_oracle, sample_oracle


@torch.no_grad()
def given_oracle(orc: GPTOracle, cond, given, mask, max_new_tokens, emb_masks=None, cfg_scale=1.0, cfg_interval=-1, temperature=1.0,
                 top_k=0, top_p=1.0, sample_logits=True, negative=None, negative_emb_masks=None, generator=None):
    """given [B, S] int, mask [B, S] bool (True: given). Returns (tokens int32 [B, S], mixed logits fp32 [S, B, V] with rows k < P
    zero, P the leading run given to every image)."""
    c = orc.cfg
    S = max_new_tokens
    B = given.shape[0]
    use_cfg = cfg_scale > 1.0
    mask = mask.to(orc.device).bool()
    gv = given.to(orc.device).long()
    P = 0
    while P < S and bool(mask[:, P].all()):
        P += 1
    assert P < S, "every token is given"
    if c.model_type == "c2i":
        T = 1
        cond_all = torch.cat([cond, torch.ones_like(cond) * c.num_classes]) if use_cfg else cond
    else:
        T = cond.shape[1]
        unc = (negative.to(cond.device, cond.dtype).expand_as(cond) if negative is not None
               else torch.zeros_like(cond) + orc.sd["cls_embedding.uncond_embedding"])
        cond_all = torch.cat([cond, unc]) if use_cfg else cond
    orc.setup(2 * B if use_cfg else B, T + S)
    if emb_masks is not None or negative is not None:
        ones = torch.ones(B, T, device=cond.device)
        em = ones if emb_masks is None else emb_masks.to(cond.device).float()
        nm = em if negative is None else (ones if negative_emb_masks is None else negative_emb_masks.to(cond.device).float().expand(B, T))
        orc.apply_emb_masks(torch.cat([em, nm]) if use_cfg else em, T)
    sd = orc.sd
    lead = torch.cat([gv[:, :P], gv[:, :P]]) if use_cfg else gv[:, :P]
    x = torch.cat([orc.embed_cond(cond_all)[:, : c.cls_token_num], torch.nn.functional.embedding(lead, sd["tok_embeddings.weight"])], 1)
    pos = torch.arange(0, T + P, device=orc.device)
    orc.math_sdp = False
    for l in range(c.n_layer):
        x = orc._layer(l, x, orc.freqs[pos], pos, orc.mask[: x.shape[0], None, pos])
    logits = torch.nn.functional.linear(orc._rms(x, sd["norm.weight"]), sd["output.weight"]).float()[:, -1:]
    orc.math_sdp = True
    V = logits.shape[-1]
    sk = dict(temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits, generator=generator)
    toks = [gv[:, :P]]
    mixed_all = [torch.zeros(B, V, device=orc.device) for _ in range(P)]
    cur_pos = torch.tensor([T + P], device=orc.device, dtype=torch.int)
    for k in range(P, S):
        cfg_flag = not (cfg_interval > -1 and k - 1 > cfg_interval)       # generate.py:113-114, by token index
        mixed = (cfg_mix_oracle(logits, cfg_scale) if cfg_flag else logits[: logits.shape[0] // 2]) if use_cfg else logits
        mixed_all.append(mixed[:, -1].clone())
        nxt = torch.where(mask[:, k:k + 1], gv[:, k:k + 1], sample_oracle(mixed[:, -1], **sk)[0])
        toks.append(nxt)
        if k == S - 1:
            break
        xin = torch.cat([nxt, nxt]) if use_cfg else nxt
        logits = orc.forward(xin.view(-1, 1), None, cur_pos)
        cur_pos += 1
    return torch.cat(toks, dim=1).to(torch.int32), torch.stack(mixed_all)
