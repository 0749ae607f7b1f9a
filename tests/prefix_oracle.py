"""Prefix-completion oracle (TEST INFRASTRUCTURE ONLY): the semantics of `generate(..., prefix=tokens)`.

GPTOracle.forward runs the condition and the prefix embeddings at positions 0 .. T + P - 1 in ONE call (the inference branch of
gpt.py:341-368 over a multi-token input, with the causal mask rows of those positions and the emb-masks as generate.py:154-163
applies them), CFG-mixed as generate.py:79-82. Token P is sampled from the last position with token index P; decoding then continues
exactly as GPTOracle.generate does from index P + 1 (cfg_interval counted by token index)."""
import torch

from oracle import GPTOracle, cfg_mix_oracle, sample_oracle


@torch.no_grad()
def prefix_oracle(orc: GPTOracle, cond, prefix, max_new_tokens, emb_masks=None, cfg_scale=1.0, cfg_interval=-1, temperature=1.0,
                  top_k=0, top_p=1.0, sample_logits=True, teacher=None, generator=None):
    """prefix [B, P]. Returns (tokens int32 [B, S] with tokens[:, :P] == prefix, mixed logits fp32 [S, B, V] with rows k < P zero).
    teacher [B, S]: feed teacher[:, k] instead of the token sampled at index k >= P."""
    c = orc.cfg
    B, P = prefix.shape
    S = max_new_tokens
    use_cfg = cfg_scale > 1.0
    if c.model_type == "c2i":
        T = 1
        cond_all = torch.cat([cond, torch.ones_like(cond) * c.num_classes]) if use_cfg else cond
    else:
        T = cond.shape[1]
        null = torch.zeros_like(cond) + orc.sd["cls_embedding.uncond_embedding"]
        cond_all = torch.cat([cond, null]) if use_cfg else cond
    orc.setup(2 * B if use_cfg else B, T + S)
    if emb_masks is not None:
        orc.apply_emb_masks(torch.cat([emb_masks, emb_masks]) if use_cfg else emb_masks, T)
    sd = orc.sd
    pf = prefix.to(orc.device).long()
    pf = torch.cat([pf, pf]) if use_cfg else pf
    # one forward over positions 0 .. T + P - 1: the condition embedding, then the prefix token embeddings
    x = torch.cat([orc.embed_cond(cond_all)[:, : c.cls_token_num], torch.nn.functional.embedding(pf, sd["tok_embeddings.weight"])], 1)
    pos = torch.arange(0, T + P, device=orc.device)
    mask = orc.mask[: x.shape[0], None, pos]
    fr = orc.freqs[pos]
    orc.math_sdp = False
    for l in range(c.n_layer):
        x = orc._layer(l, x, fr, pos, mask)
    logits = torch.nn.functional.linear(orc._rms(x, sd["norm.weight"]), sd["output.weight"]).float()[:, -1:]
    orc.math_sdp = True
    V = logits.shape[-1]
    sk = dict(temperature=temperature, top_k=top_k, top_p=top_p, sample_logits=sample_logits, generator=generator)
    toks = [prefix.to(orc.device).to(torch.int64)]
    mixed_all = [torch.zeros(B, V, device=orc.device) for _ in range(P)]
    cur_pos = torch.tensor([T + P], device=orc.device, dtype=torch.int)
    for k in range(P, S):
        cfg_flag = not (cfg_interval > -1 and k - 1 > cfg_interval)       # generate.py:113-114, by token index
        if use_cfg:
            mixed = cfg_mix_oracle(logits, cfg_scale) if cfg_flag else logits[: logits.shape[0] // 2]
        else:
            mixed = logits
        mixed_all.append(mixed[:, -1].clone())
        nxt = sample_oracle(mixed[:, -1], **sk)[0]
        toks.append(nxt)
        if k == S - 1:
            break
        cur = nxt if teacher is None else teacher[:, k:k + 1].to(nxt.dtype)
        xin = torch.cat([cur, cur]) if use_cfg else cur
        logits = orc.forward(xin.view(-1, 1), None, cur_pos)
        cur_pos += 1
    return torch.cat(toks, dim=1).to(torch.int32), torch.stack(mixed_all)
