"""float64 restatement of the sample kernel's token log-probabilities (include/llamagen_b200.h, lg_logprobs).

x is the fp32 row a draw takes its token from (rounded, mixed, divided by temperature), `kept` the tokens top-k / top-p keep. With the
row restricted to the kept tokens, logprob(v) = (x_v - max) - log(sum exp(x - max)); rank(v) = 1 + #{u kept : x_u > x_v}; the top N are
the kept tokens ordered by (x descending, id ascending), padded with id -1 and logprob -inf."""
import numpy as np


def logprobs(x, kept):
    """float64 logprob of every token of the fp32 row x under the kept mask (-inf for the others)."""
    xk = np.where(kept, np.asarray(x, np.float64), -np.inf)
    m = xk.max()
    return (xk - m) - np.log(np.exp(xk - m).sum())


def rank(x, kept, v):
    """1 + the number of kept tokens whose fp32 value exceeds x_v (the kernel compares fp32 values)."""
    xk = np.where(kept, np.asarray(x, np.float32), -np.inf)
    return 1 + int((xk > xk[v]).sum())


def top(x, kept, n):
    """(ids int64 [n], float64 logprobs [n]): the n best kept tokens by (x desc, id asc), -1 / -inf past the kept ones."""
    xk = np.where(kept, np.asarray(x, np.float32), -np.inf)
    order = np.lexsort((np.arange(xk.shape[0]), -xk.astype(np.float64)))
    ids = [int(i) for i in order[:n] if kept[i]]
    lp = logprobs(x, kept)
    return (np.array(ids + [-1] * (n - len(ids)), np.int64),
            np.array([lp[i] for i in ids] + [-np.inf] * (n - len(ids)), np.float64))


def completion_logprobs(tokens, lp, rank_row, top_ids, top_lp, n, P=0):
    """The serving per-token dicts of one sample, built from generate()'s rows as serve.LLM builds them from its own: None for the
    P given tokens, then {token: (logprob, rank)} plus the n best alternatives with ranks 1 .. n (the drawn token keeps its own)."""
    out = [None] * P
    for k in range(P, len(tokens)):
        d = {int(tokens[k]): (float(lp[k]), int(rank_row[k]))}
        for r in range(n):
            if top_ids[k, r] >= 0:
                d.setdefault(int(top_ids[k, r]), (float(top_lp[k, r]), r + 1))
        out.append(d)
    return out
