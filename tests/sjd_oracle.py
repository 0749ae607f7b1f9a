"""Test-side restatement of speculative Jacobi decoding (lg_generate_sjd, include/llamagen_b200.h): the acceptance rule, the
refresh of the window and the keyed uniforms, on plain numpy rows. It replays a GPU run from the p rows the engine dumps
(dbg_probs), and runs on a toy Markov model to show that the rule is lossless."""
import numpy as np

M64 = (1 << 64) - 1
C1, C2, C3 = 0xA0761D6478BD642F, 0xE7037ED1A0B428DB, 0x8EBC6AF09C88C6E3
C4, C5 = 0x9E6C63D0676A9A99, 0xD6E8FEB86659FD93
ACCEPT, RESIDUAL, INIT = 1, 2, 3


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _u(r):
    return np.float32((r >> 40) * (1.0 / 16777216.0))


def uniform(seed, b, k, purpose):
    """u_purpose(k) of image b."""
    r = splitmix64(splitmix64(splitmix64(seed ^ ((C1 * (k + 1)) & M64)) ^ ((C2 * (b + 1)) & M64)) ^ ((C3 * purpose) & M64))
    return _u(r)


def pass_seed(seed, b, j):
    return splitmix64(splitmix64(seed ^ ((C4 * (b + 1)) & M64)) ^ ((C5 * (j + 1)) & M64))


def sample_uniform(seed_row, step):
    """The sample kernel's uniform for a row with its own seed (lg_sample_rows)."""
    return _u(splitmix64(splitmix64(seed_row ^ ((C1 * (step + 1)) & M64)) ^ C2))


def inv_cdf(w, u):
    """First index whose running sum of the weights w passes u * sum(w) (float64 sums); the last positive weight past the end."""
    w = np.asarray(w, dtype=np.float64)
    c = np.cumsum(w)
    hit = np.nonzero((c > float(u) * c[-1]) & (w > 0))[0]
    return int(hit[0]) if hit.size else int(np.nonzero(w > 0)[0][-1])


class Image:
    """One image's loop state: tokens, n (final count), s (window start), window inputs, q rows (None = uniform)."""

    def __init__(self, S, L, V, seed, b, token0):
        self.S, self.L, self.V, self.seed, self.b = S, L, V, seed, b
        self.out = [token0] + [-1] * (S - 1)
        self.n, self.s = 1, 1
        self.win = [token0] + [self._init(k) for k in range(1, L)]
        self.q = [None] * L

    def _init(self, k):
        return min(int(uniform(self.seed, self.b, k, INIT) * np.float32(self.V)), self.V - 1)

    @property
    def done(self):
        return self.n >= self.S

    def step(self, p, x, greedy):
        """One pass: p [L][V] float32 rows for tokens s .. s + L - 1, x [L] the draws from them. Returns the tokens made final."""
        S, L, V, s = self.S, self.L, self.V, self.s
        i = self.n - s
        made = []
        while i <= L - 2:
            d, k = self.win[i + 1], s + i
            if greedy:
                acc = d == x[i]
            else:
                qd = np.float32(1.0) / np.float32(V) if self.q[i] is None else self.q[i][d]
                acc = uniform(self.seed, self.b, k, ACCEPT) * np.float32(qd) < p[i][d]
            if not acc:
                break
            self.out[k] = d
            made.append(d)
            i += 1
        if i <= L - 2 and not greedy:
            q = np.full(V, np.float32(1.0) / np.float32(V), np.float32) if self.q[i] is None else self.q[i]
            w = np.maximum(np.float32(0), p[i].astype(np.float32) - q)
            tok = inv_cdf(w, uniform(self.seed, self.b, s + i, RESIDUAL)) if w.sum() > 0 else int(x[i])
        else:
            tok = int(x[min(i, L - 1)])
        k = s + i
        self.out[k] = tok
        made.append(tok)
        n2 = k + 1
        s2 = min(n2, S - L)
        # refresh: slot t feeds token s2 + t - 1
        win, q = [0] * L, [None] * L
        for t in range(L):
            kk = s2 + t - 1
            if kk < n2:
                win[t] = self.out[kk]
                continue
            j = kk - s
            if j <= L - 1:
                win[t], q[t - 1] = int(x[j]), np.asarray(p[j], np.float32).copy()
            else:
                win[t], q[t - 1] = self._init(kk), None
        self.win, self.q, self.n, self.s = win, q, n2, s2
        return made


def draws(p, seed, b, j, s, greedy):
    """x for pass j of image b: the sample kernel's draw from each row of p (argmax when greedy)."""
    if greedy:
        return [int(np.argmax(r)) for r in p]
    sr = pass_seed(seed, b, j)
    return [inv_cdf(r, sample_uniform(sr, s + i)) for i, r in enumerate(p)]


def replay(dbg, token0, S, L, V, seed, greedy):
    """Tokens [B][S] and the pass count of a GPU run from its p rows dbg [passes][B][L][V] and its token 0 [B]."""
    imgs = [Image(S, L, V, seed, b, int(t)) for b, t in enumerate(token0)]
    j = 0
    while not all(im.done for im in imgs):
        for b, im in enumerate(imgs):
            if not im.done:
                im.step(dbg[j][b], draws(dbg[j][b], seed, b, j, im.s, greedy), greedy)
        j += 1
    return np.array([im.out for im in imgs]), j


def toy_run(p0, table, S, L, seed, greedy, b=0):
    """SJD on a Markov model: token 0 ~ p0 (the GPU's prefill draw is replaced by inv_cdf with u_init(0)), then token k ~ table[token
    k - 1]. Returns the tokens and the pass count."""
    V = table.shape[0]
    t0 = int(np.argmax(p0)) if greedy else inv_cdf(p0, uniform(seed, b, 0, INIT))
    im = Image(S, L, V, seed, b, t0)
    j = 0
    while not im.done:
        p = np.stack([table[im.win[i]] for i in range(L)])
        im.step(p, draws(p, seed, b, j, im.s, greedy), greedy)
        j += 1
    return im.out, j
