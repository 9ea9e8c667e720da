"""The client's sampling rule restated with explicit draws, for the sampling tests.

numpy.random.Philox(key=seed) is Philox4x64-10 with key (seed, 0); draw d (0-based) of its stream is word d % 4 of the
block at counter (d // 4 + 1, 0, 0, 0) -- numpy increments the counter before its first block -- and Generator.random()
turns a word w into (w >> 11) * 2**-53.  Generator.choice(n, p=p) spends one random() u and returns
searchsorted(cumsum(p) / cumsum(p)[-1], u, side="right")."""
import numpy as np

from distributedllm_b200.client import _softmax

M0, M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
W0, W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B
MASK = (1 << 64) - 1
# ids may differ from the host twin only where u lies this close to a boundary of its CDF
AMBIGUOUS = 1e-9


def philox4x64_10(ctr, key):
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> 64) ^ c1 ^ k0, p1 & MASK, (p0 >> 64) ^ c3 ^ k1, p0 & MASK
    return c0, c1, c2, c3


def philox_word(seed: int, d: int) -> int:
    return philox4x64_10((d // 4 + 1, 0, 0, 0), (seed, 0))[d % 4]


def uniform(seed: int, d: int) -> float:
    return (philox_word(seed, d) >> 11) * 2.0 ** -53


def cdf_of(logits, temperature, repeat_penalty, prev):
    """Sampler.__call__'s arithmetic up to Generator.choice's normalised cumulative sum."""
    logits = np.array(logits)
    ids = np.arange(len(logits))
    seen = np.isin(ids, prev)
    p = _softmax(logits / ((seen * repeat_penalty + ~seen) * (temperature + 10 ** (-5))))
    cdf = p.cumsum()
    cdf /= cdf[-1]
    return p, cdf


def sample(logits, temperature, repeat_penalty, prev, u):
    """-> (id, distance from u to the nearest CDF boundary, probability of the id)."""
    p, cdf = cdf_of(logits, temperature, repeat_penalty, prev)
    i = int(cdf.searchsorted(u, side="right"))
    return i, float(np.min(np.abs(cdf - u))), float(p[i])


class Twin:
    """One session's host twin: draws from numpy.random.Philox(key=seed) from draw first_draw, history penalised."""

    def __init__(self, temperature, repeat_penalty, seed, first_draw=0, history=()):
        self.T, self.rp, self.seed, self.d = temperature, repeat_penalty, seed, first_draw
        self.prev = list(history)

    def __call__(self, logits):
        """-> (id, ambiguous)."""
        i, margin, _ = sample(logits, self.T, self.rp, self.prev, uniform(self.seed, self.d))
        self.d += 1
        self.prev.append(i)
        return i, margin <= AMBIGUOUS
