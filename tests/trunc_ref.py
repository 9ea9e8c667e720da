"""Top-k / top-p truncation restated for the tests: the host twin's arithmetic with its two ambiguity margins.

client.Sampler(T, rp, rng, top_k, top_p) ranks the ids by y = x / d descending (equal y: lower id first), keeps the first
top_k (0: all) as K, then drops an id of K whose probability ranked strictly before it (within K) is >= top_p * S_K, and
draws with one random() u from the kept probabilities.  The device computes the same rule with its own float64 exp and
fixed-point masses, so its id may differ from the twin's only where
  - u lies within sample_ref.AMBIGUOUS of a boundary of the twin's CDF, or
  - the twin's mass before the last kept id, or before the first dropped one, lies within AMBIGUOUS * S_K of
    top_p * S_K."""
import numpy as np

import sample_ref
from distributedllm_b200.client import _softmax

AMBIGUOUS = sample_ref.AMBIGUOUS


def scaled(logits, temperature, repeat_penalty, prev):
    """Sampler.__call__'s y = x / d."""
    logits = np.array(logits)
    ids = np.arange(len(logits))
    seen = np.isin(ids, prev)
    return logits / ((seen * repeat_penalty + ~seen) * (temperature + 10 ** (-5)))


def keep_mask(y, top_k, top_p):
    """-> (kept ids as a bool mask, the top-p margin relative to S_K: inf when no top-p cut applies)."""
    n = len(y)
    ids = np.arange(n)
    p = _softmax(y)
    order = np.lexsort((ids, -y))
    K = order[:top_k] if top_k else order
    keep = np.zeros(n, bool)
    keep[K] = True
    margin = np.inf
    if top_p and top_p < 1:
        pk = p[K]
        before = np.concatenate(([0.0], np.cumsum(pk)[:-1]))
        SK = pk.sum()
        drop = before >= top_p * SK
        keep[K[drop]] = False
        last = int(np.count_nonzero(~drop)) - 1              # the kept ids are a prefix of K
        edges = [before[last]] + ([before[last + 1]] if last + 1 < len(K) else [])
        margin = min(abs(b - top_p * SK) for b in edges) / SK
    return keep, margin


def sample(logits, temperature, repeat_penalty, prev, u, top_k, top_p):
    """-> (id, ambiguous, kept mask)."""
    y = scaled(logits, temperature, repeat_penalty, prev)
    keep, pm = keep_mask(y, top_k, top_p)
    p = np.where(keep, _softmax(y), 0.0)
    p = p / p.sum()
    cdf = p.cumsum()
    cdf /= cdf[-1]
    i = int(cdf.searchsorted(u, side="right"))
    return i, bool(np.min(np.abs(cdf - u)) <= AMBIGUOUS or pm <= AMBIGUOUS), keep


class Twin:
    """One session's host twin with truncation: draws from numpy.random.Philox(key=seed) from draw first_draw."""

    def __init__(self, temperature, repeat_penalty, seed, top_k, top_p, first_draw=0, history=()):
        self.T, self.rp, self.seed, self.d = temperature, repeat_penalty, seed, first_draw
        self.top_k, self.top_p = top_k, top_p
        self.prev = list(history)

    def __call__(self, logits):
        """-> (id, ambiguous)."""
        i, amb, _ = sample(logits, self.T, self.rp, self.prev, sample_ref.uniform(self.seed, self.d), self.top_k, self.top_p)
        self.d += 1
        self.prev.append(i)
        return i, amb
