"""The client's perplexity arithmetic restated per row, for the scoring tests.

DistributedLLM.perplexity (reference cli_api/common.py:129-139) takes scipy.special.softmax of the [n][n_vocab] logits in
float64 along each row, picks p[j, tokens[j + 1]], and sums `nll -= log p` one token at a time.  Row by row that is
nll_row() below; perplexity() is the sequential sum.  The device (k_nll_rows) computes the same formula; its value may
differ only by the last ulps of float64 exp and the summation order, hence TOL."""
import numpy as np
import scipy.special

# |nll_device - nll_host| <= TOL * max(1, |nll_host|)
TOL = 1e-12


def nll_row(logits, target: int) -> float:
    """-log softmax(logits)[target] in float64: NaN for a row with a NaN or +inf logit or all -inf, +inf when the
    target's probability underflows, as numpy gives them."""
    with np.errstate(all="ignore"):
        return float(-np.log(scipy.special.softmax(np.asarray(logits, np.float32).astype(np.float64))[target]))


def nll_rows(logits, targets) -> np.ndarray:
    return np.array([nll_row(x, int(t)) for x, t in zip(logits, targets)], np.float64)


def perplexity(nlls) -> float:
    """exp(nll / n) with nll summed in the reference's order."""
    nll = 0.0
    for v in nlls:
        nll += v
    return float(np.exp(nll / len(nlls)))


def within(dev, host) -> np.ndarray:
    """Elementwise: dev equals host within TOL, or both are the same non-finite value."""
    dev, host = np.asarray(dev, np.float64), np.asarray(host, np.float64)
    with np.errstate(all="ignore"):
        ok = np.abs(dev - host) <= TOL * np.maximum(1.0, np.abs(host))
    return ok | (np.isnan(dev) & np.isnan(host)) | (np.isinf(dev) & (dev == host))
