"""CPU: the per-row restatement of the client's perplexity (tests/score_ref.py), which the device scoring (k_nll_rows,
b200_score) is held to, against the reference's own formula: scipy.special.softmax over the whole [n][n_vocab] matrix
along axis 1, then a sequential `nll -= log p` loop."""
import numpy as np
import pytest
import scipy.special

import score_ref


def _reference_perplexity(logits, targets):
    """DistributedLLM.perplexity's arithmetic after get_logits (reference cli_api/common.py:129-139)."""
    n = len(targets)
    pmf = scipy.special.softmax(np.asarray(logits, np.float32).astype(np.float64).reshape(n, -1), axis=1)
    probabilities = pmf[np.arange(n), targets]
    nll = 0
    for t in range(n):
        nll -= np.log(probabilities[t])
    return np.exp(nll / n), probabilities


@pytest.mark.parametrize("n_vocab", [512, 32000])
def test_twin_equals_the_reference_formula(n_vocab):
    rng = np.random.default_rng(n_vocab)
    for n, scale in ((1, 1.0), (7, 3.0), (64, 12.0)):
        logits = (rng.standard_normal((n, n_vocab)) * scale).astype(np.float32)
        targets = rng.integers(0, n_vocab, n)
        want, p = _reference_perplexity(logits, targets)
        rows = score_ref.nll_rows(logits, targets)
        assert (rows == -np.log(p)).all(), (n, scale)           # row by row, bit for bit
        assert score_ref.perplexity(rows) == want, (n, scale)


def test_non_finite_rows_follow_numpy():
    """What the device must reproduce: NaN for a NaN or +inf logit and for an all -inf row, +inf for a target whose
    probability underflows, a finite value for a -inf logit elsewhere in the row."""
    x = np.zeros(512, np.float32)
    for bad in (np.nan, np.inf):
        y = x.copy()
        y[9] = bad
        assert np.isnan(score_ref.nll_row(y, 3)) and np.isnan(score_ref.nll_row(y, 9))
    assert np.isnan(score_ref.nll_row(np.full(512, -np.inf, np.float32), 0))
    y = x.copy()
    y[5] = -1000.0                                              # exp(-1000) underflows float64
    assert score_ref.nll_row(y, 5) == np.inf
    y[7] = -np.inf
    assert score_ref.nll_row(y, 7) == np.inf and np.isfinite(score_ref.nll_row(y, 0))
    assert score_ref.within([np.nan, np.inf, 1.0 + 5e-13], [np.nan, np.inf, 1.0]).all()
    assert not score_ref.within([np.inf, 1.0 + 3e-12, np.nan], [np.nan, 1.0, 1.0]).any()
