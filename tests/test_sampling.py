"""CPU: the facts the device sampler (k_sample_rows) rests on -- numpy's Philox4x64-10 stream, Generator.random() and
Generator.choice -- and the explicit-draw restatement (tests/sample_ref.py) against client.Sampler."""
import numpy as np
import pytest

import sample_ref
from distributedllm_b200.client import Sampler

KEYS = [0, 1, 7, 12345, 2 ** 32 + 5, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 12345, 2 ** 64 - 1]


@pytest.mark.parametrize("key", KEYS)
def test_philox_port_equals_numpy(key):
    raw = np.random.Philox(key=key).random_raw(23).tolist()
    assert [sample_ref.philox_word(key, d) for d in range(23)] == raw
    for start in (1, 2, 3, 6, 13):                      # offsets that are not multiples of 4
        bg = np.random.Philox(key=key)
        bg.random_raw(start)
        assert bg.random_raw(5).tolist() == [sample_ref.philox_word(key, d) for d in range(start, start + 5)]


@pytest.mark.parametrize("key", KEYS[:5])
def test_uniform_is_generator_random(key):
    g = np.random.Generator(np.random.Philox(key=key))
    got = [g.random() for _ in range(40)]
    assert got == [sample_ref.uniform(key, d) for d in range(40)]
    assert got == [(w >> 11) * 2.0 ** -53 for w in np.random.Philox(key=key).random_raw(40).tolist()]


def test_choice_is_searchsorted_on_one_random():
    rng = np.random.default_rng(0)
    for trial in range(300):
        n = int(rng.integers(1, 300))
        p = rng.random(n) ** int(rng.integers(1, 6))
        p[rng.random(n) < 0.2] = 0.0
        if p.sum() == 0:
            p[0] = 1.0
        p /= p.sum()
        key = int(rng.integers(0, 2 ** 63))
        g = np.random.Generator(np.random.Philox(key=key))
        got = [int(g.choice(np.arange(n), p=p)) for _ in range(3)]
        cdf = p.cumsum()
        cdf /= cdf[-1]
        want = [int(cdf.searchsorted(sample_ref.uniform(key, d), side="right")) for d in range(3)]
        assert got == want, trial


def test_eps_literal():
    assert 10 ** (-5) == 1e-5


@pytest.mark.parametrize("T,rp", [(0.0, 1.1), (0.2, 1.5), (0.7, 1.1), (1.0, 1.0), (5.0, 1.1)])
def test_twin_equals_client_sampler(T, rp):
    """The explicit-draw twin equals client.Sampler with a Philox generator, over sequences where penalised ids have
    negative logits (dividing one by rp > 1 raises it): ids 0..7 start in both histories and stay negative."""
    rng = np.random.default_rng(int(T * 10 + rp * 100))
    n = 64
    for key in (3, 2 ** 63 + 9):
        sampler = Sampler(T, rp, rng=np.random.Generator(np.random.Philox(key=key)))
        sampler.previous_ids = list(range(8))
        twin = sample_ref.Twin(T, rp, key, history=range(8))
        for step in range(40):
            logits = (rng.standard_normal(n) * 2).astype(np.float32)
            logits[:8] = -np.abs(logits[:8]) - 0.5         # ids 0..7 negative: penalising them raises their logits
            if step % 5 == 0:
                logits[rng.integers(0, n, 3)] = -np.inf
            want = sampler(logits)
            got, _ = twin(logits)
            assert got == want, (key, step)
        assert twin.prev == sampler.previous_ids
