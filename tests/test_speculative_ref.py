"""CPU: the speculative loop's acceptance rule (tests/spec_ref.py) gives the plain loop's ids and the stated counts, for
scripted target and draft models."""
import pytest

from spec_ref import plain, speculate

PROMPT = [1, 17, 300]


def target(ctx):
    """A deterministic 'model': the next id is a hash of the whole context."""
    h = 0
    for t in ctx:
        h = (h * 1000003 + t + 7) % 32000
    return h


def passes_for(n_steps, k):
    return -(-(n_steps - 1) // (k + 1))


@pytest.mark.parametrize("k", [1, 2, 4, 7, 15])
@pytest.mark.parametrize("n_steps", [1, 2, 33, 100])
def test_every_draft_accepted(k, n_steps):
    ids, st = speculate(target, lambda ctx, i: target(ctx), PROMPT, n_steps, k)
    assert ids == plain(target, PROMPT, n_steps)
    assert st["passes"] == passes_for(n_steps, k)
    assert st["drafted"] == st["passes"] * k == st["accepted"]


@pytest.mark.parametrize("k", [1, 4, 15])
def test_none_accepted(k):
    ids, st = speculate(target, lambda ctx, i: (target(ctx) + 1) % 32000, PROMPT, 40, k)
    assert ids == plain(target, PROMPT, 40)
    assert st == {"passes": 39, "drafted": 39 * k, "accepted": 0}


@pytest.mark.parametrize("j", range(1, 9))
def test_first_mismatch_at_each_j(j):
    k = 8
    ids, st = speculate(target, lambda ctx, i: target(ctx) if i != j else -5, PROMPT, 50, k)
    assert ids == plain(target, PROMPT, 50)
    # every pass keeps j - 1 proposals and emits j ids (the last pass may be cut by the budget)
    assert st["passes"] == -(-49 // j)
    assert st["drafted"] == st["passes"] * k
    assert st["accepted"] == st["passes"] * (j - 1)


def test_budget_ends_mid_iteration():
    ids, st = speculate(target, lambda ctx, i: target(ctx), PROMPT, 8, 4)      # 1 + 5 + 2 ids
    assert ids == plain(target, PROMPT, 8)
    assert st == {"passes": 2, "drafted": 8, "accepted": 8}


def test_one_step_runs_no_pass():
    ids, st = speculate(target, lambda ctx, i: target(ctx), PROMPT, 1, 4)
    assert ids == [target(PROMPT)]
    assert st == {"passes": 0, "drafted": 0, "accepted": 0}


def test_fifteen_drafts_with_a_wandering_draft():
    # the draft agrees on contexts of even length only: acceptance varies from pass to pass
    draft = lambda ctx, i: target(ctx) if len(ctx) % 2 == 0 else 3
    ids, st = speculate(target, draft, PROMPT, 100, 15)
    assert ids == plain(target, PROMPT, 100)
    assert st["drafted"] == st["passes"] * 15
    assert 0 <= st["accepted"] <= st["drafted"]
