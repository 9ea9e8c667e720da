"""CPU: the host twin of top-k / top-p truncation (client.Sampler) against a brute-force restatement of the rule, its
draws, and the argument checks of the capi wrappers, which refuse bad settings before anything reaches the library."""
import numpy as np
import pytest

import sample_ref
import trunc_ref
from distributedllm_b200.client import Sampler, _softmax


def _brute_keep(y, top_k, top_p):
    """The rule with an explicit sort and loop."""
    n = len(y)
    ranked = sorted(range(n), key=lambda i: (-y[i], i))
    K = ranked[:top_k] if top_k and top_k < n else ranked
    p = _softmax(np.asarray(y, np.float64))
    keep = set(K)
    if top_p and top_p < 1:
        SK = sum(p[i] for i in K)
        acc, keep = 0.0, set()
        for i in K:
            if acc >= top_p * SK:
                break
            keep.add(i)
            acc += p[i]
    return np.array([i in keep for i in range(n)])


def _rows(rng, n):
    rows = [rng.standard_normal(n) * s for s in (0.5, 3.0, 10.0)]
    rows.append(np.round(rng.standard_normal(n) * 2) / 2)                   # many ties
    rows.append(np.full(n, 1.25))                                           # all tied
    r = np.zeros(n)
    r[int(rng.integers(0, n))] = 4.0
    rows.append(r)                                                          # one-hot
    r = np.full(n, -np.inf)
    r[rng.integers(0, n, 5)] = rng.standard_normal(5)
    rows.append(r)                                                          # a few finite ids, the rest -inf
    rows.append(-np.abs(rng.standard_normal(n)) * 2)                        # all negative
    return [np.asarray(r, np.float32) for r in rows]


KS = (None, 0, 1, 2, 5, 40, 63, 64, 1000)
PS = (None, 0.0, 1e-6, 0.3, 0.5, 0.9, 0.95, 1.0, 2.0)


def test_twin_equals_the_brute_force_rule():
    rng = np.random.default_rng(1)
    n = 64
    checked = 0
    for row in _rows(rng, n):
        for T, rp in ((0.7, 1.1), (1.0, 1.5), (0.0, 1.1)):
            prev = rng.integers(0, n, 6).tolist()
            y = trunc_ref.scaled(row, T, rp, prev)
            for k in KS:
                for p in PS:
                    keep, margin = trunc_ref.keep_mask(y, k, p)
                    if margin > trunc_ref.AMBIGUOUS:                # the loop sums in another order than numpy
                        assert (keep == _brute_keep(y.tolist(), k, p)).all(), (T, rp, k, p)
                    # the twin's draw: only kept ids of positive probability, one random() per draw
                    seed = int(rng.integers(0, 2 ** 63))
                    s = Sampler(T, rp, rng=np.random.Generator(np.random.Philox(key=seed)), top_k=k, top_p=p)
                    s.previous_ids = list(prev)
                    i = s(row)
                    assert keep[i] and _softmax(y)[i] > 0, (k, p, i)
                    want, _, _ = trunc_ref.sample(row, T, rp, prev, sample_ref.uniform(seed, 0), k, p)
                    assert i == want
                    checked += 1
    assert checked == 8 * 3 * len(KS) * len(PS)


def test_off_is_the_untruncated_sampler():
    rng = np.random.default_rng(2)
    for row in _rows(rng, 200):
        a = Sampler(0.8, 1.2, rng=np.random.Generator(np.random.Philox(key=9)))
        b = Sampler(0.8, 1.2, rng=np.random.Generator(np.random.Philox(key=9)), top_k=None, top_p=None)
        assert [a(row) for _ in range(20)] == [b(row) for _ in range(20)]


def test_one_random_per_draw():
    rng = np.random.default_rng(3)
    row = rng.standard_normal(300).astype(np.float32)
    g = np.random.Generator(np.random.Philox(key=77))
    s = Sampler(0.7, 1.1, rng=g, top_k=40, top_p=0.95)
    for _ in range(10):
        s(row)
    ref = np.random.Generator(np.random.Philox(key=77))
    ref.random(10)
    assert g.random() == ref.random()                                      # exactly 10 draws were spent


def test_top_k_1_is_the_argmax_and_a_tiny_top_p_is_top_k_1():
    rng = np.random.default_rng(4)
    for row in _rows(rng, 128):
        for T, rp in ((0.7, 1.1), (2.0, 1.5)):
            prev = rng.integers(0, 128, 10).tolist()
            y = trunc_ref.scaled(row, T, rp, prev)
            top = int(np.flatnonzero(y == y.max())[0])                     # lowest id among the maxima
            seeds = rng.integers(0, 2 ** 63, 5)
            for seed in seeds:
                got = []
                for kw in (dict(top_k=1), dict(top_p=1e-12), dict(top_k=7, top_p=1e-12)):
                    s = Sampler(T, rp, rng=np.random.Generator(np.random.Philox(key=int(seed))), **kw)
                    s.previous_ids = list(prev)
                    got.append(s(row))
                assert got == [top] * 3, (got, top)


def test_penalty_reorders_before_ranking():
    row = np.array([5.0, 4.9, -1.0, -2.0], np.float32)
    s = Sampler(1.0, 2.0, rng=np.random.Generator(np.random.Philox(key=1)), top_k=1)
    s.previous_ids = [0]                                                   # id 0 drops to 2.5: id 1 ranks first
    assert s(row) == 1


class _FakeLib:
    def __init__(self):
        self.calls = []

    def b200_extra_sample(self, h, x, n, sp, out):
        self.calls.append(("sample", sp._obj.top_k, sp._obj.top_p))
        return 0

    def b200_generate_sample(self, handles, n_slices, extra, ids, counts, n_seq, toks, n_steps, sp, out):
        self.calls.append(("generate", sp._obj.top_k, sp._obj.top_p))
        return 0

    def b200_stream_open(self, handles, n, extra, max_rows, lookahead, out):
        out._obj.value = 1
        return 0

    def b200_stream_add(self, h, session, prompt, n_prompt, max_tokens, sp, stops, n_stop):
        self.calls.append(("add", None if sp is None else (sp._obj.top_k, sp._obj.top_p)))
        return 0

    def b200_stream_close(self, h):
        return 0


class _Handle:
    handle = None
    n_vocab = 100
    n_embd = 8


BAD = [
    (ValueError, dict(top_k=-1)),
    (TypeError, dict(top_k=1.5)),
    (TypeError, dict(top_k=True)),
    (TypeError, dict(top_k="40")),
    (ValueError, dict(top_k=2 ** 31)),
    (ValueError, dict(top_p=-0.1)),
    (ValueError, dict(top_p=float("nan"))),
    (TypeError, dict(top_p="0.9")),
    (TypeError, dict(top_p=None)),
    (TypeError, dict(top_p=False)),
]


def test_capi_refuses_bad_truncation_before_the_library(monkeypatch):
    from distributedllm_b200 import capi
    f = _FakeLib()
    monkeypatch.setattr(capi, "lib", lambda: f)
    extra = object.__new__(capi.Extra)
    extra._h, extra.n_vocab, extra.n_embd = None, 100, 8
    rows = np.zeros((2, 100), np.float32)
    for exc, kw in BAD:
        with pytest.raises(exc):
            extra.sample(rows, 0.7, 1.1, [1, 2], **kw)
        with pytest.raises(exc):
            capi.generate_sample([_Handle()], extra, [0], [[1]], 4, 0.7, 1.1, [1], **kw)
    st = capi.Stream([_Handle()], _Handle())
    for exc, kw in BAD:
        with pytest.raises(exc):
            st.add(0, [1, 2], 4, temperature=0.7, **kw)
    with pytest.raises(ValueError):
        st.add(0, [1, 2], 4, top_k=40)                                     # greedy sessions take no truncation
    with pytest.raises(ValueError):
        st.add(0, [1, 2], 4, top_p=0.9)
    assert f.calls == []
    extra.sample(rows, 0.7, 1.1, [1, 2], top_k=40, top_p=0.95)
    extra.sample(rows, 0.7, 1.1, [1, 2])
    capi.generate_sample([_Handle()], extra, [0], [[1]], 4, 0.7, 1.1, [1], top_k=np.int64(3), top_p=float("inf"))
    st.add(0, [1, 2], 4, temperature=0.7, top_k=1, top_p=1)
    st.add(1, [1, 2], 4)
    st.close()
    extra._h = None
    assert f.calls == [("sample", 40, 0.95), ("sample", 0, 0.0), ("generate", 3, float("inf")), ("add", (1, 1.0)),
                       ("add", None)]


def test_sampling_struct_keeps_the_six_field_form():
    from distributedllm_b200 import capi
    sp = capi.Sampling(temperature=0.7, repeat_penalty=1.1, seeds=None, first_draw=0, history=None, history_counts=None)
    assert sp.top_k == 0 and sp.top_p == 0.0                                # off: the untruncated rule
    names = [f[0] for f in capi.Sampling._fields_]
    assert names[-2:] == ["top_k", "top_p"]


def test_header_documents_the_truncation_fields():
    import os
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200_slice.h")).read()
    body = text[text.index("typedef struct b200_sampling"):text.index("} b200_sampling_t;")]
    fields = [line.split("/*")[0].split() for line in body.splitlines()[1:] if line.split("/*")[0].strip()]
    assert fields[-2:] == [["int32_t", "top_k;"], ["double", "top_p;"]]         # appended: the old layout is a prefix
    assert "top-p" in text
