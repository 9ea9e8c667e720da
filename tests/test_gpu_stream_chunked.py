"""GPU: generation streams whose prompts are fed in chunks (b200_stream_open_ex, capi.Stream(prefill_chunk=C)).  Every
session's ids must equal the reference arrangement on a twin set of handles: b200_session_forward of each non-final
chunk [0, C), [C, 2C), ..., then b200_generate_* with the last chunk as the prompt, bit for bit, whatever joined, ran
beside it or left; and its positions must follow the position rule (old + n_prompt + delivered - 1)."""
import numpy as np
import pytest

from test_gpu_generate import _model
from test_gpu_stream import _by_session, _prefill

pytestmark = pytest.mark.gpu

N_CTX = 256


def _chunks(prompt, C):
    return [prompt[i:i + C] for i in range(0, len(prompt), C)] if C else [prompt]


def _reference(capi, twin, extra, k, prompt, C, n, mode, logprobs=None):
    """The reference arrangement on the twin handles: session_forward of every non-final chunk, then one generate call
    with the last chunk as the prompt.  mode = (temperature or None, repeat penalty, seed, top_k, top_p)."""
    parts = _chunks(prompt, C)
    for part in parts[:-1]:
        _prefill(extra, (twin,), k, part)
    T, rp, seed, top_k, top_p = mode
    if T is None:
        out = capi.generate_greedy(twin, extra, [k], [parts[-1]], n, logprobs=logprobs)
    else:
        out = capi.generate_sample(twin, extra, [k], [parts[-1]], n, T, rp, [seed], top_k=top_k, top_p=top_p,
                                   logprobs=logprobs)
    return out if logprobs is not None else out[:, 0].tolist()


def _add(st, k, prompt, budget, mode, **kw):
    T, rp, seed, top_k, top_p = mode
    if T is None:
        st.add(k, prompt, budget, **kw)
    else:
        st.add(k, prompt, budget, temperature=T, repeat_penalty=rp, seed=seed, top_k=top_k, top_p=top_p, **kw)


def _drain(st, pairs, cap=7):
    while True:
        more = st.read(cap)
        if not more:
            return pairs
        pairs += more


def _handles(capi, paths, n_sess):
    return [capi.Slice(p, 0, N_CTX, n_sessions=n_sess) for p in paths]


def _close(extra, *sets):
    extra.close()
    for hs in sets:
        for s in hs:
            s.close()


GREEDY = (None, 1.1, 0, 0, 0.0)
SAMPLED = {0: (0.8, 1.1, 11, 0, 0.0), 1: GREEDY, 2: (0.7, 1.3, 2 ** 63 + 5, 40, 0.9), 3: (1.0, 1.0, 977, 0, 0.0),
           4: (0.5, 1.5, 3, 0, 0.0), 5: (0.9, 1.2, 2 ** 40 + 1, 0, 0.0)}


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
@pytest.mark.parametrize("sampled", [False, True])
def test_chunked_stream_equals_the_reference_arrangement(tmp_path, kind, sampled):
    """C = 8, max_rows = 20: prompts shorter than C, equal to C, between C and max_rows and longer than max_rows, one
    session mid-context, joins staggered across reads."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    C, max_rows = 8, 20
    gpu, twin = _handles(capi, paths, 6), _handles(capi, paths, 6)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(61)
    _prefill(extra, (gpu, twin), 3, rng.integers(0, sh.n_vocab, 20).tolist())    # session 3 starts mid-context
    plan = {0: (5, 12), 1: (8, 20), 2: (14, 9), 3: (45, 15), 4: (27, 10), 5: (3, 14)}
    prompts = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, (n, _) in plan.items()}
    modes = SAMPLED if sampled else {k: GREEDY for k in plan}
    start = {k: [s.session_n_past(k) for s in gpu] for k in plan}
    pairs = []
    with capi.Stream(gpu, extra, max_rows=max_rows, lookahead=3, prefill_chunk=C) as st:
        for k in (0, 1, 2, 3):
            _add(st, k, prompts[k], plan[k][1], modes[k])
        while len(pairs) < 5:
            pairs += st.read(1)
        _add(st, 4, prompts[4], plan[4][1], modes[4])
        while len(pairs) < 17:
            pairs += st.read(1)
        _add(st, 5, prompts[5], plan[5][1], modes[5])
        _drain(st, pairs)
        assert st.stats()["most_rows"] <= max_rows
    got = _by_session(pairs)
    for k, (n, budget) in plan.items():
        assert len(got[k]) == budget, k
        assert [s.session_n_past(k) for s in gpu] == [p + n + budget - 1 for p in start[k]], k
        assert _reference(capi, twin, extra, k, prompts[k], C, budget, modes[k]) == got[k], (kind, sampled, k)
    assert [s.session_n_past(k) for s in gpu for k in plan] == [s.session_n_past(k) for s in twin for k in plan]
    assert len(set(sum(got.values(), []))) > 3
    _close(extra, gpu, twin)


def test_no_split_equals_the_unchunked_stream(tmp_path):
    """C >= every prompt: the same adds give every session the same ids, and the same positions, as a prefill_chunk = 0
    stream.  (The order of the pairs across sessions may differ: a chunked stream's read tops up its lookahead only while
    it holds no id, so a session added between reads can join another step.)"""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu, twin = _handles(capi, paths, 5), _handles(capi, paths, 5)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(62)
    _prefill(extra, (gpu, twin), 2, rng.integers(0, sh.n_vocab, 11).tolist())
    plan = {0: (16, 12), 1: (3, 20), 2: (9, 8), 3: (1, 15), 4: (16, 6)}
    prompts = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, (n, _) in plan.items()}

    def run(handles, C):
        pairs = []
        with capi.Stream(handles, extra, max_rows=24, lookahead=2, prefill_chunk=C) as st:
            for k in (0, 1, 2):
                _add(st, k, prompts[k], plan[k][1], SAMPLED[k])
            while len(pairs) < 4:
                pairs += st.read(1)
            for k in (3, 4):
                _add(st, k, prompts[k], plan[k][1], SAMPLED[k])
            return _drain(st, pairs)

    chunked, whole = run(gpu, 16), run(twin, 0)
    assert _by_session(chunked) == _by_session(whole)
    assert len(chunked) == sum(b for _, b in plan.values())
    assert [s.session_n_past(k) for s in gpu for k in plan] == [s.session_n_past(k) for s in twin for k in plan]
    _close(extra, gpu, twin)


def test_decoding_continues_during_a_prefill(tmp_path):
    """max_rows = C + 1, lookahead 1: a decoding session A keeps its row in every step while B's k * C-id prompt is fed
    one chunk per step, so A draws at least k ids after B's add and before B's first, one beside each chunk.  The steps
    enqueued before the add give A at most lookahead + 1 = 2 of them, so a scheduler that leaves A out of the chunk steps
    fails.  No step carries more than max_rows rows."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_K_M")
    C, k_chunks = 8, 6
    gpu, twin = _handles(capi, paths, 2), _handles(capi, paths, 2)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(63)
    a_prompt, b_prompt = rng.integers(0, sh.n_vocab, 4).tolist(), rng.integers(0, sh.n_vocab, k_chunks * C).tolist()
    with capi.Stream(gpu, extra, max_rows=C + 1, lookahead=1, prefill_chunk=C) as st:
        _add(st, 0, a_prompt, 40, SAMPLED[0])
        before = st.read(1)
        _add(st, 1, b_prompt, 5, SAMPLED[2])
        pairs = _drain(st, [])
        stats = st.stats()
    first_b = [k for k, _ in pairs].index(1)
    assert sum(1 for k, _ in pairs[:first_b] if k == 0) >= k_chunks, (before, pairs[:first_b + 1])
    pairs = before + pairs
    assert 0 < stats["most_rows"] <= C + 1, stats
    assert stats["rows"] == len(a_prompt) + 39 + len(b_prompt) + 4, stats     # every fed row counted once
    got = _by_session(pairs)
    assert got[0] == _reference(capi, twin, extra, 0, a_prompt, C, 40, SAMPLED[0])
    assert got[1] == _reference(capi, twin, extra, 1, b_prompt, C, 5, SAMPLED[2])
    _close(extra, gpu, twin)


def test_steps_with_no_draw(tmp_path):
    """One session with a 20 * C-id prompt and lookahead 1: 19 steps draw nothing, and read still blocks until the id
    comes.  Then a close while such steps are in flight leaves the session at old, with no trace in its cache."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    C = 8
    gpu, twin = _handles(capi, paths, 2), _handles(capi, paths, 2)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(64)
    prompt = rng.integers(0, sh.n_vocab, 20 * C).tolist()
    with capi.Stream(gpu, extra, lookahead=1, prefill_chunk=C) as st:
        _add(st, 0, prompt, 10, SAMPLED[0])
        first = st.read(64)
        pairs = _drain(st, list(first))
        stats = st.stats()
    assert first and stats["steps"] == 19 + 10, stats
    assert _by_session(pairs)[0] == _reference(capi, twin, extra, 0, prompt, C, 10, SAMPLED[0])
    assert [s.session_n_past(0) for s in gpu] == [len(prompt) + 9] * len(gpu)
    # close with chunk steps in flight: session 1 decodes, session 0 (now at len(prompt) + 9) is fed a new long prompt
    old = gpu[0].session_n_past(0)
    again = rng.integers(0, sh.n_vocab, 10 * C).tolist()
    with capi.Stream(gpu, extra, lookahead=4, prefill_chunk=C) as st:
        _add(st, 1, [3, 4], 30, GREEDY)
        _add(st, 0, again, 5, GREEDY)
        got = st.read(1)
    assert got == [(1, _reference(capi, twin, extra, 1, [3, 4], C, 1, GREEDY)[0])]
    assert [s.session_n_past(0) for s in gpu] == [old] * len(gpu)
    assert [s.session_n_past(1) for s in gpu] == [2] * len(gpu)
    # the abandoned chunks left no trace: feeding the same prompt again equals the reference from the same position
    with capi.Stream(gpu, extra, prefill_chunk=C) as st:
        _add(st, 0, again, 5, GREEDY)
        pairs = _drain(st, [])
    assert _by_session(pairs)[0] == _reference(capi, twin, extra, 0, again, C, 5, GREEDY)
    _close(extra, gpu, twin)


def test_cancel_mid_prefill(tmp_path):
    """Sessions 1 and 2 are cancelled while their chunks are in flight: 2 is back at old after close; 1 is added again
    at once and equals the reference.  The decoding neighbour is untouched."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    C = 8
    gpu, twin = _handles(capi, paths, 3), _handles(capi, paths, 3)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(65)
    _prefill(extra, (gpu, twin), 2, rng.integers(0, sh.n_vocab, 9).tolist())
    prompts = {0: rng.integers(0, sh.n_vocab, 4).tolist(), 1: rng.integers(0, sh.n_vocab, 10 * C).tolist(),
               2: rng.integers(0, sh.n_vocab, 10 * C).tolist()}
    start = {k: [s.session_n_past(k) for s in gpu] for k in prompts}
    with capi.Stream(gpu, extra, max_rows=1 + 2 * C, lookahead=4, prefill_chunk=C) as st:
        _add(st, 0, prompts[0], 30, SAMPLED[3])
        _add(st, 1, prompts[1], 6, SAMPLED[4])
        _add(st, 2, prompts[2], 6, GREEDY)
        pairs = st.read(1)
        assert pairs[0][0] == 0
        st.cancel(1)
        st.cancel(2)
        _add(st, 1, prompts[1], 6, SAMPLED[4])
        _drain(st, pairs)
    got = _by_session(pairs)
    assert 2 not in got and len(got[1]) == 6
    assert [s.session_n_past(2) for s in gpu] == start[2]
    assert [s.session_n_past(1) for s in gpu] == [p + 10 * C + 5 for p in start[1]]
    assert got[0] == _reference(capi, twin, extra, 0, prompts[0], C, 30, SAMPLED[3])
    assert got[1] == _reference(capi, twin, extra, 1, prompts[1], C, 6, SAMPLED[4])
    _close(extra, gpu, twin)


@pytest.mark.parametrize("sampled", [False, True])
def test_logprobs_of_a_chunked_session(tmp_path, sampled):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_K_M")
    C, n_top, budget = 8, 5, 9
    gpu, twin = _handles(capi, paths, 2), _handles(capi, paths, 2)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(66)
    prompt, other = rng.integers(0, sh.n_vocab, 3 * C + 5).tolist(), rng.integers(0, sh.n_vocab, 6).tolist()
    mode = SAMPLED[2] if sampled else GREEDY
    recs = []
    with capi.Stream(gpu, extra, max_rows=C + 2, prefill_chunk=C) as st:
        _add(st, 1, other, 12, SAMPLED[0])                 # a neighbour without log-probabilities
        _add(st, 0, prompt, budget, mode, logprobs=n_top)
        while True:
            more = st.read_logprobs(3)
            if not more:
                break
            recs += more
    mine = [r for r in recs if r[0] == 0]
    ids, lp, top_ids, top_lp = _reference(capi, twin, extra, 0, prompt, C, budget, mode, logprobs=n_top)
    assert [r[1] for r in mine] == ids[:, 0].tolist()
    assert np.array([r[2] for r in mine]).tobytes() == np.ascontiguousarray(lp[:, 0], np.float64).tobytes()
    assert [[a for a, _ in r[3]] for r in mine] == top_ids[:, 0].tolist()
    assert np.array([[b for _, b in r[3]] for r in mine]).tobytes() == \
        np.ascontiguousarray(top_lp[:, 0], np.float64).tobytes()
    theirs = [r for r in recs if r[0] == 1]
    assert all(np.isnan(r[2]) and r[3] == [] for r in theirs)
    assert [r[1] for r in theirs] == _reference(capi, twin, extra, 1, other, C, 12, SAMPLED[0])
    _close(extra, gpu, twin)


def test_fork_refuses_a_prefilling_session(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    C = 8
    gpu, twin = _handles(capi, paths, 3), _handles(capi, paths, 3)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(67)
    prompt = rng.integers(0, sh.n_vocab, 6 * C).tolist()
    with capi.Stream(gpu, extra, max_rows=C + 1, prefill_chunk=C) as st:
        _add(st, 1, [5, 6], 20, GREEDY)
        _add(st, 0, prompt, 4, GREEDY)
        pairs = st.read(1)                                 # session 0's chunks are in flight, its last one is not
        with pytest.raises(capi.B200Error) as ei:
            st.fork(0, 2, 8)
        assert ei.value.code == 1 and "active" in str(ei.value)
        _drain(st, pairs)
        st.fork(0, 2, 6 * C)                               # ended: its prompt's rows go to session 2
        _add(st, 2, [7], 3, GREEDY)
        _drain(st, pairs)
    got = _by_session(pairs)
    assert got[0] == _reference(capi, twin, extra, 0, prompt, C, 4, GREEDY)
    for s in twin:
        s.session_copy(0, [2], 6 * C)
    assert got[2] == capi.generate_greedy(twin, extra, [2], [[7]], 3)[:, 0].tolist()
    _close(extra, gpu, twin)


def test_refusals(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = _handles(capi, paths, 2)
    extra = capi.Extra(extra_path, 0)
    lib = capi.lib()
    import ctypes as C
    handles = (C.c_void_p * len(gpu))(*[s.handle for s in gpu])
    out = C.c_void_p()
    for max_rows, chunk in ((16, -1), (16, 17), (0, N_CTX + 1)):
        assert lib.b200_stream_open_ex(handles, len(gpu), extra.handle, max_rows, 0, chunk, C.byref(out)) == 1, chunk
        assert not out.value
    with capi.Stream(gpu, extra, max_rows=0, prefill_chunk=N_CTX) as st:        # C = the resolved max_rows is accepted
        st.add(0, [1] * 40, 2)
        assert len(_drain(st, [])) == 2
    for s in gpu:
        s.session_clear(-1)
    with capi.Stream(gpu, extra, max_rows=8) as st:
        with pytest.raises(capi.B200Error) as ei:
            st.add(0, [1] * 9, 2)                                                # prefill_chunk 0: never split
        assert ei.value.code == 1 and "max_rows" in str(ei.value)
    with capi.Stream(gpu, extra, max_rows=8, prefill_chunk=4) as st:
        st.add(0, [1] * 9, 2)                                                    # chunked: accepted
        with pytest.raises(capi.B200Error) as ei:
            st.add(1, [1] * 200, N_CTX - 199 + 1)                                # one past n_ctx
        assert ei.value.code == 5
        st.add(1, [1] * 200, N_CTX - 199)                                        # ends exactly at n_ctx
        pairs = _drain(st, [])
    assert len(pairs) == 2 + N_CTX - 199
    assert [s.session_n_past(1) for s in gpu] == [N_CTX] * len(gpu)
    _close(extra, gpu)
