"""GPU: log-probabilities of generated ids (b200_generate_lp, b200_generate_speculative_lp, b200_stream_add_lp /
b200_stream_read_lp, b200_extra_logprobs).  The door's lp is exactly -nll of k_nll_rows; every loop's values equal the door
on that step's logits, bit for bit, alone, in a batch, split across calls, in a stream or under speculative decoding; and
asking for them changes no id."""
import ctypes as C

import numpy as np
import pytest
from scipy.special import log_softmax

from distributedllm_b200 import ggjt
from test_gpu_generate import _model

pytestmark = pytest.mark.gpu

SAMPLED = dict(temperature=0.7, repeat_penalty=1.1, top_k=40, top_p=0.95)


def _eq(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _extra(tmp_path, n_vocab, seed=62):
    from distributedllm_b200 import capi
    path = str(tmp_path / ("extra_%d.bin" % n_vocab))
    ggjt.write_synth_extra(path, ggjt.ModelShape(n_vocab, 256, 256, 4, 1), ggjt.T_Q4_0, seed=seed)
    return capi.Extra(path, 0)


def _door_rows(rng, V):
    chunk = (V + 1023) // 1024
    rows = [rng.standard_normal(V) * 3, rng.integers(-2, 2, V).astype(np.float64)]     # random, and ties everywhere
    r = rng.standard_normal(V)
    r[V - chunk:] = 7.0                                     # a tie across the last thread's chunk, at the vocabulary tail
    rows.append(r)
    r = rng.standard_normal(V)
    r[::5] = -np.inf
    r[11] = -1e4                                            # e_t underflows: -inf
    rows.append(r)
    for bad in (np.nan, np.inf):
        r = rng.standard_normal(V)
        r[V // 2] = bad
        rows.append(r)
    rows.append(np.full(V, -np.inf))
    x = np.array(rows, np.float32)
    ids = rng.integers(0, V, len(x)).astype(np.int32)
    ids[2], ids[3] = V - 1, 11
    return x, ids


@pytest.mark.parametrize("V", [512, 32000, 49953])
def test_door_equals_nll_lexsort_and_scipy(tmp_path, V):
    extra = _extra(tmp_path, V)
    x, ids = _door_rows(np.random.default_rng(V), V)
    nll = extra.nll(x, ids)
    good = [r for r in range(len(x)) if np.isfinite(x[r]).any() and not np.isnan(x[r]).any() and not (x[r] == np.inf).any()]
    assert len(good) == 4
    for n_top in (0, 1, 5, 20):
        lp, ti, tl = extra.logprobs(x, ids, n_top)
        assert _eq(lp, -nll), n_top                                         # the shared m and S: bit for bit
        for r in range(len(x)):
            if r not in good:
                assert np.isnan(lp[r]) and (ti[r] == -1).all() and np.isnan(tl[r]).all()
                continue
            order = np.lexsort((np.arange(V), -x[r]))[:n_top]
            assert ti[r].tolist() == order.tolist(), (n_top, r)
            if n_top:
                own, _, _ = extra.logprobs(np.repeat(x[r:r + 1], n_top, 0), order.astype(np.int32), 0)
                assert _eq(tl[r], own), (n_top, r)
                ref = log_softmax(x[r].astype(np.float64))[order]
                ref[np.exp(x[r][order].astype(np.float64) - x[r].max()) == 0] = -np.inf
                fin = np.isfinite(ref)
                assert _eq(np.isinf(tl[r]), ~fin)
                assert np.all(np.abs(tl[r][fin] - ref[fin]) <= 1e-12 * np.maximum(1.0, np.abs(ref[fin])))
    assert lp[3] == -np.inf


def _chain(capi, paths, n_sessions=8, n_ctx=128):
    return [capi.Slice(p, 0, n_ctx, n_sessions=n_sessions) for p in paths]


def _gen(capi, slices, extra, sessions, prompts, n, sampled, logprobs=None, seeds=None, first_draw=0, history=None):
    if not sampled:
        return capi.generate_greedy(slices, extra, sessions, prompts, n, logprobs=logprobs)
    seeds = seeds if seeds is not None else [100 + k for k in sessions]
    return capi.generate_sample(slices, extra, sessions, prompts, n, SAMPLED["temperature"], SAMPLED["repeat_penalty"],
                                seeds, first_draw=first_draw, history=history, top_k=SAMPLED["top_k"],
                                top_p=SAMPLED["top_p"], logprobs=logprobs)


@pytest.mark.parametrize("kind", ["q4_0", "q4_K_M"])
@pytest.mark.parametrize("sampled", [False, True])
def test_closed_loop(tmp_path, kind, sampled):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    slices = _chain(capi, paths)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(3)
    sessions = list(range(8))
    prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in (5, 1, 9, 3, 12, 2, 7, 4)]
    n, n_top = 12, 5

    def run(ses, prm, steps, **kw):
        for s in slices:
            s.session_clear(-1)
        return _gen(capi, slices, extra, ses, prm, steps, sampled, **kw)

    plain8 = run(sessions, prompts, n)
    ids8, lp8, ti8, tl8 = run(sessions, prompts, n, logprobs=n_top)
    assert _eq(ids8, plain8)                                                    # logprobs change no id
    assert np.isfinite(lp8).all() and (lp8 <= 0).all()
    if not sampled:
        assert _eq(ti8[:, :, 0], ids8)
    for k in (0, 4):                                                            # batch 1: alone, same values
        plain1 = run([k], [prompts[k]], n, seeds=[100 + k])
        ids1, lp1, ti1, tl1 = run([k], [prompts[k]], n, logprobs=n_top, seeds=[100 + k])
        assert _eq(ids1, plain1) and _eq(ids1[:, 0], ids8[:, k])
        assert _eq(lp1[:, 0], lp8[:, k]) and _eq(ti1[:, 0], ti8[:, k]) and _eq(tl1[:, 0], tl8[:, k])
    # split across two calls: the second continues from the first's last id
    k, a = 4, 5
    for s in slices:
        s.session_clear(-1)
    first = _gen(capi, slices, extra, [k], [prompts[k]], a, sampled, logprobs=n_top, seeds=[100 + k])
    hist = [first[0][:, 0].tolist()] if sampled else None
    second = _gen(capi, slices, extra, [k], [[int(first[0][-1, 0])]], n - a, sampled, logprobs=n_top,
                  seeds=[100 + k], first_draw=a, history=hist)
    for j in range(4):
        joined = np.concatenate([first[j][:, 0], second[j][:, 0]])
        assert _eq(joined, (ids8, lp8, ti8, tl8)[j][:, k]), j
    # the door on the host loop's logits (b200_extra_embed -> b200_session_forward -> b200_extra_logits): bit for bit
    for s in slices:
        s.session_clear(-1)
    toks, rows = prompts[k], []
    for j in range(n):
        x = extra.embed(toks)
        for s in slices:
            x = s.session_forward(k, x)
        rows.append(extra.logits(x[-1:])[0])
        toks = [int(ids8[j, k])]
    lp, ti, tl = extra.logprobs(np.array(rows), ids8[:, k].astype(np.int32), n_top)
    assert _eq(lp, lp8[:, k]) and _eq(ti, ti8[:, k]) and _eq(tl, tl8[:, k])


def test_stream_records_equal_generate_lp(tmp_path):
    """Sessions with and without logprobs, greedy and sampled, joining late, leaving early, and one forked from another's
    prefix: each session's (ids, lp, top) equal generate_* of it alone with logprobs; read() gives the same ids.  Output
    row 2i + 1 is a copy of row 2i, so every row of logits is full of ties; and one session is checked against k_nll_rows
    and np.lexsort on the host loop's logits, so the records do not only agree with the same kernel elsewhere."""
    from distributedllm_b200 import capi
    from test_gpu_vocab_sizes import _edit_output
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    tied = str(tmp_path / "tied_extra.bin")
    _edit_output(extra_path, tied, {2 * i + 1: 2 * i for i in range(sh.n_vocab // 2)}, 1.0)
    extra = capi.Extra(tied, 0)
    rng = np.random.default_rng(9)
    # session -> (prompt, budget, sampled, n_top or None)
    plan = {0: (rng.integers(0, 512, 6).tolist(), 8, False, 5), 1: (rng.integers(0, 512, 3).tolist(), 10, True, 3),
            2: (rng.integers(0, 512, 4).tolist(), 5, False, None), 3: (rng.integers(0, 512, 2).tolist(), 9, True, 0),
            4: (rng.integers(0, 512, 7).tolist(), 7, True, 20), 5: ([17, 30], 6, False, 5)}
    n_keep = len(plan[0][0]) + 3

    def add(st, k):
        prompt, budget, sampled, n_top = plan[k]
        kw = dict(temperature=SAMPLED["temperature"], repeat_penalty=SAMPLED["repeat_penalty"], seed=100 + k,
                  top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"]) if sampled else {}
        st.add(k, prompt, budget, logprobs=n_top, **kw)

    def run(with_lp):
        slices = _chain(capi, paths)
        recs = []
        read = (lambda st: st.read_logprobs(4)) if with_lp else (lambda st: [(s, t) for s, t in st.read(4)])
        with capi.Stream(slices, extra) as st:
            for k in (0, 1, 2, 3):
                add(st, k)
            while len(recs) < 12:
                recs += read(st)
            add(st, 4)                                                  # joins while the others run
            while True:
                more = read(st)
                if not more:
                    break
                recs += more
            st.fork(0, 5, n_keep)
            add(st, 5)
            while True:
                more = read(st)
                if not more:
                    break
                recs += more
        for s in slices:
            s.close()
        out = {}
        for r in recs:
            out.setdefault(r[0], []).append(r[1:])
        return out

    got = run(True)
    ids_only = run(False)
    twin = _chain(capi, paths)
    for k in range(6):
        prompt, budget, sampled, n_top = plan[k]
        if k == 5:
            for s in twin:
                s.session_copy(0, [5], n_keep)
        want = _gen(capi, twin, extra, [k], [prompt], budget, sampled, logprobs=n_top if n_top is not None else 0,
                    seeds=[100 + k])
        ids = [r[0] for r in got[k]]
        assert ids == want[0][:, 0].tolist(), k
        assert [r[0] for r in ids_only[k]] == ids, k
        lp = np.array([r[1] for r in got[k]])
        if n_top is None:
            assert np.isnan(lp).all() and all(r[2] == [] for r in got[k])
            continue
        assert _eq(lp, want[1][:, 0]), k
        assert _eq(np.array([[a for a, _ in r[2]] for r in got[k]]).reshape(budget, n_top), want[2][:, 0]), k
        assert _eq(np.array([[b for _, b in r[2]] for r in got[k]]).reshape(budget, n_top), want[3][:, 0]), k
        if not sampled and n_top:
            assert want[2][:, 0, 0].tolist() == ids
    # session 0 through the host loop: its logits are bit-identical to the device loop's
    host = _chain(capi, paths)
    toks, rows = plan[0][0], []
    for t in got[0]:
        x = extra.embed(toks)
        for s in host:
            x = s.session_forward(0, x)
        rows.append(extra.logits(x[-1:])[0])
        toks = [t[0]]
    rows = np.array(rows)
    ids0 = np.array([t[0] for t in got[0]], np.int32)
    assert _eq(np.array([t[1] for t in got[0]]), -extra.nll(rows, ids0))
    for j, t in enumerate(got[0]):
        order = np.lexsort((np.arange(sh.n_vocab), -rows[j]))[:5]
        assert [a for a, _ in t[2]] == order.tolist(), j
        assert rows[j][order[0]] == rows[j][order[1]]                 # the tie the rule decides


@pytest.mark.parametrize("sampled", [False, True])
def test_speculative_equals_the_plain_loop(tmp_path, sampled):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    fdir = tmp_path / "draft"
    fdir.mkdir()
    dpaths, dextra_path, _ = _model(fdir, "f16")                       # slice 0 of it: a 2-layer draft, n_embd 256
    prompt = np.random.default_rng(4).integers(0, sh.n_vocab, 6).tolist()
    n, n_top = 20, 5
    plain_sl = _chain(capi, paths, 1)
    extra = capi.Extra(extra_path, 0)
    want = _gen(capi, plain_sl, extra, [0], [prompt], n, sampled, logprobs=n_top, seeds=[7])
    target = _chain(capi, paths, 1)
    drafts = {"self": (_chain(capi, paths, 1), capi.Extra(extra_path, 0)),
              "2-layer": (_chain(capi, dpaths[:1], 1), capi.Extra(dextra_path, 0))}
    kw = dict(temperature=SAMPLED["temperature"], repeat_penalty=SAMPLED["repeat_penalty"], seed=7,
              top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"]) if sampled else {}
    for name, (dsl, dex) in drafts.items():
        for s in target + dsl:
            s.session_clear(-1)
        (ids, lp, ti, tl), stats = capi.generate_speculative(target, extra, 0, dsl, dex, 0, prompt, n, 4, logprobs=n_top,
                                                             **kw)
        assert _eq(ids, want[0][:, 0]), name
        assert _eq(lp, want[1][:, 0]) and _eq(ti, want[2][:, 0]) and _eq(tl, want[3][:, 0]), name


def test_refusals_change_nothing(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    slices = _chain(capi, paths, 2)
    extra = capi.Extra(extra_path, 0)
    L = capi.lib()
    handles = (C.c_void_p * 2)(*[s.handle for s in slices])
    sess, cnt, toks = np.array([0], np.int32), np.array([3], np.int32), np.array([1, 2, 3], np.int32)
    ids = np.full((4, 1), 77, np.int32)
    lp, ti, tl = np.full(4, 5.0), np.full((4, 21), 9, np.int32), np.full((4, 21), 5.0)
    cases = [capi.Logprobs(-1, lp.ctypes.data, ti.ctypes.data, tl.ctypes.data),
             capi.Logprobs(21, lp.ctypes.data, ti.ctypes.data, tl.ctypes.data),
             capi.Logprobs(3, None, ti.ctypes.data, tl.ctypes.data),
             capi.Logprobs(3, lp.ctypes.data, None, tl.ctypes.data),
             capi.Logprobs(3, lp.ctypes.data, ti.ctypes.data, None)]
    for c in cases:
        for rc in (L.b200_generate_lp(handles, 2, extra.handle, capi._ptr(sess), capi._ptr(cnt), 1, capi._ptr(toks), 4,
                                      None, capi._ptr(ids), C.byref(c)),):
            assert rc == 1
        assert [s.session_n_past(0) for s in slices] == [0, 0]
        assert (ids == 77).all() and (lp == 5.0).all() and (ti == 9).all()
    assert L.b200_generate_lp(handles, 2, extra.handle, capi._ptr(sess), capi._ptr(cnt), 1, capi._ptr(toks), 4, None,
                              capi._ptr(ids), None) == 1
    small = _extra(tmp_path, 16)
    x = np.zeros((1, 16), np.float32)
    i0 = np.zeros(1, np.int32)
    for n_top in (-1, 17, 21):
        assert L.b200_extra_logprobs(small.handle, capi._ptr(x), 1, capi._ptr(i0), n_top, capi._ptr(lp), capi._ptr(ti),
                                     capi._ptr(tl)) == 1
    with capi.Stream(slices, extra) as st:
        for n_top in (-2, 21):
            assert L.b200_stream_add_lp(st._h, 0, capi._ptr(toks), 3, 4, None, None, 0, n_top) == 1
        assert st.read(4) == []                                         # nothing was queued
    assert [s.session_n_past(0) for s in slices] == [0, 0]
    ok = capi.generate_greedy(slices, extra, [0], [[1, 2, 3]], 4, logprobs=20)
    assert ok[2].shape == (4, 1, 20)


def test_local_pipeline_generate_and_the_host_twin(tmp_path):
    from distributedllm_b200 import capi
    from distributedllm_b200.client import LocalPipeline, Sampler, token_logprobs
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    lp = LocalPipeline(paths, devices=[0, 0], n_ctx=128)
    out = list(lp.generate(extra_path, "hello world", 12, temperature=0.7, seed=5, logprobs=5))
    extra = capi.Extra(extra_path, 0)
    toks = extra.tokenize("hello world")
    lp.clear_context()
    sampler = Sampler(0.7, 1.1, rng=np.random.Generator(np.random.Philox(key=5)))
    for j, (text, v, alts) in enumerate(out):
        x = extra.embed(toks)
        for s in lp.slices:
            x = s.forward(x)
        logits = extra.logits(x[-1:])[0]
        t = sampler(logits)
        want, want_alts = token_logprobs(logits, t, 5)
        assert text == extra.token_text(t), j
        assert [a for a, _ in alts] == [a for a, _ in want_alts], j
        assert abs(v - want) <= 1e-12 * max(1.0, abs(want)), j
        assert all(abs(b - c) <= 1e-12 * max(1.0, abs(c)) for (_, b), (_, c) in zip(alts, want_alts)), j
        toks = [t]
    greedy = lp.generate_greedy(extra_path, "hello world", 6, logprobs=3)
    assert [g[0] for g in greedy] == lp.generate_greedy(extra_path, "hello world", 6)
    assert all(g[2][0][0] == g[0] for g in greedy)
    extra.close()
    lp.close()
