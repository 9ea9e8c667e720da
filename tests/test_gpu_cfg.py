"""GPU: classifier-free guidance (b200_generate_cfg, b200_extra_cfg, LocalPipeline's cfg_* options).

* The door (k_cfg_rows on host rows) equals client.cfg_logits with correctly rounded expf / logf bit for bit, NaN positions
  included, at vocabulary sizes that are and are not multiples of 32, and its greedy ids follow max_element.
* b200_generate_cfg's ids and log-probabilities equal a host loop (session_forward on both sessions, b200_extra_logits,
  cfg_logits, then max_element or the device sampler's door on the guided row), alone, in a batch of 8 pairs and split
  across two calls; the log-probabilities are those of the raw rows.
* Refused calls leave every position and cache byte as they were."""
import numpy as np
import pytest

from distributedllm_b200 import capi, client, ggjt
from test_gpu_generate import _model

pytestmark = pytest.mark.gpu

SAMPLED = dict(temperature=0.7, repeat_penalty=1.1, top_k=40, top_p=0.95)
SCALE, SF = 1.75, 0.5


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.where(np.isnan(a), 0, a).view(np.uint32), np.where(np.isnan(b), 0, b).view(np.uint32))


def _rows(rng, V):
    b, g = [], []
    for s in (1.0, 4.0):
        b.append(rng.standard_normal(V) * s)
        g.append(rng.standard_normal(V) * s)
    x = rng.standard_normal(V)
    x[rng.choice(V, 7, replace=False)] -= 150                           # lb underflows: sf 1 gives NaN there
    b.append(x)
    g.append(rng.standard_normal(V))
    x, y = rng.standard_normal(V), rng.standard_normal(V)
    x[V - 1] -= 200                                                     # both underflow at the tail: all NaN
    y[V - 1] -= 300
    b.append(x)
    g.append(y)
    x = rng.standard_normal(V)
    x[[1, V // 2, V - 1]] = 9.0                                         # ties for the max
    b.append(x)
    g.append(np.round(rng.standard_normal(V), 1))
    return np.array(b, np.float32), np.array(g, np.float32)


def _extra(tmp_path, V):
    path = str(tmp_path / ("extra_%d.bin" % V))
    ggjt.write_synth_extra(path, ggjt.ModelShape(V, 256, 256, 4, 1), ggjt.T_Q4_0, seed=62)
    return capi.Extra(path, 0)


@pytest.mark.parametrize("V", [32000, 1031, 32001, 49953])
def test_door_equals_the_twin(tmp_path, V):
    extra = _extra(tmp_path, V)
    b, g = _rows(np.random.default_rng(V), V)
    for scale, sf in ((SCALE, SF), (1.5, 1.0), (3.0, 0.0)):
        out, greedy = extra.cfg(b, g, scale, sf)
        want = client.cfg_logits(b, g, scale, sf)
        for k in range(len(b)):
            assert _same(out[k], want[k]), (scale, sf, k)
            assert greedy[k] == client.cfg_greedy(want[k]), (scale, sf, k)
        if sf == 1.0:
            assert 0 < np.isnan(out[2]).sum() < V and np.isnan(out[3]).all() and greedy[3] == 0
    # an all -inf input has no distribution: NaN row, id -1; a NaN or +inf input is refused
    ninf = np.full((1, V), -np.inf, np.float32)
    out, greedy = extra.cfg(ninf, g[:1], SCALE, SF)
    assert np.isnan(out).all() and greedy[0] == -1
    for bad in (np.nan, np.inf):
        x = b[:1].copy()
        x[0, 3] = bad
        with pytest.raises(capi.B200Error, match="non-finite"):
            extra.cfg(x, g[:1], SCALE, SF)
        with pytest.raises(capi.B200Error, match="non-finite"):
            extra.cfg(g[:1], x, SCALE, SF)


def _chain(paths, n_sessions=16, n_ctx=128):
    return [capi.Slice(p, 0, n_ctx, n_sessions=n_sessions) for p in paths]


def _gen(slices, extra, sessions, prompts, guids, negs, n, sampled, logprobs=None, first_draw=0, history=None,
         scale=SCALE, sf=SF):
    guidance = (guids, negs, scale, sf)
    if not sampled:
        return capi.generate_greedy(slices, extra, sessions, prompts, n, logprobs=logprobs, guidance=guidance)
    return capi.generate_sample(slices, extra, sessions, prompts, n, SAMPLED["temperature"], SAMPLED["repeat_penalty"],
                                [100 + k for k in sessions], first_draw=first_draw, history=history,
                                top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"], logprobs=logprobs, guidance=guidance)


def _clear(slices):
    for s in slices:
        s.session_clear(-1)


@pytest.mark.parametrize("sampled", [False, True])
def test_generate_cfg_equals_the_host_loop(tmp_path, sampled):
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    slices = _chain(paths)
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(5)
    sessions, guids = list(range(8)), list(range(8, 16))
    prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in (5, 1, 9, 3, 12, 2, 7, 4)]
    negs = [rng.integers(0, sh.n_vocab, n).tolist() for n in (3, 6, 1, 9, 2, 12, 4, 5)]
    n, n_top = 10, 5

    _clear(slices)
    ids8, lp8, ti8, tl8 = _gen(slices, extra, sessions, prompts, guids, negs, n, sampled, logprobs=n_top)
    for s in slices:                                                    # both contexts of every pair moved
        for k in range(8):
            assert s.session_n_past(k) == len(prompts[k]) + n - 1
            assert s.session_n_past(8 + k) == len(negs[k]) + n - 1
    _clear(slices)
    plain = _gen(slices, extra, sessions, prompts, guids, negs, n, sampled)
    assert np.array_equal(plain, ids8)                                  # logprobs change no id
    for k in (0, 4):                                                    # alone, other session numbers
        _clear(slices)
        one = _gen(slices, extra, [k], [prompts[k]], [15 - k], [negs[k]], n, sampled, logprobs=n_top)
        for j, arr in enumerate((ids8, lp8, ti8, tl8)):
            assert np.array_equal(one[j][:, 0], arr[:, k], equal_nan=True), (k, j)
    k, a = 4, 4                                                         # split across two calls
    _clear(slices)
    first = _gen(slices, extra, [k], [prompts[k]], [9], [negs[k]], a, sampled, logprobs=n_top)
    last = [int(first[0][-1, 0])]
    second = _gen(slices, extra, [k], [last], [9], [last], n - a, sampled, logprobs=n_top, first_draw=a,
                  history=[first[0][:, 0].tolist()] if sampled else None)
    for j, arr in enumerate((ids8, lp8, ti8, tl8)):
        assert np.array_equal(np.concatenate([first[j][:, 0], second[j][:, 0]]), arr[:, k], equal_nan=True), j

    # the host loop, fed the device's ids
    _clear(slices)
    toks, gtoks, base_rows = prompts[k], negs[k], []
    for j in range(n):
        xb, xg = extra.embed(toks), extra.embed(gtoks)
        for s in slices:
            xb, xg = s.session_forward(k, xb), s.session_forward(9, xg)
        b, g = extra.logits(xb[-1:])[0], extra.logits(xg[-1:])[0]
        row = client.cfg_logits(b[None], g[None], SCALE, SF)[0]
        if sampled:
            want = extra.sample(row[None], SAMPLED["temperature"], SAMPLED["repeat_penalty"], [100 + k], first_draw=j,
                                history=[ids8[:j, k].tolist()], top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"])[0]
        else:
            want = client.cfg_greedy(row)
        assert want == ids8[j, k], j
        base_rows.append(b)
        toks = gtoks = [int(ids8[j, k])]
    lp, ti, tl = extra.logprobs(np.array(base_rows), ids8[:, k].astype(np.int32), n_top)
    assert np.array_equal(lp, lp8[:, k]) and np.array_equal(ti, ti8[:, k]) and np.array_equal(tl, tl8[:, k])
    assert np.isfinite(lp8).all() and (lp8 <= 0).all()


def test_refusals_change_nothing(tmp_path):
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    slices = _chain(paths, n_ctx=64)
    extra = capi.Extra(extra_path, 0)
    _clear(slices)
    capi.generate_greedy(slices, extra, [0, 1], [[1, 2, 3], [4, 5]], 3, guidance=([2, 3], [[6], [7, 8]], SCALE, SF))
    before = [[s.session_save(k) for k in range(16)] for s in slices]
    n_past = [[s.session_n_past(k) for k in range(16)] for s in slices]
    V = sh.n_vocab
    bad = [
        ([0], [[1]], [0], [[2]], SCALE, SF, "also a listed session"),
        ([0, 1], [[1], [2]], [2, 2], [[2], [3]], SCALE, SF, "listed twice"),
        ([0], [[1]], [16], [[2]], SCALE, SF, "outside"),
        ([0], [[1]], [-1], [[2]], SCALE, SF, "outside"),
        ([0], [[1]], [2], [[]], SCALE, SF, "at least 1"),
        ([0], [[1]], [2], [[V]], SCALE, SF, "outside"),
        ([0], [[1]], [2], [[-1]], SCALE, SF, "outside"),
        ([0], [[1]], [2], [[2]], 1.0, SF, "scale"),
        ([0], [[1]], [2], [[2]], float("nan"), SF, "scale"),
        ([0], [[1]], [2], [[2]], SCALE, float("inf"), "smooth_factor"),
        ([0], [[1]], [2], [[2] * 60], SCALE, SF, "context overflow"),
        ([0], [[1]], [0, 2], [[2], [3]], SCALE, SF, "per listed session"),
    ]
    for ses, prm, gs, negs, scale, sf, msg in bad:
        with pytest.raises((capi.B200Error, ValueError), match=msg):
            capi.generate_greedy(slices, extra, ses, prm, 4, guidance=(gs, negs, scale, sf))
    with pytest.raises(capi.B200Error, match="context overflow"):
        capi.generate_greedy(slices, extra, [0], [[1]], 62, guidance=([2], [[2]], SCALE, SF))
    assert [[s.session_save(k) for k in range(16)] for s in slices] == before
    assert [[s.session_n_past(k) for k in range(16)] for s in slices] == n_past


def test_local_pipeline_cfg(tmp_path):
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    pipe = client.LocalPipeline(paths, devices=[0, 0], n_ctx=128, n_sessions=2)
    try:
        extra = pipe._device_extra(extra_path, "test")
        prompt, neg = "Hello world", "Goodbye"
        plain = pipe.generate_greedy(extra_path, prompt, 8)
        assert pipe.generate_greedy(extra_path, prompt, 8, cfg_negative_prompt=neg, cfg_scale=1.0) == plain
        got = pipe.generate_greedy(extra_path, prompt, 8, cfg_negative_prompt=neg, cfg_scale=2.5, cfg_smooth_factor=0.75)
        _clear(pipe.slices)
        want = capi.generate_greedy(pipe.slices, extra, [0], [extra.tokenize(prompt)], 8,
                                    guidance=([1], [extra.tokenize(neg)], 2.5, 0.75))[:, 0].tolist()
        assert got == want
        texts = list(pipe.generate(extra_path, prompt, 6, temperature=0.7, seed=3, cfg_negative_prompt=neg, cfg_scale=2.0))
        _clear(pipe.slices)
        ids = capi.generate_sample(pipe.slices, extra, [0], [extra.tokenize(prompt)], 6, 0.7, 1.1, [3],
                                   guidance=([1], [extra.tokenize(neg)], 2.0, 1.0))[:, 0]
        assert texts == [extra.token_text(int(t)) for t in ids]
    finally:
        pipe.close()
    one = client.LocalPipeline(paths, devices=[0, 0], n_ctx=64, n_sessions=1)
    try:
        with pytest.raises(ValueError, match="n_sessions >= 2"):
            one.generate_greedy(extra_path, "Hi", 4, cfg_negative_prompt="x", cfg_scale=2.0)
    finally:
        one.close()


def test_main_goldens(tmp_path):
    """Guided greedy generation fed the ids llama.cpp's main printed (tests/golden/cfg_main.json), on slices cut from the
    same model, prints main's text; where oracle/_ref/main exists it is also run now."""
    import json
    import os
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "golden"))
    import gen_golden_cfg as gen
    with open(os.path.join(here, "golden", "cfg_main.json")) as f:
        fx = json.load(f)
    full = str(tmp_path / "full.bin")
    assert gen.write_model(full) == fx["model_sha256"]
    sh = ggjt.SHAPES[gen.SHAPE]
    sl_path, extra_path = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl_path, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra_path)
    sl = capi.Slice(sl_path, 0, gen.N_CTX, n_sessions=2)
    extra = capi.Extra(extra_path, 0)
    live = os.path.isfile(gen.BINARY)
    for case in fx["cases"]:
        sl.session_clear(-1)
        ids = capi.generate_greedy([sl], extra, [0], [fx["prompt_ids"]], fx["n_predict"],
                                   guidance=([1], [fx["negative_ids"]], case["scale"], case["smooth_factor"]))[:, 0]
        assert "".join(extra.token_text(int(t)) for t in ids) == case["text"], case
        if live:
            p, n, text = gen.run_main(full, case["scale"], case["smooth_factor"])
            assert (p, n, text) == (fx["prompt_ids"], fx["negative_ids"], case["text"])
    extra.close()
    sl.close()


def _chunks(ids, C):
    """-> (non-final chunks, final chunk) of a prompt fed in chunks of C ids (C = 0: whole)."""
    if not C or len(ids) <= C:
        return [], list(ids)
    cut = [list(ids[i:i + C]) for i in range(0, len(ids), C)]
    return cut[:-1], cut[-1]


def _expect(slices, extra, k, prompt, n, C, sampled, seed, guide=None):
    """The stream contract for session k alone: session_forward of the non-final chunks, then the one-shot call with the
    final chunk(s).  -> (ids, lp)."""
    _clear(slices)
    heads, last = _chunks(prompt, C)
    for ch in heads:
        x = extra.embed(ch)
        for s in slices:
            x = s.session_forward(k, x)
    kw = dict(logprobs=2)
    if guide is not None:
        g, neg, scale, sf = guide
        gheads, glast = _chunks(neg, C)
        for ch in gheads:
            x = extra.embed(ch)
            for s in slices:
                x = s.session_forward(g, x)
        kw["guidance"] = ([g], [glast], scale, sf)
    if sampled:
        out = capi.generate_sample(slices, extra, [k], [last], n, SAMPLED["temperature"], SAMPLED["repeat_penalty"], [seed],
                                   top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"], **kw)
    else:
        out = capi.generate_greedy(slices, extra, [k], [last], n, **kw)
    return out[0][:, 0].tolist(), out[1][:, 0]


@pytest.mark.parametrize("C", [0, 3])
def test_stream_guided_sessions(tmp_path, C):
    """Guided pairs beside unguided sessions that join and leave: each session's ids and log-probabilities equal the
    one-shot contract; negative prompts longer and shorter than the prompt, and (C > 0) longer than max_rows."""
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(21 + C)
    max_rows = 32 if C == 0 else 8
    r = lambda n: rng.integers(0, sh.n_vocab, n).tolist()                               # noqa: E731
    # session -> (prompt, budget, sampled, guidance (g, neg, scale, sf) or None)
    plan = {0: (r(5), 9, False, (10, r(11 if C else 9), 1.75, 0.5)), 1: (r(9), 7, True, (11, r(2), 2.5, 1.0)),
            2: (r(4), 6, False, None), 3: (r(6), 8, True, None), 4: (r(3), 5, True, (12, r(13 if C else 4), 1.5, 0.0))}

    def add(st, k):
        prompt, budget, sampled, guide = plan[k]
        kw = dict(temperature=SAMPLED["temperature"], repeat_penalty=SAMPLED["repeat_penalty"], seed=100 + k,
                  top_k=SAMPLED["top_k"], top_p=SAMPLED["top_p"]) if sampled else {}
        st.add(k, prompt, budget, logprobs=2, guidance=guide, **kw)

    slices = _chain(paths)
    got = {}
    with capi.Stream(slices, extra, max_rows=max_rows, prefill_chunk=C) as st:
        for k in (0, 1, 2):
            add(st, k)
        with pytest.raises(capi.B200Error, match="guidance session of session 0"):
            st.add(10, [1], 2)
        with pytest.raises(capi.B200Error, match="guidance session of session 0"):
            st.cancel(10)
        with pytest.raises(capi.B200Error, match="guidance session of session 1"):
            st.fork(11, 13, 0)
        with pytest.raises(capi.B200Error, match="already in the stream"):
            st.add(5, [1], 2, guidance=(2, [3], 2.0, 1.0))
        recs = []
        while len(recs) < 6:
            recs += st.read_logprobs(3)
        add(st, 3)
        add(st, 4)
        while True:
            more = st.read_logprobs(4)
            if not more:
                break
            recs += more
        stats = st.stats()
    for rec in recs:
        got.setdefault(rec[0], []).append(rec[1:3])
    for k, (prompt, budget, sampled, guide) in plan.items():
        for s in slices:
            assert s.session_n_past(k) == len(prompt) + budget - 1
            if guide:
                assert s.session_n_past(guide[0]) == len(guide[1]) + budget - 1
    rows = sum(len(p) + b - 1 + (len(g[1]) + b - 1 if g else 0) for p, b, _, g in plan.values())
    assert stats["rows"] == rows, stats
    for k, (prompt, budget, sampled, guide) in plan.items():
        ids, lp = _expect(slices, extra, k, prompt, budget, C, sampled, 100 + k, guide)
        assert [t for t, _ in got[k]] == ids, k
        assert np.array_equal([v for _, v in got[k]], lp), k


def test_stream_cancel_mid_prefill(tmp_path):
    """A guided pair cancelled while its prompts are still being fed in chunks: both sessions are back where they were."""
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    extra = capi.Extra(extra_path, 0)
    slices = _chain(paths)
    _clear(slices)
    with capi.Stream(slices, extra, max_rows=5, prefill_chunk=2) as st:
        st.add(0, [5], 40)
        st.add(1, list(range(1, 30)), 4, guidance=(2, list(range(3, 40)), 2.0, 1.0))
        got = []
        while len(got) < 3:
            got += st.read(1)
        assert all(k == 0 for k, _ in got)
        st.cancel(1)
        st.cancel(0)
    for s in slices:
        assert s.session_n_past(1) == 0 and s.session_n_past(2) == 0 and s.session_n_past(0) == 3
