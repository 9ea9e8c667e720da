"""GPU: top-k / top-p truncation in the device sampler (sample_row's truncation stage, through k_sample_rows and
k_stream_draw) against the host twin client.Sampler(..., top_k, top_p) (tests/trunc_ref.py), and against the device's
own untruncated draws where the rule says nothing may change.

A device id may differ from the twin's only under the ambiguity rule of trunc_ref: u within 1e-9 of a boundary of the
twin's CDF, or the twin's mass before the last kept / first dropped id within 1e-9 S_K of top_p S_K.  Each test prints
how many draws were that close (expected: 0); a session is not compared past its first ambiguous draw.  On the device
itself there is no tolerance."""
import ctypes as C

import numpy as np
import pytest

import sample_ref
import trunc_ref
from distributedllm_b200 import ggjt
from test_gpu_generate import _model, _serve
from test_gpu_sample import RPS, TS, _raw_sample, _rows

pytestmark = pytest.mark.gpu


def _extra(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    path = str(tmp_path / "extra.bin")
    if n_vocab == 512:
        ggjt.write_synth_extra(path, ggjt.SHAPES["tiny128"], ggjt.T_Q4_0, seed=61)
    else:
        ggjt.write_fast_q4_extra(path, ggjt.SHAPES["3b"], seed=61)
    extra = capi.Extra(path, 0)
    assert extra.n_vocab == n_vocab
    return extra


def _edge_rows(rng, n):
    """-> (rows, histories): the edges of the rule."""
    rows, hist = [], []
    r = np.full(n, -1.0)
    ids = rng.permutation(n)
    r[ids[:30]] = 3.0
    r[ids[30:50]] = 2.0
    rows.append(r); hist.append([])                         # ties straddling rank 40 (and rank 2, 1000 ...)
    r = np.full(n, -5.0)
    r[ids[0]] = 5.0
    r[ids[1:101]] = 4.0
    rows.append(r); hist.append([])                         # a top-p cut inside a run of equal y
    r = rng.standard_normal(n) * 2
    top = int(np.argmax(r))
    r[top] += 6.0
    rows.append(r); hist.append([top])                      # a penalised id that would rank first without the penalty
    r = np.full(n, -np.inf)
    r[ids[:30]] = rng.standard_normal(30)
    rows.append(r); hist.append([])                         # fewer finite logits than top_k 40
    return rows, hist


def _settings(n):
    return [(1, 0.0), (2, 0.0), (40, 0.0), (1000, 0.0), (n, 0.0), (0, 1e-6), (0, 0.5), (0, 0.9), (0, 0.95), (0, 1.0),
            (40, 0.95), (2, 0.5), (1000, 0.9), (40, 1e-6), (n, 1.0)]


@pytest.mark.parametrize("n_vocab", [512, 32000])
def test_extra_sample_truncated_equals_the_twin(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    extra = _extra(tmp_path, n_vocab)
    rng = np.random.default_rng(n_vocab + 1)
    base = list(_rows(rng, n_vocab))
    edges, edge_hist = _edge_rows(rng, n_vocab)
    n_draws = ambiguous = 0
    for T in TS:
        for rp in RPS:
            for top_k, top_p in _settings(n_vocab):
                rows = np.asarray(base + edges, np.float32)
                hist = [rng.integers(0, n_vocab, int(rng.integers(0, 40))).tolist() for _ in base] + edge_hist
                seeds = [int(s) for s in rng.integers(0, 2 ** 63, len(rows), dtype=np.int64)]
                first_draw = int(rng.integers(0, 50))
                ids = extra.sample(rows, T, rp, seeds, first_draw, hist, top_k=top_k, top_p=top_p)
                for k in range(len(rows)):
                    want, amb, keep = trunc_ref.sample(rows[k], T, rp, hist[k], sample_ref.uniform(seeds[k], first_draw),
                                                       top_k, top_p)
                    n_draws += 1
                    assert 0 <= ids[k] < n_vocab and keep[ids[k]], (T, rp, top_k, top_p, k, int(ids[k]))
                    if amb:
                        ambiguous += 1
                        continue
                    assert ids[k] == want, (T, rp, top_k, top_p, k, int(ids[k]), want)
    print("n_vocab %d: %d draws, %d ambiguous" % (n_vocab, n_draws, ambiguous))
    # rows without a distribution still give the existing error
    for bad in (np.nan, np.inf):
        rows = np.asarray(base[:3], np.float32)
        rows[1, 7] = bad
        with pytest.raises(capi.B200Error) as ei:
            extra.sample(rows, 0.7, 1.1, [1, 2, 3], top_k=40, top_p=0.95)
        assert ei.value.code == 1 and "row 1" in str(ei.value)
    rows = np.asarray(base[:2], np.float32)
    rows[1] = -np.inf
    with pytest.raises(capi.B200Error) as ei:
        extra.sample(rows, 0.7, 1.1, [1, 2], top_k=40, top_p=0.95)
    assert ei.value.code == 1 and "row 1" in str(ei.value)
    extra.close()


@pytest.mark.parametrize("n_vocab", [512, 32000])
def test_truncation_that_drops_nothing_changes_no_bit(tmp_path, n_vocab):
    """Device against device: top_k = n_vocab with top_p = 1, and cuts that only drop ids of weight 0, give the
    untruncated ids; a row's id does not depend on its batch position."""
    extra = _extra(tmp_path, n_vocab)
    rng = np.random.default_rng(n_vocab + 2)
    for T, rp in ((0.7, 1.1), (1.0, 1.0), (5.0, 1.5)):
        for first_draw in range(0, 40, 3):
            rows = list(_rows(rng, n_vocab))
            n_fin = []
            for F in (1, 7, 40, 300):                        # F finite logits, the rest -inf (weight 0)
                r = np.full(n_vocab, -np.inf)
                r[rng.permutation(n_vocab)[:F]] = rng.standard_normal(F) * 3
                rows.append(r)
                n_fin.append(F)
            rows = np.asarray(rows, np.float32)
            seeds = [int(s) for s in rng.integers(0, 2 ** 63, len(rows), dtype=np.int64)]
            hist = [rng.integers(0, n_vocab, 20).tolist() for _ in rows]
            off = extra.sample(rows, T, rp, seeds, first_draw, hist)
            assert (extra.sample(rows, T, rp, seeds, first_draw, hist, top_k=n_vocab, top_p=1.0) == off).all()
            tail = len(rows) - len(n_fin)
            for j, F in enumerate(n_fin):
                r = rows[tail + j:tail + j + 1]
                for kw in (dict(top_k=F), dict(top_k=F + 5), dict(top_k=F, top_p=1.0)):
                    got = extra.sample(r, T, rp, seeds[tail + j:tail + j + 1], first_draw, hist[tail + j:tail + j + 1], **kw)
                    assert got[0] == off[tail + j], (T, rp, F, kw)
            # the same rows in another order and beside copies: the same ids
            perm = rng.permutation(len(rows))
            for kw in (dict(top_k=40, top_p=0.95), dict(top_p=0.5), dict(top_k=2)):
                a = extra.sample(rows, T, rp, seeds, first_draw, hist, **kw)
                idx = np.concatenate([perm, perm[:5]])
                b = extra.sample(rows[idx], T, rp, [seeds[i] for i in idx], first_draw, [hist[i] for i in idx], **kw)
                assert (b == a[idx]).all(), (T, rp, kw)
    extra.close()


def _host_loop(slices, extra, session, prompt, n_steps, T, rp, seed, top_k, top_p):
    """The client's loop through the host with client.Sampler(top_k, top_p) on Philox(key=seed): -> (ids, draws it
    is safe to compare)."""
    from distributedllm_b200.client import Sampler
    sampler = Sampler(T, rp, rng=np.random.Generator(np.random.Philox(key=seed)), top_k=top_k, top_p=top_p)
    ids, toks, safe = [], list(prompt), None
    for step in range(n_steps):
        x = extra.embed(toks)
        for s in slices:
            x = s.session_forward(session, x)
        logits = extra.logits(x)[-1]
        _, amb, _ = trunc_ref.sample(logits, T, rp, sampler.previous_ids, sample_ref.uniform(seed, step), top_k, top_p)
        if safe is None and amb:
            safe = step
        ids.append(sampler(logits))
        toks = [ids[-1]]
    return ids, n_steps if safe is None else safe


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
def test_generate_sample_truncated(tmp_path, kind):
    """top_k 40, top_p 0.95: the batch equals each session alone and the host loop with the twin, and a run split
    across calls continues exactly."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_sess, n_steps, K, P = 5, 12, 40, 0.95
    extra = capi.Extra(extra_path, 0)
    sessions, lengths = [3, 0, 4, 1, 2], [5, 1, 12, 3, 9]
    seeds = [11, 2 ** 63 + 5, 977, 3, 2 ** 40 + 1]
    T, rp = 0.9, 1.1
    gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    rng = np.random.default_rng(23)
    prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in lengths]
    ids = capi.generate_sample(gpu, extra, sessions, prompts, n_steps, T, rp, seeds, top_k=K, top_p=P)
    untrunc = capi.generate_sample(twin, extra, sessions, prompts, n_steps, T, rp, seeds)
    for s in twin:
        s.session_clear(-1)
    assert ids.tolist() != untrunc.tolist()                      # the cut changes some draws
    ambiguous = 0
    for j, k in enumerate(sessions):
        alone = capi.generate_sample(twin, extra, [k], [prompts[j]], n_steps, T, rp, [seeds[j]], top_k=K, top_p=P)[:, 0]
        assert alone.tolist() == ids[:, j].tolist(), (kind, k)
        for s in twin:
            s.session_rewind(k, 0)
        host, safe = _host_loop(twin, extra, k, prompts[j], n_steps, T, rp, seeds[j], K, P)
        assert host[:safe] == ids[:safe, j].tolist(), (kind, k)
        ambiguous += safe < n_steps
    print("%s: %d sessions stopped at an ambiguous draw" % (kind, ambiguous))
    # split runs: a steps, then n - a continued with the first ids as history and first_draw = a
    for a in (1, 6):
        for s in twin:
            s.session_clear(-1)
        first = capi.generate_sample(twin, extra, sessions, prompts, a, T, rp, seeds, top_k=K, top_p=P)
        rest = capi.generate_sample(twin, extra, sessions, [[int(t)] for t in first[-1]], n_steps - a, T, rp, seeds,
                                    first_draw=a, history=[first[:, j].tolist() for j in range(n_sess)], top_k=K, top_p=P)
        assert np.concatenate([first, rest]).tolist() == ids.tolist(), (kind, a)
    extra.close()
    for s in gpu + twin:
        s.close()


# session -> (temperature or None for greedy, repeat penalty, seed, top_k, top_p)
MODES = {0: (None, 1.1, 0, 0, 0.0), 1: (0.8, 1.1, 11, 40, 0.95), 2: (0.9, 1.3, 2 ** 63 + 5, 0, 0.0),
         3: (1.0, 1.0, 977, 0, 0.5), 4: (0.7, 1.1, 3, 5, 0.0), 5: (None, 1.1, 0, 0, 0.0), 6: (1.2, 1.2, 2 ** 40 + 1, 1000, 0.9)}


def _one_shot(capi, slices, extra, k, prompt, n):
    T, rp, seed, top_k, top_p = MODES[k]
    if T is None:
        return capi.generate_greedy(slices, extra, [k], [prompt], n)[:, 0].tolist()
    return capi.generate_sample(slices, extra, [k], [prompt], n, T, rp, [seed], top_k=top_k, top_p=top_p)[:, 0].tolist()


def _add(st, k, prompt, budget):
    T, rp, seed, top_k, top_p = MODES[k]
    if T is None:
        st.add(k, prompt, budget)
    else:
        st.add(k, prompt, budget, temperature=T, repeat_penalty=rp, seed=seed, top_k=top_k, top_p=top_p)


@pytest.mark.parametrize("kind", ["q4_0", "q4_K_M"])
def test_stream_mixing_greedy_untruncated_and_truncated_sessions(tmp_path, kind):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    gpu = [capi.Slice(p, 0, 128, n_sessions=8) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=8) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(44)
    plan = {0: (3, 20), 1: (17, 12), 2: (9, 25), 3: (5, 20), 4: (1, 30), 5: (12, 6), 6: (25, 15)}
    prompts = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, (n, _) in plan.items()}
    pairs = []
    with capi.Stream(gpu, extra, lookahead=2) as st:
        for k in (0, 1, 2):
            _add(st, k, prompts[k], plan[k][1])
        for pair in st:
            pairs.append(pair)
            if len(pairs) == 4:
                for k in (3, 4, 5):
                    _add(st, k, prompts[k], plan[k][1])
            if len(pairs) == 13:
                _add(st, 6, prompts[6], plan[6][1])
    got = {}
    for k, t in pairs:
        got.setdefault(k, []).append(t)
    for k, (n, budget) in plan.items():
        assert len(got[k]) == budget, k
        assert _one_shot(capi, twin, extra, k, prompts[k], budget) == got[k], (kind, k)
    assert [s.session_n_past(k) for s in gpu for k in plan] == [s.session_n_past(k) for s in twin for k in plan]
    extra.close()
    for s in gpu + twin:
        s.close()


def test_local_pipeline_generate_truncated_equals_the_node_path(tmp_path):
    """LocalPipeline.generate(top_k, top_p) (device stream) against DistributedLLM.generate(top_k, top_p) through a node
    (host loop, client.Sampler) with the same Philox key."""
    from distributedllm_b200.client import DistributedLLM, LocalPipeline
    from distributedllm_b200.compute_node.slices import import_llm
    from distributedllm_b200.control_center import Connection
    llm = import_llm()
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=0)
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    cases = [(4, 40, 0.95), (2 ** 63 + 1, 3, None), (9, None, 0.6)]
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        want = [list(DistributedLLM([addr], extra).generate("the the a in", 12, temperature=1.0, repeat_penalty=1.1,
                                                            rng=np.random.Generator(np.random.Philox(key=s)),
                                                            top_k=k, top_p=p))
                for s, k, p in cases]
    finally:
        srv.shutdown()
        srv.server_close()
        llm.unload_slice()
    lp = LocalPipeline([sl], [0])
    for (s, k, p), w in zip(cases, want):
        assert len(w) == 12
        assert list(lp.generate(extra, "the the a in", 12, temperature=1.0, repeat_penalty=1.1, seed=s, top_k=k,
                                top_p=p)) == w, (s, k, p)
    lp.close()


def test_bad_truncation_settings_are_refused_and_move_nothing(tmp_models, tmp_path):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=45), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=45)]
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=45)
    extra = capi.Extra(extra_path, 0)
    x = extra.embed(list(range(3, 13)))
    for s in gpu:
        x = s.session_forward(1, x)

    def positions():
        return [s.session_n_past(k) for s in gpu for k in range(3)]

    before = positions()
    keys = np.array([1, 2], np.uint64)
    bad = [dict(top_k=-1), dict(top_k=-2 ** 31), dict(top_p=-0.5), dict(top_p=float("nan")), dict(top_p=-float("inf"))]
    for kw in bad:
        sp = capi.Sampling(temperature=0.7, repeat_penalty=1.1, seeds=keys.ctypes.data, first_draw=0, **kw)
        assert _raw_sample(gpu, extra, [0, 1], [[1, 2], [3]], 4, sp) == 1, kw
        assert positions() == before, kw
    with capi.Stream(gpu, extra) as st:
        prompt = np.array([1, 2], np.int32)
        for kw in bad:
            sp = capi.Sampling(temperature=0.7, repeat_penalty=1.1, seeds=keys.ctypes.data, first_draw=0, **kw)
            rc = capi.lib().b200_stream_add(st._handle(), 0, capi._ptr(prompt), 2, 4, C.byref(sp), None, 0)
            assert rc == 1, kw
        assert st.read(8) == []                                  # nothing was queued
    assert positions() == before
    # accepted: large top_k, top_p above 1 and infinite
    ok = capi.generate_sample(gpu, extra, [0, 2], [[1, 2], [3]], 3, 0.7, 1.1, [1, 2], top_k=10 ** 6, top_p=float("inf"))
    assert ok.shape == (3, 2) and (ok >= 0).all()
    extra.close()
    for s in gpu:
        s.close()
