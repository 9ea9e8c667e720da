"""GPU: the client's Sampler on the device (k_sample_rows): b200_extra_sample against the explicit-draw host twin
(tests/sample_ref.py), and b200_generate_sample against single-session runs, split runs and the host loop with
client.Sampler on a Philox generator.

The first step of the rule (y = x / d in float64) is correctly rounded on both sides; the last ulp of float64 exp and the
summation order are not.  So a device id may differ from the host twin only where u lies within ~1e-12 of a boundary of
the host's CDF: ids must be equal whenever u is more than sample_ref.AMBIGUOUS = 1e-9 from every boundary, and each
test prints how many draws were that close (expected: 0).  On the device itself there is no tolerance."""
import ctypes as C

import numpy as np
import pytest

import sample_ref
from distributedllm_b200 import ggjt
from test_gpu_generate import _bits, _host_step, _model, _serve

pytestmark = pytest.mark.gpu
TS = (0.0, 0.2, 0.7, 1.0, 5.0)
RPS = (1.0, 1.1, 1.5)


def _rows(rng, n_vocab):
    """Logit rows of every kind the sampler meets: normal at three scales, exact ties, one-hot, -inf entries."""
    rows = []
    for scale in (0.5, 3.0, 10.0):
        rows.append(rng.standard_normal(n_vocab) * scale)
    rows.append(np.round(rng.standard_normal(n_vocab) * 2) / 2)          # many exact ties
    r = np.zeros(n_vocab)
    r[:] = 1.25
    rows.append(r)                                                        # all tied
    r = np.zeros(n_vocab)
    r[int(rng.integers(0, n_vocab))] = 4.0
    rows.append(r)                                                        # one-hot over zeros
    r = np.full(n_vocab, -np.inf)
    r[int(rng.integers(0, n_vocab))] = -3.0
    rows.append(r)                                                        # one finite id, the rest -inf
    r = rng.standard_normal(n_vocab) * 3
    r[rng.random(n_vocab) < 0.5] = -np.inf
    rows.append(r)                                                        # half -inf
    r = -np.abs(rng.standard_normal(n_vocab)) * 2
    rows.append(r)                                                        # all negative (penalised ids rise)
    return np.asarray(rows, np.float32)


@pytest.mark.parametrize("n_vocab", [512, 32000])
def test_extra_sample_equals_the_host_twin(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    path = str(tmp_path / "extra.bin")
    if n_vocab == 512:
        ggjt.write_synth_extra(path, ggjt.SHAPES["tiny128"], ggjt.T_Q4_0, seed=60)
    else:
        ggjt.write_fast_q4_extra(path, ggjt.SHAPES["3b"], seed=60)
    extra = capi.Extra(path, 0)
    assert extra.n_vocab == n_vocab
    rng = np.random.default_rng(n_vocab)
    base = _rows(rng, n_vocab)
    n_draws = ambiguous = 0
    for T in TS:
        for rp in RPS:
            for first_draw in (0, 1, 2, 3, 5, 6, 9, 2 ** 40 + 3):
                rows = base[rng.permutation(len(base))]
                seeds = [int(s) for s in rng.integers(0, 2 ** 63, len(rows), dtype=np.int64)]
                seeds[0] += 2 ** 63                                  # a key >= 2^63
                sizes = [(0, 1, 300)[(k + first_draw) % 3] for k in range(len(rows))]
                history = [rng.integers(0, n_vocab, n).tolist() for n in sizes]
                ids = extra.sample(rows, T, rp, seeds, first_draw, history)
                for k in range(len(rows)):
                    u = sample_ref.uniform(seeds[k], first_draw)
                    want, margin, _ = sample_ref.sample(rows[k], T, rp, history[k], u)
                    p, _ = sample_ref.cdf_of(rows[k], T, rp, history[k])
                    assert 0 <= ids[k] < n_vocab and p[ids[k]] > 0, (T, rp, first_draw, k, int(ids[k]))   # never p = 0
                    n_draws += 1
                    if margin <= sample_ref.AMBIGUOUS:
                        ambiguous += 1
                        continue
                    assert ids[k] == want, (T, rp, first_draw, k, margin)
    print("n_vocab %d: %d draws, %d ambiguous" % (n_vocab, n_draws, ambiguous))
    assert n_draws >= 1000
    # logits numpy rejects ("probabilities contain NaN")
    for bad in (np.nan, np.inf):
        rows = base[:3].copy()
        rows[1, 7] = bad
        with pytest.raises(capi.B200Error) as ei:
            extra.sample(rows, 0.7, 1.1, [1, 2, 3])
        assert ei.value.code == 1 and "row 1" in str(ei.value)
    rows = base[:2].copy()
    rows[1] = -np.inf
    with pytest.raises(capi.B200Error) as ei:
        extra.sample(rows, 0.7, 1.1, [1, 2])
    assert ei.value.code == 1 and "row 1" in str(ei.value)
    assert extra.sample(base[:2], 0.7, 1.1, [1, 2]).shape == (2,)      # the handle still works
    extra.close()


def _host_loop(slices, extra, session, prompt, n_steps, T, rp, seed):
    """The client's loop through the host with client.Sampler on Philox(key=seed): -> (ids, draws it is safe to
    compare: up to the first ambiguous one)."""
    from distributedllm_b200.client import Sampler
    sampler = Sampler(T, rp, rng=np.random.Generator(np.random.Philox(key=seed)))
    ids, toks, safe = [], list(prompt), None
    for step in range(n_steps):
        x = extra.embed(toks)
        for s in slices:
            x = s.session_forward(session, x)
        logits = extra.logits(x)[-1]
        _, margin, _ = sample_ref.sample(logits, T, rp, sampler.previous_ids, sample_ref.uniform(seed, step))
        if safe is None and margin <= sample_ref.AMBIGUOUS:
            safe = step
        ids.append(sampler(logits))
        toks = [ids[-1]]
    return ids, n_steps if safe is None else safe


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
def test_sessions_equal_single_session_runs_and_the_host_loop(tmp_path, kind):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_sess, n_steps = 5, 12
    extra = capi.Extra(extra_path, 0)
    sessions = [3, 0, 4, 1, 2]
    lengths = [5, 1, 12, 3, 9]
    distinct = {}
    for T, rp in ((0.8, 1.1), (0.0, 1.1)):
        gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
        twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
        rng = np.random.default_rng(17)
        for sess, n in ((1, 7), (3, 20)):              # mid-context sessions: the same history on both handle sets
            pre = rng.integers(0, sh.n_vocab, n).tolist()
            for hs in (gpu, twin):
                x = extra.embed(pre)
                for s in hs:
                    x = s.session_forward(sess, x)
        prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in lengths]
        seeds = [11, 2 ** 63 + 5, 977, 3, 2 ** 40 + 1]
        before = [s.session_n_past(k) for s in gpu for k in range(n_sess)]
        ids = capi.generate_sample(gpu, extra, sessions, prompts, n_steps, T, rp, seeds)
        assert ids.shape == (n_steps, len(sessions))
        for s in gpu:
            for j, k in enumerate(sessions):
                assert s.session_n_past(k) == before[k] + lengths[j] + n_steps - 1
        ambiguous = 0
        for j, k in enumerate(sessions):
            start = twin[0].session_n_past(k)
            alone = capi.generate_sample(twin, extra, [k], [prompts[j]], n_steps, T, rp, [seeds[j]])[:, 0]
            assert alone.tolist() == ids[:, j].tolist(), (kind, T, k)
            for s in twin:
                s.session_rewind(k, start)
            host, safe = _host_loop(twin, extra, k, prompts[j], n_steps, T, rp, seeds[j])
            assert host[:safe] == ids[:safe, j].tolist(), (kind, T, k)
            if safe < n_steps:
                ambiguous += 1
                continue
            # the positions the loop left behind: one more host step on each handle set gives the same bits
            a = _host_step(gpu, extra, k, int(ids[-1, j]))
            b = _host_step(twin, extra, k, host[-1])
            assert (_bits(a) == _bits(b)).all(), (kind, T, k)
        print("%s T=%g rp=%g: %d sessions stopped at an ambiguous draw" % (kind, T, rp, ambiguous))
        # five fresh sessions with one prompt and five keys: sampling at T 0.8 gives more distinct id sequences than
        # T 0, where the 1e-5 divisor leaves the argmax (with the penalty) whatever the key
        for s in gpu:
            s.session_clear(-1)
        same = capi.generate_sample(gpu, extra, list(range(n_sess)), [prompts[0]] * n_sess, 6, T, rp, seeds)
        distinct[T] = len({tuple(same[:, j].tolist()) for j in range(n_sess)})
        for s in gpu + twin:
            s.close()
    assert distinct[0.8] > distinct[0.0], distinct
    extra.close()


def test_split_calls_equal_one_call(tmp_path):
    """n steps in one call are identical to a steps, then n - a steps continued from the last id, the first call's ids
    as history and first_draw = a."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    extra = capi.Extra(extra_path, 0)
    one = [capi.Slice(p, 0, 128, n_sessions=3) for p in paths]
    two = [capi.Slice(p, 0, 128, n_sessions=3) for p in paths]
    rng = np.random.default_rng(5)
    sessions, prompts, seeds = [2, 0, 1], [rng.integers(0, sh.n_vocab, n).tolist() for n in (4, 9, 1)], [8, 9, 2 ** 64 - 1]
    n = 14
    for T, rp in ((0.9, 1.3), (0.0, 1.1)):
        for s in one + two:
            s.session_clear(-1)
        full = capi.generate_sample(one, extra, sessions, prompts, n, T, rp, seeds)
        for a in (1, 6):
            for s in two:
                s.session_clear(-1)
            first = capi.generate_sample(two, extra, sessions, prompts, a, T, rp, seeds)
            rest = capi.generate_sample(two, extra, sessions, [[int(t)] for t in first[-1]], n - a, T, rp, seeds,
                                        first_draw=a, history=[first[:, j].tolist() for j in range(len(sessions))])
            assert np.concatenate([first, rest]).tolist() == full.tolist(), (T, a)
            assert [s.session_n_past(k) for s in two for k in sessions] == [s.session_n_past(k) for s in one for k in sessions]
    extra.close()
    for s in one + two:
        s.close()


def _raw_sample(slices, extra, sessions, prompts, n_steps, sp):
    from distributedllm_b200 import capi
    ids = np.ascontiguousarray(sessions, dtype=np.int32)
    counts = np.array([len(p) for p in prompts], np.int32)
    toks = np.ascontiguousarray([t for p in prompts for t in p] or [0], dtype=np.int32)
    handles = (C.c_void_p * len(slices))(*[s.handle for s in slices])
    out = np.zeros((max(n_steps, 1), len(ids)), np.int32)
    return capi.lib().b200_generate_sample(handles, len(slices), extra.handle, capi._ptr(ids), capi._ptr(counts), len(ids),
                                            capi._ptr(toks), n_steps, None if sp is None else C.byref(sp), capi._ptr(out))


def test_errors_change_nothing(tmp_models, tmp_path):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=45), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=45)]
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=45)
    extra = capi.Extra(extra_path, 0)
    other_path = str(tmp_path / "other.bin")           # n_embd 256
    ggjt.write_synth_slice(other_path, ggjt.SHAPES["tiny"], 0, 0, ggjt.T_Q4_0, seed=45)
    other = capi.Slice(other_path, 0, 64)
    gap = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 2, 2, seed=45), 0, 64)
    pre = list(range(3, 53))                            # session 1 at n_past 50
    x = extra.embed(pre)
    for s in gpu:
        x = s.session_forward(1, x)

    def positions():
        return [s.session_n_past(k) for s in gpu for k in range(3)]

    before = positions()
    V = sh.n_vocab
    cases = [
        ("slices out of layer order", [gpu[1], gpu[0]], [0], [[1, 2]], 4, 1),
        ("a gap in the layers", [gpu[0], gap], [0], [[1, 2]], 4, 1),
        ("another n_embd", [other], [0], [[1, 2]], 4, 1),
        ("a handle listed twice", [gpu[0], gpu[0]], [0], [[1, 2]], 4, 1),
        ("session out of range", gpu, [3], [[1, 2]], 4, 1),
        ("session listed twice", gpu, [0, 0], [[1, 2], [3]], 4, 1),
        ("empty prompt", gpu, [0, 2], [[1, 2], []], 4, 1),
        ("negative token", gpu, [0], [[1, -1]], 4, 1),
        ("token past the vocabulary", gpu, [0], [[V]], 4, 1),
        ("no steps", gpu, [0], [[1, 2]], 0, 1),
        ("context overflow", gpu, [0, 1], [[1, 2], [5, 6, 7, 8, 9]], 11, 5),
        ("prompt overflow", gpu, [1], [[1] * 15], 1, 5),
    ]
    for what, slices, sessions, prompts, n_steps, code in cases:
        with pytest.raises(capi.B200Error) as ei:
            capi.generate_sample(slices, extra, sessions, prompts, n_steps, 0.7, 1.1, [1] * len(sessions))
        assert ei.value.code == code, (what, str(ei.value))
        assert positions() == before, what
    keys = np.array([1, 2], np.uint64)
    hist = np.array([3, 4, 5], np.int32)

    def sp(**kw):
        f = dict(temperature=0.7, repeat_penalty=1.1, seeds=keys.ctypes.data, first_draw=0, history=None,
                 history_counts=None)
        f.update(kw)
        return capi.Sampling(**f)

    ones, neg_count = np.array([1, 1], np.int32), np.array([-1, 1], np.int32)
    bad_hist, neg_hist = np.array([3, V], np.int32), np.array([-1, 4], np.int32)
    new_cases = [
        ("null settings", None),
        ("null seeds", sp(seeds=None)),
        ("negative temperature", sp(temperature=-0.1)),
        ("NaN temperature", sp(temperature=float("nan"))),
        ("infinite temperature", sp(temperature=float("inf"))),
        ("zero penalty", sp(repeat_penalty=0.0)),
        ("negative penalty", sp(repeat_penalty=-1.1)),
        ("NaN penalty", sp(repeat_penalty=float("nan"))),
        ("infinite penalty", sp(repeat_penalty=float("inf"))),
        ("negative first draw", sp(first_draw=-1)),
        ("history without counts", sp(history=hist.ctypes.data)),
        ("negative history count", sp(history=hist.ctypes.data, history_counts=neg_count.ctypes.data)),
        ("history id past the vocabulary", sp(history=bad_hist.ctypes.data, history_counts=ones.ctypes.data)),
        ("negative history id", sp(history=neg_hist.ctypes.data, history_counts=ones.ctypes.data)),
    ]
    for what, settings in new_cases:
        rc = _raw_sample(gpu, extra, [0, 2], [[1, 2], [3]], 4, settings)
        assert rc == 1, (what, rc)
        assert positions() == before, what
    # a valid call with a history moves the positions as generate_greedy does
    ok = capi.generate_sample(gpu, extra, [0, 2], [[1, 2], [3]], 4, 0.7, 1.1, [1, 2], history=[[3, 4], [5]])
    assert ok.shape == (4, 2) and (ok >= 0).all()
    assert gpu[0].session_n_past(0) == 5 and gpu[1].session_n_past(2) == 4
    # an extra-layers file whose norm.weight holds a NaN: every logit is NaN from step 0.  Its output.weight is F16, whose
    # lm_head multiplies in float; a quantised one would round the NaN activation to the code 0 in its Q8_0 pre-pass.
    nan_path = str(tmp_path / "extra_nan.bin")
    ggjt.write_synth_extra(nan_path, sh, ggjt.T_F16, seed=45)
    norm = next(raw for name, _, _, raw in ggjt.synth_extra_tensors(sh, ggjt.T_F16, 45) if name == "norm.weight")
    data = bytearray(open(nan_path, "rb").read())
    at = bytes(data).index(norm) + 4 * 3
    data[at:at + 4] = np.array([np.nan], np.float32).tobytes()
    open(nan_path, "wb").write(bytes(data))
    nan_extra = capi.Extra(nan_path, 0)
    for s in gpu:
        s.session_clear(-1)
    with pytest.raises(capi.B200Error) as ei:
        capi.generate_sample(gpu, nan_extra, [2, 0], [[1, 2], [3]], 3, 0.7, 1.1, [1, 2])
    assert ei.value.code == 1 and "step 0 session 2" in str(ei.value), str(ei.value)
    assert gpu[0].session_n_past(2) == 4                                # the loop ran on: positions have moved
    nan_extra.close()
    extra.close()
    for s in [other, gap] + gpu:
        s.close()


def test_local_pipeline_generate_equals_the_node_path(tmp_path):
    """LocalPipeline.generate (device loop) against DistributedLLM.generate through a node (host loop, client.Sampler)
    with the same Philox key."""
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
    seeds = (4, 2 ** 63 + 1)
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        want = [list(DistributedLLM([addr], extra).generate("the the a in", 12, temperature=0.8, repeat_penalty=1.1,
                                                            rng=np.random.Generator(np.random.Philox(key=s))))
                for s in seeds]
    finally:
        srv.shutdown()
        srv.server_close()
        llm.unload_slice()
    lp = LocalPipeline([sl], [0])
    for s, w in zip(seeds, want):
        assert len(w) == 12
        assert list(lp.generate(extra, "the the a in", 12, temperature=0.8, repeat_penalty=1.1, seed=s)) == w
    assert lp.slices[0].n_past == len(llm.tokenize_prompt(extra, "the the a in")) + 11
    assert len(list(lp.generate(extra, "the the a in", 5, temperature=0.8))) == 5       # unseeded
    lp.close()
