"""GPU: generation streams (b200_stream_*, capi.Stream).  Every session's ids must equal b200_generate_greedy /
b200_generate_sample for that session alone, bit for bit, whatever joined, ran beside it or left; and its positions must
follow the position rule (old + n_prompt + delivered - 1), so that a continuation call picks up exactly where the stream
stopped."""
import numpy as np
import pytest

from distributedllm_b200 import ggjt
from test_gpu_generate import _model, _serve

pytestmark = pytest.mark.gpu

# session -> (temperature or None for greedy, repeat penalty, seed)
MODES = {0: (None, 1.1, 0), 1: (0.8, 1.1, 11), 2: (0.0, 1.3, 2 ** 63 + 5), 3: (None, 1.1, 0), 4: (1.0, 1.0, 977),
         5: (0.5, 1.5, 3), 6: (None, 1.1, 0), 7: (0.9, 1.2, 2 ** 40 + 1), 8: (0.7, 1.1, 8), 9: (None, 1.1, 0)}


def _one_shot(capi, slices, extra, k, prompt, n, mode, first_draw=0, history=None):
    T, rp, seed = mode
    if T is None:
        return capi.generate_greedy(slices, extra, [k], [prompt], n)[:, 0].tolist()
    return capi.generate_sample(slices, extra, [k], [prompt], n, T, rp, [seed], first_draw=first_draw,
                                history=None if history is None else [history])[:, 0].tolist()


def _add(st, k, prompt, budget, mode, stops=()):
    T, rp, seed = mode
    st.add(k, prompt, budget, temperature=T, repeat_penalty=rp, seed=seed, stop_ids=stops)


def _by_session(pairs):
    out = {}
    for k, t in pairs:
        out.setdefault(k, []).append(t)
    return out


def _prefill(extra, handle_sets, session, tokens):
    for hs in handle_sets:
        x = extra.embed(tokens)
        for s in hs:
            x = s.session_forward(session, x)


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
@pytest.mark.parametrize("sampled", [False, True])
def test_static_stream_equals_one_call(tmp_path, kind, sampled):
    """Every session added before the first read, no stops: ids and positions equal one generate_greedy /
    generate_sample call over the same lists."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_sess, n_steps = 5, 10
    gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(27)
    _prefill(extra, (gpu, twin), 3, rng.integers(0, sh.n_vocab, 20).tolist())      # one session mid-context
    sessions, lengths = [3, 0, 4, 1, 2], [5, 1, 12, 3, 9]
    prompts = [rng.integers(0, sh.n_vocab, n).tolist() for n in lengths]
    seeds = [11, 2 ** 63 + 5, 977, 3, 2 ** 40 + 1]
    T, rp = 0.8, 1.1
    if sampled:
        want = capi.generate_sample(twin, extra, sessions, prompts, n_steps, T, rp, seeds)
    else:
        want = capi.generate_greedy(twin, extra, sessions, prompts, n_steps)
    with capi.Stream(gpu, extra) as st:
        for j, k in enumerate(sessions):
            st.add(k, prompts[j], n_steps, temperature=T if sampled else None, repeat_penalty=rp, seed=seeds[j])
        pairs = st.read(1000)
        while True:
            more = st.read(1000)
            if not more:
                break
            pairs += more
    got = _by_session(pairs)
    for j, k in enumerate(sessions):
        assert got[k] == want[:, j].tolist(), (kind, sampled, k)
    assert len(pairs) == n_steps * len(sessions)
    assert [s.session_n_past(k) for s in gpu for k in range(n_sess)] == [s.session_n_past(k) for s in twin for k in range(n_sess)]
    assert len(set(want.ravel().tolist())) > 3
    extra.close()
    for s in gpu + twin:
        s.close()


def _join_and_leave(capi, gpu, twin, extra, sh, seed):
    """Sessions join after 0, 3 and 11 pairs (prompts of 1 to 40 ids, budgets of 6 to 40, greedy and sampled sessions
    with different T and rp), and one prompt joins while 7 sessions decode.  -> nothing; asserts."""
    rng = np.random.default_rng(seed)
    _prefill(extra, (gpu, twin), 2, rng.integers(0, sh.n_vocab, 13).tolist())
    _prefill(extra, (gpu, twin), 5, rng.integers(0, sh.n_vocab, 7).tolist())
    plan = {0: (1, 30), 1: (17, 12), 2: (40, 25), 3: (5, 20), 4: (9, 40), 5: (2, 6), 6: (33, 15), 7: (28, 10)}
    prompts = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, (n, _) in plan.items()}
    start = {k: [s.session_n_past(k) for s in gpu] for k in plan}
    pairs = []
    with capi.Stream(gpu, extra, lookahead=2) as st:
        for k in (0, 1, 2):
            _add(st, k, prompts[k], plan[k][1], MODES[k])
        for pair in st:
            pairs.append(pair)
            if len(pairs) == 3:
                for k in (3, 4, 5, 6):
                    _add(st, k, prompts[k], plan[k][1], MODES[k])
            if len(pairs) == 11:
                _add(st, 7, prompts[7], plan[7][1], MODES[7])
    got = _by_session(pairs)
    first7 = [i for i, (k, _) in enumerate(pairs) if k == 7][0]
    assert sorted(k for k, _ in pairs[first7 - 7:first7]) == list(range(7)), pairs[first7 - 8:first7 + 1]
    for k, (n, budget) in plan.items():
        assert len(got[k]) == budget, k
        assert [s.session_n_past(k) for s in gpu] == [p + n + budget - 1 for p in start[k]], k
        assert [s.session_n_past(k) for s in twin] == start[k]
        assert _one_shot(capi, twin, extra, k, prompts[k], budget, MODES[k]) == got[k], k
    assert [s.session_n_past(k) for s in gpu for k in plan] == [s.session_n_past(k) for s in twin for k in plan]


@pytest.mark.parametrize("kind", ["q4_0", "q4_K_M"])
def test_join_and_leave(tmp_path, kind):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    gpu = [capi.Slice(p, 0, 128, n_sessions=10) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=10) for p in paths]
    extra = capi.Extra(extra_path, 0)
    _join_and_leave(capi, gpu, twin, extra, sh, 31)
    extra.close()
    for s in gpu + twin:
        s.close()


def test_join_and_leave_at_7b_layer_shape(tmp_path):
    """The same schedule on one LLaMA-7B-shape Q4_0 layer with a 32000 x 4096 Q6_K lm_head."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    path, extra_path = str(tmp_path / "layer.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=51)
    ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=51)
    gpu = [capi.Slice(path, 0, 128, n_sessions=10)]
    twin = [capi.Slice(path, 0, 128, n_sessions=10)]
    extra = capi.Extra(extra_path, 0)
    _join_and_leave(capi, gpu, twin, extra, sh, 32)
    extra.close()
    for s in gpu + twin:
        s.close()


@pytest.mark.parametrize("k", [0, 1])     # greedy, sampled
def test_stops_end_the_session_and_a_continuation_resumes(tmp_path, k):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 128, n_sessions=3) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=3) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(40 + k)
    prompt, other = rng.integers(0, sh.n_vocab, 6).tolist(), rng.integers(0, sh.n_vocab, 4).tolist()
    n = 24
    full = _one_shot(capi, twin, extra, k, prompt, n, MODES[k])
    stop = full[9]
    cut = full.index(stop) + 1                             # the first occurrence ends the run, inclusive
    absent = [t for t in range(sh.n_vocab) if t not in full][:2]
    with capi.Stream(gpu, extra) as st:
        _add(st, k, prompt, n, MODES[k], stops=[absent[0], stop, absent[1]])
        _add(st, 2, other, n, MODES[4])                    # a neighbour with no stop runs its whole budget
        got = _by_session(list(st))
    assert got[k] == full[:cut] and len(got[2]) == n
    assert [s.session_n_past(k) for s in gpu] == [len(prompt) + cut - 1] * len(gpu)
    rest = _one_shot(capi, gpu, extra, k, [got[k][-1]], n - cut, MODES[k], first_draw=cut, history=got[k])
    assert got[k] + rest == full
    assert [s.session_n_past(k) for s in gpu] == [s.session_n_past(k) for s in twin]
    assert _one_shot(capi, twin, extra, 2, other, n, MODES[4]) == got[2]
    extra.close()
    for s in gpu + twin:
        s.close()


def test_cancel_and_early_close(tmp_path):
    """After r ids of a session have been read, cancel (or close) leaves its positions at old + n_prompt + r - 1, and a
    continuation equals the uninterrupted run: steps the device ran ahead of the caller leave no trace."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 128, n_sessions=4) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=4) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(50)
    prompts = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, n in ((0, 7), (1, 3), (2, 11), (3, 5))}
    modes = {0: MODES[1], 1: MODES[0], 2: MODES[4], 3: MODES[5]}
    n = 30
    full = {k: _one_shot(capi, twin, extra, k, prompts[k], n, modes[k]) for k in prompts}
    for s in twin:
        s.session_clear(-1)
    read, cancelled = [], False
    with capi.Stream(gpu, extra, lookahead=6) as st:
        for k in (0, 1, 2):
            _add(st, k, prompts[k], n, modes[k])
        st.cancel(2)                                       # queued, never run: positions untouched
        for pair in st:
            read.append(pair)
            got = _by_session(read)
            if not cancelled and len(got.get(0, [])) == 4:
                st.cancel(0)                               # the device has run steps ahead for it
                cancelled = True
                _add(st, 3, prompts[3], n, modes[3])
            if len(got.get(1, [])) == 16:
                break
    # the stream closed with session 1 after 16 ids and session 3 part-way; the device had run steps ahead of both
    got = _by_session(read)
    assert got[0] == full[0][:4] and got[1] == full[1][:16] and 2 not in got
    assert got[3] == full[3][:len(got[3])]
    for k in (0, 1, 3):
        r = len(got[k])
        want = len(prompts[k]) + r - 1 if r else 0
        assert [s.session_n_past(k) for s in gpu] == [want] * len(gpu), k
        if r:
            rest = _one_shot(capi, gpu, extra, k, [got[k][-1]], n - r, modes[k], first_draw=r, history=got[k])
            assert got[k] + rest == full[k], k
    assert [s.session_n_past(2) for s in gpu] == [0, 0]
    extra.close()
    for s in gpu + twin:
        s.close()


def _nan_extra(tmp_path, sh):
    """An extra-layers file whose norm.weight holds a NaN: every logit is NaN (as tests/test_gpu_sample.py builds it)."""
    path = str(tmp_path / "extra_nan.bin")
    ggjt.write_synth_extra(path, sh, ggjt.T_F16, seed=45)
    norm = next(raw for name, _, _, raw in ggjt.synth_extra_tensors(sh, ggjt.T_F16, 45) if name == "norm.weight")
    data = bytearray(open(path, "rb").read())
    at = bytes(data).index(norm) + 4 * 3
    data[at:at + 4] = np.array([np.nan], np.float32).tobytes()
    open(path, "wb").write(bytes(data))
    return path


def test_errors_change_nothing(tmp_models, tmp_path):
    import ctypes as C
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=45), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=45)]
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    twin = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=45)
    extra = capi.Extra(extra_path, 0)
    _prefill(extra, (gpu, twin), 1, list(range(3, 53)))   # session 1 at n_past 50
    V, lib = sh.n_vocab, capi.lib()

    def positions(hs):
        return [s.session_n_past(k) for s in hs for k in range(3)]

    before = positions(gpu)
    st = capi.Stream(gpu, extra, max_rows=8)
    keys, hist = np.array([5], np.uint64), np.array([3, 4], np.int32)

    def sp(**kw):
        f = dict(temperature=0.7, repeat_penalty=1.1, seeds=keys.ctypes.data, first_draw=0, history=hist.ctypes.data,
                 history_counts=np.array([2], np.int32).ctypes.data)
        f.update(kw)
        return capi.Sampling(**f)

    def raw_add(session, prompt, max_tokens, settings=None, stops=()):
        p = np.array(prompt or [0], np.int32)
        s = np.array(list(stops) or [0], np.int32)
        return lib.b200_stream_add(st._h, session, capi._ptr(p), len(prompt), max_tokens,
                                   None if settings is None else C.byref(settings), capi._ptr(s), len(stops))

    assert raw_add(0, [1, 2], 4) == 0                     # session 0 is in the stream from here on
    bad_hist, bad_counts = np.array([3, V], np.int32), np.array([2], np.int32)
    cases = [
        ("session out of range", 1, (3, [1, 2], 4)),
        ("negative session", 1, (-1, [1, 2], 4)),
        ("session already in the stream", 1, (0, [1, 2], 4)),
        ("empty prompt", 1, (2, [], 4)),
        ("prompt past max_rows", 1, (2, [1] * 9, 4)),
        ("token past the vocabulary", 1, (2, [1, V], 4)),
        ("negative token", 1, (2, [-1], 4)),
        ("no tokens to draw", 1, (2, [1], 0)),
        ("stop id past the vocabulary", 1, (2, [1], 4, None, [2, V])),
        ("negative temperature", 1, (2, [1], 4, sp(temperature=-1.0))),
        ("NaN penalty", 1, (2, [1], 4, sp(repeat_penalty=float("nan")))),
        ("null seeds", 1, (2, [1], 4, sp(seeds=None))),
        ("negative first draw", 1, (2, [1], 4, sp(first_draw=-2))),
        ("history id past the vocabulary", 1, (2, [1], 4, sp(history=bad_hist.ctypes.data, history_counts=bad_counts.ctypes.data))),
        ("context overflow", 5, (1, [5, 6, 7, 8, 9], 11)),
    ]
    for what, code, args in cases:
        assert raw_add(*args) == code, (what, capi.lib().b200_last_error())
    # the handles belong to the stream: every other call fails at once with B200_EINVAL and changes nothing
    with pytest.raises(capi.B200Error) as ei:
        gpu[0].session_forward(2, np.zeros((1, sh.n_embd), np.float32))
    assert ei.value.code == 1 and "stream" in str(ei.value)
    for call in (lambda: extra.embed([1]), lambda: capi.generate_greedy(gpu, extra, [2], [[1]], 2),
                 lambda: capi.generate_greedy(twin, extra, [2], [[1]], 2), lambda: gpu[1].session_clear(-1),
                 lambda: gpu[0].n_past, lambda: capi.Stream(gpu, extra), lambda: capi.Stream(twin, extra)):
        with pytest.raises(capi.B200Error) as ei:
            call()
        assert ei.value.code == 1 and "stream" in str(ei.value), str(ei.value)
    assert gpu[0].session_n_past(0) == -1
    assert extra.token_text(5) and gpu[0].launch_count() > 0
    # the largest add that fits: session 1 ends exactly at n_ctx
    assert raw_add(1, [5, 6, 7, 8, 9], 10) == 0
    got = _by_session(list(st))
    st.close()
    assert positions(gpu)[1] == 64 and positions(gpu)[0] == 5 and positions(gpu)[2] == before[2]
    assert got[0] == capi.generate_greedy(twin, extra, [0], [[1, 2]], 4)[:, 0].tolist()
    assert got[1] == capi.generate_greedy(twin, extra, [1], [[5, 6, 7, 8, 9]], 10)[:, 0].tolist()
    assert positions(gpu) == positions(twin)
    # after close the handles work again
    gpu[0].session_forward(2, np.zeros((1, sh.n_embd), np.float32))
    for s in gpu:
        s.session_clear(-1)
    # logits with no distribution end that session with -1; a greedy neighbour completes as it would alone
    nan_extra = capi.Extra(_nan_extra(tmp_path, sh), 0)
    for s in twin:
        s.session_clear(-1)
    with capi.Stream(gpu, nan_extra) as st:
        st.add(2, [1, 2], 5, temperature=0.7, seed=1)
        st.add(0, [3], 5)
        got = _by_session(list(st))
    assert got[2] == [-1] and got[0] == capi.generate_greedy(twin, nan_extra, [0], [[3]], 5)[:, 0].tolist()
    assert gpu[0].session_n_past(2) == 2 and gpu[1].session_n_past(0) == 5
    nan_extra.close()
    extra.close()
    for s in gpu + twin:
        s.close()


def _local(tmp_path):
    from distributedllm_b200.client import LocalPipeline
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=0)
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    return LocalPipeline([sl], [0]), extra


def test_local_pipeline_generate_streams(tmp_path):
    from distributedllm_b200 import client
    lp, extra = _local(tmp_path)
    prompt, n = "the the a in", 64
    kw = dict(temperature=0.8, repeat_penalty=1.1, seed=9)
    c0 = lp.slices[0].launch_count()
    full = list(lp.generate(extra, prompt, n, **kw))
    per_run = lp.slices[0].launch_count() - c0
    n_prompt = lp.slices[0].n_past - n + 1
    assert len(full) == n
    # the first string arrives long before the run is done, and breaking off cancels the rest
    g = lp.generate(extra, prompt, n, **kw)
    c0 = lp.slices[0].launch_count()
    assert next(g) == full[0]
    assert lp.slices[0].launch_count() - c0 < per_run / 4, (lp.slices[0].launch_count() - c0, per_run)
    got = [full[0]] + [next(g) for _ in range(6)]
    g.close()
    assert got == full[:7] and lp.slices[0].n_past == n_prompt + 7 - 1
    # stop_at_eos: a key whose run draws the end-of-sequence id
    ex = lp._device_extra(extra, "sampled generation")
    tokens = ex.tokenize(prompt)
    for seed in range(200):
        lp.clear_context()
        ids = lp.capi.generate_sample(lp.slices, ex, [0], [tokens], 100, 5.0, 1.1, [seed])[:, 0].tolist()
        if client.EOS_ID in ids:
            break
    else:
        pytest.fail("no key in 200 drew the end-of-sequence id")
    at = ids.index(client.EOS_ID)
    plain = list(lp.generate(extra, prompt, 100, temperature=5.0, seed=seed))
    assert lp.slices[0].n_past == len(tokens) + 99
    stopped = list(lp.generate(extra, prompt, 100, temperature=5.0, seed=seed, stop_at_eos=True))
    assert stopped == plain[:at + 1] and stopped[-1] == ex.token_text(client.EOS_ID)
    assert lp.slices[0].n_past == len(tokens) + at
    lp.close()


def test_local_pipeline_generate_equals_the_node_path_with_stops_off(tmp_path):
    """The streaming LocalPipeline.generate yields the node path's strings (DistributedLLM.generate, which never stops
    at EOS) for a key whose run passes the end-of-sequence id."""
    from distributedllm_b200.client import DistributedLLM, EOS_ID
    from distributedllm_b200.compute_node.slices import import_llm
    from distributedllm_b200.control_center import Connection
    llm = import_llm()
    lp, extra = _local(tmp_path)
    sl = lp.slices
    ex = lp._device_extra(extra, "sampled generation")
    tokens = ex.tokenize("the the a in")
    for seed in range(200):
        lp.clear_context()
        ids = lp.capi.generate_sample(sl, ex, [0], [tokens], 40, 5.0, 1.1, [seed])[:, 0].tolist()
        if EOS_ID in ids[:-1]:
            break
    else:
        pytest.fail("no key in 200 drew the end-of-sequence id")
    lp.close()
    sh = ggjt.SHAPES["tiny128"]
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(str(tmp_path / "slice.bin"), "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        want = list(DistributedLLM([addr], extra).generate("the the a in", 40, temperature=5.0, repeat_penalty=1.1,
                                                           rng=np.random.Generator(np.random.Philox(key=seed))))
    finally:
        srv.shutdown()
        srv.server_close()
        llm.unload_slice()
    lp, _ = _local(tmp_path)
    assert list(lp.generate(extra, "the the a in", 40, temperature=5.0, seed=seed)) == want
    lp.close()
