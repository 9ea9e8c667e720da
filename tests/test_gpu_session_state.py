"""GPU: session state on the device and off it (b200_session_copy, b200_session_save / _restore, b200_stream_fork).  A
copied, restored or forked session holds its source's rows and position, so it must continue bit for bit as the source
would have: against the reference's own hidden states, against the source itself, and against one-shot generation."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from test_gpu_generate import _model
from test_gpu_stream import MODES, _add, _by_session, _one_shot, _prefill

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_SETS = ["slices", "slices_q4_1", "slices_q5_0", "slices_q5_1", "slices_kquant"]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _kv(sl):
    """Both caches as uint16 [2][n_sessions][n_layer][n_ctx][n_embd] (debug_read 7 and 8)."""
    i = sl.info
    shape = (sl.n_sessions, i.n_layer, i.n_ctx, i.n_embd)
    words = int(np.prod(shape)) // 2
    return np.stack([sl.debug_read(w, words, np.uint16).reshape(shape) for w in (7, 8)])


def _golden_cases():
    for stem in GOLDEN_SETS:
        for name, m in json.load(open(os.path.join(GOLD, stem + ".json"))).items():
            yield pytest.param(stem, name, m, id=name)


def _write_golden(path, m):
    sh = ggjt.SHAPES[m["shape"]]
    if "mix" in m:
        ggjt.write_kquant_slice(path, sh, m["layers"][0], m["layers"][1], m["mix"], seed=0)
    else:
        ggjt.write_synth_slice(path, sh, m["layers"][0], m["layers"][1], m["wtype"], seed=0)


@pytest.mark.parametrize("stem,name,m", list(_golden_cases()))
def test_copied_and_restored_sessions_continue_as_the_reference(tmp_path, stem, name, m):
    """Session 0 takes the golden schedule's first calls; sessions 1-3 hold longer garbage, then get session 0's rows by
    session_copy (and later by save + restore, also into a handle of another n_ctx and n_sessions); each continues with
    the remaining calls and must give the reference's hidden states."""
    from distributedllm_b200 import capi
    gold = np.load(os.path.join(GOLD, stem + ".npz"))
    path = str(tmp_path / (name + ".bin"))
    _write_golden(path, m)
    sched = m["schedule"]
    k = len(sched) // 2
    n_embd = ggjt.SHAPES[m["shape"]].n_embd
    x = [gold["%s/x%d" % (name, i)] for i in range(len(sched))]
    y = [gold["%s/y%d" % (name, i)] for i in range(len(sched))]
    sl = capi.Slice(path, 0, 512, n_sessions=4)
    for i in range(k):
        assert (_bits(sl.session_forward(0, x[i])) == _bits(y[i])).all(), (name, i)
    keep = sum(sched[:k])
    rng = np.random.default_rng(3)
    for d in (1, 2, 3):
        sl.session_forward(d, rng.standard_normal((keep + 17 * d, n_embd), dtype=np.float32))

    def rest(h, d, how):
        assert h.session_n_past(d) == keep, how
        for i in range(k, len(sched)):
            assert (_bits(h.session_forward(d, x[i])) == _bits(y[i])).all(), (name, how, d, i)

    sl.session_copy(0, [3, 1, 2], keep)
    for d in (1, 2, 3):
        rest(sl, d, "copy")
    blob = sl.session_save(0)
    assert len(blob) == 64 + keep * sl.info.kv_bytes_per_pos and blob[:4] == b"B2KV"
    sl.session_restore(2, blob)
    rest(sl, 2, "restore")
    other = capi.Slice(path, 0, sum(sched) + 3, n_sessions=2)
    other.session_forward(1, rng.standard_normal((5, n_embd), dtype=np.float32))
    other.session_restore(1, blob)
    rest(other, 1, "restore into another handle")
    assert other.session_n_past(0) == 0 and sl.session_n_past(0) == keep
    other.close()
    sl.close()


def test_copy_moves_exactly_the_kept_rows(tmp_models):
    """debug_read of both caches around a copy: each destination's rows [0, n_keep) equal the source's in every layer;
    every other byte (the source, the other sessions, the destinations' rows from n_keep on) is unchanged."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    sl = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 0, 2, seed=61), 0, 64, n_sessions=5)
    rng = np.random.default_rng(61)
    for d, n in enumerate((12, 50, 7, 61, 33)):
        sl.session_forward(d, rng.standard_normal((n, sh.n_embd), dtype=np.float32))
    for src, dsts, keep in ((3, [4], 61), (1, [3, 0], 29), (2, [1, 4, 0, 3], 7), (4, [2], 0)):
        before = [sl.session_n_past(d) for d in range(5)]
        a = _kv(sl)
        sl.session_copy(src, dsts, keep)
        b = _kv(sl)
        want = a.copy()
        for d in dsts:
            want[:, d, :, :keep] = a[:, src, :, :keep]
        assert (b == want).all(), (src, dsts, keep)
        assert [sl.session_n_past(d) for d in range(5)] == [keep if d in dsts else before[d] for d in range(5)]
    sl.close()


def test_partial_keep_equals_the_source_rewound(tmp_models):
    """Copy with n_keep < the source's position, then feed the destination a chunk and a single step: the outputs equal
    the source's after session_rewind(n_keep) fed the same rows."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny3b"]
    sl = capi.Slice(tmp_models("tiny3b", ggjt.T_Q4_0, 0, 1, seed=62), 0, 96, n_sessions=3)
    rng = np.random.default_rng(62)
    sl.session_forward(0, rng.standard_normal((41, sh.n_embd), dtype=np.float32))
    sl.session_forward(2, rng.standard_normal((70, sh.n_embd), dtype=np.float32))
    sl.session_copy(0, [2], 23)
    chunk, step = (rng.standard_normal((n, sh.n_embd), dtype=np.float32) for n in (9, 1))
    got = [sl.session_forward(2, chunk), sl.session_forward(2, step)]
    sl.session_rewind(0, 23)
    want = [sl.session_forward(0, chunk), sl.session_forward(0, step)]
    for g, w in zip(got, want):
        assert (_bits(g) == _bits(w)).all()
    assert sl.session_n_past(2) == sl.session_n_past(0) == 33
    sl.close()


def test_forked_sessions_in_one_batched_step_and_mixed_pass(tmp_models):
    """Fork a session into 7 others: one batch_forward of all 8 with the same token gives 8 identical rows, equal to a
    single step of a ninth fresh copy; then the same with one mixed pass of a 5-row chunk per session."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    sl = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=63), 0, 64, n_sessions=9)
    rng = np.random.default_rng(63)
    sl.session_forward(0, rng.standard_normal((26, sh.n_embd), dtype=np.float32))
    sl.session_forward(5, rng.standard_normal((40, sh.n_embd), dtype=np.float32))
    sl.session_copy(0, list(range(1, 9)), 26)
    x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
    got = sl.batch_forward(list(range(8)), np.repeat(x, 8, axis=0))
    want = sl.session_forward(8, x)
    assert (_bits(got) == _bits(np.repeat(want, 8, axis=0))).all()
    sl.session_copy(8, list(range(8)), 27)
    chunk = rng.standard_normal((5, sh.n_embd), dtype=np.float32)
    got = sl.mixed_forward(list(range(8)), [5] * 8, np.tile(chunk, (8, 1)))
    want = sl.session_forward(8, chunk)
    assert (_bits(got) == _bits(np.tile(want, (8, 1)))).all()
    assert [sl.session_n_past(d) for d in range(9)] == [32] * 9
    sl.close()


def test_fork_at_7b_layer_shape(tmp_path):
    """One LLaMA-7B-shape Q4_0 layer at n_ctx 2048: fork 2047 rows to 7 sessions, check every cache byte, then one
    batched continuation step of the 7 equals the source's own step."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "layer.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=64)
    sl = capi.Slice(path, 0, 2048, n_sessions=8)
    rng = np.random.default_rng(64)
    for lo in range(0, 2047, 512):
        sl.session_forward(0, rng.standard_normal((min(512, 2047 - lo), sh.n_embd), dtype=np.float32))
    sl.session_forward(3, rng.standard_normal((100, sh.n_embd), dtype=np.float32))
    a = _kv(sl)
    sl.session_copy(0, list(range(1, 8)), 2047)
    b = _kv(sl)
    want = a
    want[:, 1:, :, :2047] = a[:, :1, :, :2047]
    assert (b == want).all()
    del a, b, want
    x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
    got = sl.batch_forward(list(range(1, 8)), np.repeat(x, 7, axis=0))
    assert (_bits(got) == _bits(np.repeat(sl.session_forward(0, x), 7, axis=0))).all()
    sl.close()


def _code(fn):
    from distributedllm_b200 import capi
    with pytest.raises(capi.B200Error) as ei:
        fn()
    return ei.value.code, str(ei.value)


def test_refusals_change_nothing(tmp_models, tmp_path):
    """Every refusal of session_copy, save and restore is B200_EINVAL and leaves every position and cache byte as it
    was; so are all four calls on handles an open stream owns."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    sl = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=65), 0, 64, n_sessions=4)
    rng = np.random.default_rng(65)
    for d, n in enumerate((30, 64, 5, 0)):
        if n:
            sl.session_forward(d, rng.standard_normal((n, sh.n_embd), dtype=np.float32))
    lib, h = capi.lib(), sl.handle
    kv0, pos0 = _kv(sl), [sl.session_n_past(d) for d in range(4)]
    blob = sl.session_save(0)
    small = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=65), 0, 32, n_sessions=1)
    tiny = capi.Slice(tmp_models("tiny", ggjt.T_Q4_0, 0, 1, seed=65), 0, 64, n_sessions=1)

    def raw_copy(src, dsts, n_dst, keep, handle=h):
        d = None if dsts is None else (C.c_int * max(len(dsts), 1))(*dsts)
        return lib.b200_session_copy(handle, src, d, n_dst, keep)

    def header(**kw):
        b = bytearray(blob)
        for off, v in kw.items():
            b[int(off[1:]):int(off[1:]) + 4] = int(v).to_bytes(4, "little")
        return bytes(b)

    copies = [(None, [1], 1, 0), (0, None, 1, 0), (0, [1], 0, 0), (0, [1], -1, 0), (-1, [1], 1, 0), (4, [1], 1, 0),
              (0, [4], 1, 0), (0, [-1], 1, 0), (0, [0], 1, 0), (0, [1, 2, 1], 3, 0), (0, [1], 1, 31), (0, [1], 1, -1),
              (3, [1], 1, 1)]
    for src, dsts, n_dst, keep in copies:
        handle = None if src is None else h
        assert raw_copy(src or 0, dsts, n_dst, keep, handle) == 1, (src, dsts, n_dst, keep)
    n = C.c_size_t(0)
    assert lib.b200_session_state_size(h, 4, C.byref(n)) == 1 and lib.b200_session_state_size(h, 0, None) == 1
    buf = np.full(len(blob), 0xAB, np.uint8)
    assert lib.b200_session_save(h, 0, capi._ptr(buf), len(blob) - 1, None) == 1 and (buf == 0xAB).all()
    assert lib.b200_session_save(h, -1, capi._ptr(buf), len(blob), None) == 1 and (buf == 0xAB).all()
    bad = [b"B2KW" + blob[4:], header(o4=2), header(o8=256), header(o12=8), header(o16=3), header(o20=1),
           header(o24=31), header(o24=0xFFFFFFFF), blob[:-1], blob + b"\0", blob[:63], b""]
    for i, b in enumerate(bad):
        assert _code(lambda: sl.session_restore(1, b))[0] == 1, i
    big = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=65), 0, 64, n_sessions=2)
    big.session_forward(0, rng.standard_normal((40, sh.n_embd), dtype=np.float32))
    for target in (small, tiny):                          # n_past 40 > n_ctx 32; n_embd 256 != 512
        assert _code(lambda: target.session_restore(0, big.session_save(0)))[0] == 1
        assert target.session_n_past(0) == 0
    assert _code(lambda: tiny.session_restore(0, blob))[0] == 1
    assert (_kv(sl) == kv0).all() and [sl.session_n_past(d) for d in range(4)] == pos0
    # an open stream owns the handles
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=65)
    extra = capi.Extra(extra_path, 0)
    with capi.Stream([sl], extra):
        for fn in (lambda: sl.session_copy(0, [1], 1), lambda: sl.session_save(0), lambda: sl.session_restore(1, blob)):
            code, msg = _code(fn)
            assert code == 1 and "stream" in msg, msg
        assert lib.b200_session_state_size(h, 0, C.byref(n)) == 1
    assert (_kv(sl) == kv0).all() and [sl.session_n_past(d) for d in range(4)] == pos0
    sl.session_restore(3, blob)                            # after close the handle works again
    assert sl.session_n_past(3) == 30
    for s in (sl, small, tiny, big):
        s.close()
    extra.close()


@pytest.mark.parametrize("fill", ["forward", "stream"])
def test_stream_fork_equals_one_shot_generation(tmp_path, fill):
    """A prefix session holds P (by session_forward, or by a stream add(P, max_tokens=1)); it is forked to four sessions
    while another session decodes, and each gets a suffix with greedy or sampled settings.  A fifth fork lands on a
    session cancelled with steps still in flight.  Each session's ids equal a one-shot run on a session fed P as one
    segment, then given its suffix."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 128, n_sessions=8) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=8) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(66)
    P = rng.integers(0, sh.n_vocab, 37).tolist()
    suffix = {k: rng.integers(0, sh.n_vocab, n).tolist() for k, n in ((1, 4), (2, 1), (3, 9), (4, 6), (5, 3))}
    budget = {1: 20, 2: 31, 3: 12, 4: 25, 5: 18}
    modes = {1: MODES[0], 2: MODES[1], 3: MODES[4], 4: MODES[7], 5: MODES[5]}
    other = rng.integers(0, sh.n_vocab, 11).tolist()
    if fill == "forward":
        _prefill(extra, (gpu,), 0, P)
    pairs = []
    with capi.Stream(gpu, extra, lookahead=4) as st:
        if fill == "stream":
            st.add(0, P, 1)
            pairs += list(st)
        _add(st, 7, other, 60, MODES[1])
        _add(st, 5, other[:5], 40, MODES[0])
        pairs += st.read(3)
        for k in (1, 2, 3, 4):
            st.fork(0, k, len(P))
            _add(st, k, suffix[k], budget[k], modes[k])
        while len(_by_session(pairs).get(5, [])) < 2:
            pairs += st.read(1)
        st.cancel(5)                                       # steps of session 5 may still be in flight
        st.fork(0, 5, len(P))
        _add(st, 5, suffix[5], budget[5], modes[5])
        pairs += list(st)
    got = _by_session(pairs)
    for k in suffix:
        _prefill(extra, (twin,), k, P)
        assert _one_shot(capi, twin, extra, k, suffix[k], budget[k], modes[k]) == got[k][-budget[k]:], k
        assert [s.session_n_past(k) for s in gpu] == [s.session_n_past(k) for s in twin], k
    assert len(got[7]) == 60 and [s.session_n_past(0) for s in gpu] == [len(P)] * 2
    extra.close()
    for s in gpu + twin:
        s.close()


def test_stream_fork_refusals(tmp_path):
    """Every b200_stream_fork refusal is B200_EINVAL and moves no position; a valid fork after them still works."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 64, n_sessions=6) for p in paths]
    extra = capi.Extra(extra_path, 0)
    _prefill(extra, (gpu,), 0, list(range(1, 21)))
    x = extra.embed([3, 4, 5])
    gpu[0].session_forward(4, x)                          # session 4 is at 3 on slice 0 and 0 on slice 1
    before = [s.session_n_past(k) for s in gpu for k in range(6)]
    with capi.Stream(gpu, extra) as st:
        st.add(1, [1, 2], 30)                              # queued
        st.add(2, [3], 30)
        st.read(1)                                         # 1 and 2 active
        st.add(3, [4], 30)                                 # queued behind nothing: becomes active at the next step
        lib = capi.lib()
        for src, dst, keep in ((6, 5, 0), (-1, 5, 0), (0, 6, 0), (0, -1, 0), (1, 5, 0), (0, 2, 5), (0, 3, 5),
                               (5, 5, 0), (0, 0, 3), (0, 5, 21), (0, 5, -1), (4, 5, 0)):
            assert lib.b200_stream_fork(st._h, src, dst, keep) == 1, (src, dst, keep, lib.b200_last_error())
        st.fork(0, 5, 20)
        st.add(5, [7], 2)
        list(st)
    after = [s.session_n_past(k) for s in gpu for k in range(6)]
    for i, (b, a) in enumerate(zip(before, after)):
        if i % 6 in (0, 4):
            assert a == b, i
    assert [s.session_n_past(5) for s in gpu] == [22, 22]     # 20 kept + 1 prompt id + 2 ids - 1
    extra.close()
    for s in gpu:
        s.close()
