"""GPU: decode rows (b200_session_forward_steps) against single-token steps, and speculative decoding
(b200_generate_speculative) against the plain device loops, bit for bit."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
REF = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_digests.json")))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _rows(n, E, seed):
    return np.random.default_rng(seed).standard_normal((n, E), dtype=np.float32)


# ---------------------------------------------------------------- decode rows

BLOCK = {"q4_0": ggjt.T_Q4_0, "q4_1": ggjt.T_Q4_1, "q5_0": ggjt.T_Q5_0, "q5_1": ggjt.T_Q5_1, "q8_0": ggjt.T_Q8_0,
         "f16": ggjt.T_F16}


def _slice_file(tmp_path, kind, shape):
    sh = ggjt.SHAPES[shape]
    path = str(tmp_path / ("%s_%s.bin" % (kind, shape)))
    if kind == "q4_K_M":
        ggjt.write_kquant_slice(path, sh, 0, sh.n_layer - 1, "q4_K_M", seed=5)
    else:
        ggjt.write_synth_slice(path, sh, 0, sh.n_layer - 1, BLOCK[kind], seed=5)
    return path, sh


def _check_steps(path, sh, n_ctx, session, pre, n_rows, n_sessions=3):
    """session holds `pre` rows on both handles (other sessions hold other contexts on the decode-rows handle); then n_rows
    rows as one forward_steps call on one handle and as single session_forward calls on the other."""
    from distributedllm_b200 import capi
    a = capi.Slice(path, 0, n_ctx, n_sessions=n_sessions)
    b = capi.Slice(path, 0, n_ctx, n_sessions=n_sessions)
    try:
        for k in range(n_sessions):
            if k != session:
                a.session_forward(k, _rows(3 + k, sh.n_embd, 100 + k))
        if pre:
            x = _rows(pre, sh.n_embd, 1)
            a.session_forward(session, x)
            b.session_forward(session, x)
        x = _rows(n_rows, sh.n_embd, 2)
        got = a.forward_steps(session, x)
        want = np.concatenate([b.session_forward(session, x[j:j + 1]) for j in range(n_rows)])
        assert (_bits(got) == _bits(want)).all()
        assert a.session_n_past(session) == b.session_n_past(session) == pre + n_rows
        # the caches agree too: the next single step is the same on both handles
        y = _rows(1, sh.n_embd, 3)
        assert (_bits(a.session_forward(session, y)) == _bits(b.session_forward(session, y))).all()
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("kind", ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "f16", "q4_K_M"])
def test_forward_steps_equal_single_steps_head_128(tmp_path, kind):
    path, sh = _slice_file(tmp_path, kind, "tinyk128" if kind == "q4_K_M" else "tiny128")
    for pre, n_rows in ((0, 1), (5, 2), (7, 9), (30, 16)):
        _check_steps(path, sh, 128, 1, pre, n_rows)


@pytest.mark.parametrize("kind", ["q4_0", "q5_1", "q8_0", "f16", "q4_K_M"])
def test_forward_steps_equal_single_steps_generic_head(tmp_path, kind):
    path, sh = _slice_file(tmp_path, kind, "tinyk" if kind == "q4_K_M" else "tiny")
    for pre, n_rows in ((0, 3), (11, 5), (40, 16)):
        _check_steps(path, sh, 128, 2, pre, n_rows)


@pytest.mark.parametrize("shape", ["tiny128", "tiny"])
def test_forward_steps_straddle_position_512(tmp_path, shape):
    path, sh = _slice_file(tmp_path, "q4_0", shape)
    _check_steps(path, sh, 1024, 0, 505, 12, n_sessions=2)


@pytest.mark.parametrize("env", ["B200_FAST_PREFILL", "B200_GRAPH", "B200_PDL", "B200_TILED_ATTN"])
def test_forward_steps_under_switches(tmp_path, monkeypatch, env):
    monkeypatch.setenv(env, "1" if env == "B200_FAST_PREFILL" else "0")
    path, sh = _slice_file(tmp_path, "q4_0", "tiny128")
    _check_steps(path, sh, 128, 1, 6, 16)          # fast prefill would apply to 16 rows of a prompt call (min_tokens 0 below)
    from distributedllm_b200 import capi
    a = capi.Slice(path, 0, 128)
    b = capi.Slice(path, 0, 128)
    a.set_fast_prefill(True, 1)
    x = _rows(8, sh.n_embd, 4)
    got = a.forward_steps(0, x)
    want = np.concatenate([b.session_forward(0, x[j:j + 1]) for j in range(8)])
    assert (_bits(got) == _bits(want)).all()
    a.close()
    b.close()


@pytest.mark.parametrize("kind", ["q4_0", "q4_K_M"])
def test_forward_steps_7b_layer(tmp_path, kind):
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "l7b.bin")
    if kind == "q4_0":
        ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=1)
    else:
        ggjt.write_kquant_slice(path, sh, 0, 0, "q4_K_M", seed=1)
    _check_steps(path, sh, 512, 1, 20, 9, n_sessions=2)


# ---------------------------------------------------------------- speculative decoding

def _model(tmp_path, kind, tag="t", seed=41):
    """Two target slices and an extra-layers file: (slice paths, extra path, shape)."""
    if kind == "q4_0":
        sh = ggjt.SHAPES["tiny128"]
        paths = [str(tmp_path / ("%s_a.bin" % tag)), str(tmp_path / ("%s_b.bin" % tag))]
        ggjt.write_synth_slice(paths[0], sh, 0, 0, ggjt.T_Q4_0, seed=seed)
        ggjt.write_synth_slice(paths[1], sh, 1, sh.n_layer - 1, ggjt.T_Q4_0, seed=seed)
        extra = str(tmp_path / ("%s_extra.bin" % tag))
        ggjt.write_synth_extra(extra, sh, ggjt.T_Q4_0, seed=seed)
    elif kind == "f16":
        sh = ggjt.SHAPES["tiny"]
        paths = [str(tmp_path / ("%s_a.bin" % tag)), str(tmp_path / ("%s_b.bin" % tag))]
        ggjt.write_synth_slice(paths[0], sh, 0, 1, ggjt.T_F16, seed=seed)
        ggjt.write_synth_slice(paths[1], sh, 2, sh.n_layer - 1, ggjt.T_F16, seed=seed)
        extra = str(tmp_path / ("%s_extra.bin" % tag))
        ggjt.write_synth_extra(extra, sh, ggjt.T_F16, seed=seed)
    else:
        sh = ggjt.SHAPES["tinyk128"]
        paths = [str(tmp_path / ("%s_a.bin" % tag)), str(tmp_path / ("%s_b.bin" % tag))]
        ggjt.write_kquant_slice(paths[0], sh, 0, 3, "q4_K_M", seed=seed)
        ggjt.write_kquant_slice(paths[1], sh, 4, sh.n_layer - 1, "q4_K_M", seed=seed)
        extra = str(tmp_path / ("%s_extra.bin" % tag))
        ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=seed)
    return paths, extra, sh


class Chain:
    def __init__(self, paths, extra_path, n_ctx, n_sessions=1):
        from distributedllm_b200 import capi
        self.slices = [capi.Slice(p, 0, n_ctx, n_sessions=n_sessions) for p in paths]
        self.extra = capi.Extra(extra_path, 0)

    def clear(self):
        for s in self.slices:
            s.session_clear(-1)

    def n_past(self, session=0):
        return [s.session_n_past(session) for s in self.slices]

    def close(self):
        self.extra.close()
        for s in self.slices:
            s.close()


def _drafts(tmp_path, kind, paths, extra_path, n_ctx):
    """The three drafts: the target itself (second handles), its first slice only (a layer-skip draft) and an unrelated
    model of another n_embd and head size with the same vocabulary size (F16 'tiny', d_head 64, for the head-size-128
    targets; Q4_0 'tiny128' for the F16 'tiny' target)."""
    upaths, uextra, _ = _model(tmp_path, "q4_0" if kind == "f16" else "f16", tag="u", seed=77)
    return {"same": Chain(paths, extra_path, n_ctx), "skip": Chain(paths[:1], extra_path, n_ctx),
            "unrelated": Chain(upaths, uextra, n_ctx)}


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
def test_greedy_ids_equal_generate_greedy(tmp_path, kind):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_ctx = 160
    tgt = Chain(paths, extra_path, n_ctx)
    prompt = np.random.default_rng(3).integers(0, sh.n_vocab, 5).tolist()
    want = capi.generate_greedy(tgt.slices, tgt.extra, [0], [prompt], 100)[:, 0]
    drafts = _drafts(tmp_path, kind, paths, extra_path, n_ctx)
    try:
        for name, dr in drafts.items():
            for k in (1, 2, 4, 7, 15):
                for n_steps in (1, 33, 100):
                    tgt.clear()
                    dr.clear()
                    ids, st = capi.generate_speculative(tgt.slices, tgt.extra, 0, dr.slices, dr.extra, 0, prompt, n_steps, k)
                    assert ids.tolist() == want[:n_steps].tolist(), (name, k, n_steps)
                    assert tgt.n_past() == [5 + n_steps - 1] * 2 and dr.n_past() == [5 + n_steps - 1] * len(dr.slices)
                    assert st["drafted"] == st["passes"] * k
                    if name == "same":
                        assert st["accepted"] == st["drafted"]
                        assert st["passes"] == math.ceil((n_steps - 1) / (k + 1))
    finally:
        tgt.close()
        for dr in drafts.values():
            dr.close()


def test_config1_3b_gives_the_reference_ids(tmp_path):
    """BASELINE config 1 (OpenLLaMA-3B shapes, two slices, 16-token prompt, 33 steps) with a two-layer draft of the same
    model: the reference's own greedy ids."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["3b"]
    pa, pb, pd, extra_path = (str(tmp_path / n) for n in ("a.bin", "b.bin", "d.bin", "extra.bin"))
    ggjt.write_fast_q4_slice(pa, sh, 0, 16, seed=3)
    ggjt.write_fast_q4_slice(pb, sh, 17, 25, seed=3)
    ggjt.write_fast_q4_slice(pd, sh, 0, 1, seed=3)
    ggjt.write_fast_q4_extra(extra_path, sh, seed=3)
    tgt = Chain([pa, pb], extra_path, 512)
    dr = Chain([pd], extra_path, 512)
    tokens = [1 + (i * 7919) % 31999 for i in range(16)]
    for k in (1, 4):
        tgt.clear()
        dr.clear()
        ids, st = capi.generate_speculative(tgt.slices, tgt.extra, 0, dr.slices, dr.extra, 0, tokens, 33, k)
        assert ids.tolist() == REF["config1"]["ids"]
        assert tgt.n_past() == [48, 48] and dr.n_past() == [48]
        assert st["drafted"] == st["passes"] * k
    tgt.close()
    dr.close()


@pytest.mark.parametrize("trunc", [(0, 0.0), (40, 0.95)])
def test_sampled_ids_equal_generate_sample_and_continue(tmp_path, trunc):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    n_ctx = 160
    tgt = Chain(paths, extra_path, n_ctx)
    drafts = _drafts(tmp_path, "q4_0", paths, extra_path, n_ctx)
    top_k, top_p = trunc
    prompt = [7, 100, 3, 250]
    seed = 2 ** 63 + 12345
    want = capi.generate_sample(tgt.slices, tgt.extra, [0], [prompt], 60, 0.7, 1.1, [seed], top_k=top_k, top_p=top_p)[:, 0]
    try:
        for name, dr in drafts.items():
            for k in (1, 4, 15):
                tgt.clear()
                dr.clear()
                ids, st = capi.generate_speculative(tgt.slices, tgt.extra, 0, dr.slices, dr.extra, 0, prompt, 60, k,
                                                    temperature=0.7, repeat_penalty=1.1, seed=seed, top_k=top_k, top_p=top_p)
                assert ids.tolist() == want.tolist(), (name, k)
                assert st["drafted"] == st["passes"] * k
                if name == "same":
                    assert st["accepted"] == st["drafted"]
            # two calls: 25 ids, then 35 more with the first 25 as history
            tgt.clear()
            dr.clear()
            a, _ = capi.generate_speculative(tgt.slices, tgt.extra, 0, dr.slices, dr.extra, 0, prompt, 25, 3,
                                             temperature=0.7, seed=seed, top_k=top_k, top_p=top_p)
            b, _ = capi.generate_speculative(tgt.slices, tgt.extra, 0, dr.slices, dr.extra, 0, [int(a[-1])], 35, 3,
                                             temperature=0.7, seed=seed, first_draw=25, history=a.tolist(),
                                             top_k=top_k, top_p=top_p)
            assert a.tolist() + b.tolist() == want.tolist(), name
            assert tgt.n_past() == [4 + 60 - 1] * 2
    finally:
        tgt.close()
        for dr in drafts.values():
            dr.close()


def test_greedy_continuation_and_the_next_plain_step(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    tgt = Chain(paths, extra_path, 160, n_sessions=3)
    dr = Chain(paths[:1], extra_path, 160, n_sessions=2)
    prompt = [5, 9, 11]
    # target session 2 and draft session 1, both mid-context at 4 positions; target session 0 holds something else
    pre = [1, 2, 3, 4]
    for ch, sess in ((tgt, 2), (dr, 1)):
        x = ch.extra.embed(pre)
        for s in ch.slices:
            x = s.session_forward(sess, x)
    x = tgt.extra.embed([8, 8])
    for s in tgt.slices:
        x = s.session_forward(0, x)
    a, _ = capi.generate_speculative(tgt.slices, tgt.extra, 2, dr.slices, dr.extra, 1, prompt, 20, 4)
    b, _ = capi.generate_speculative(tgt.slices, tgt.extra, 2, dr.slices, dr.extra, 1, [int(a[-1])], 30, 4)
    assert tgt.n_past(2) == [4 + 3 + 50 - 1] * 2 and dr.n_past(1) == [4 + 3 + 50 - 1]
    assert tgt.n_past(0) == [2, 2]
    x = tgt.extra.embed([int(b[-1])])
    for s in tgt.slices:
        x = s.session_forward(2, x)
    # the plain loop over the sum, on fresh handles with the same history
    twin = Chain(paths, extra_path, 160)
    y = twin.extra.embed(pre)
    for s in twin.slices:
        y = s.session_forward(0, y)
    want = capi.generate_greedy(twin.slices, twin.extra, [0], [prompt], 50)[:, 0]
    assert a.tolist() + b.tolist() == want.tolist()
    y = twin.extra.embed([int(want[-1])])
    for s in twin.slices:
        y = s.session_forward(0, y)
    assert (_bits(x) == _bits(y)).all()
    for ch in (tgt, dr, twin):
        ch.close()


def test_refusals_change_nothing(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    tgt = Chain(paths, extra_path, 64)
    dr = Chain(paths[:1], extra_path, 64)
    # a draft of another vocabulary size
    vsh = ggjt.ModelShape(256, 256, 32, 4, 1)
    vp, ve = str(tmp_path / "v.bin"), str(tmp_path / "v_extra.bin")
    ggjt.write_synth_slice(vp, vsh, 0, 0, ggjt.T_Q4_0, seed=9)
    ggjt.write_synth_extra(ve, vsh, ggjt.T_Q4_0, seed=9)
    vd = Chain([vp], ve, 64)
    prompt = [3, 4, 5]
    x = tgt.extra.embed([1, 2])
    for s in tgt.slices:
        x = s.session_forward(0, x)
    y = dr.extra.embed([1, 2])
    dr.slices[0].session_forward(0, y)
    before = (tgt.n_past(), dr.n_past())

    def refused(code, *args, **kw):
        with pytest.raises(capi.B200Error) as ei:
            capi.generate_speculative(*args, **kw)
        assert ei.value.code == code, ei.value
        assert (tgt.n_past(), dr.n_past()) == before

    T = (tgt.slices, tgt.extra, 0)
    D = (dr.slices, dr.extra, 0)
    refused(1, *T, *D, prompt, 10, 0)                                       # n_draft outside [1, 15]
    refused(1, *T, *D, prompt, 10, 16)
    refused(1, *T, vd.slices, vd.extra, 0, prompt, 10, 4)                   # vocabulary mismatch
    refused(1, *T, tgt.slices[:1], dr.extra, 0, prompt, 10, 4)              # a handle in both chains
    refused(5, *T, *D, prompt, 64 - 2 - 3 + 1 - 4 + 1, 4)                  # n_past + n_prompt + n_steps - 1 + n_draft > n_ctx
    refused(1, *T, *D, prompt, 10, 4, temperature=0.7, seed=1, repeat_penalty=0.0)
    dr.slices[0].session_forward(0, dr.extra.embed([6]))                    # unequal starting positions
    before = (tgt.n_past(), dr.n_past())
    refused(1, *T, *D, prompt, 10, 4)
    dr.slices[0].session_rewind(0, 2)
    before = (tgt.n_past(), dr.n_past())
    # the longest budget that fits, and a null draft through the C ABI
    ids, _ = capi.generate_speculative(*T, *D, prompt, 64 - 2 - 3 + 1 - 4, 4)
    out = np.zeros(4, np.int32)
    toks = np.array(prompt, np.int32)
    h = (C.c_void_p * 2)(*[s.handle for s in tgt.slices])
    dh = (C.c_void_p * 1)(dr.slices[0].handle)
    assert capi.lib().b200_generate_speculative(h, 2, tgt.extra.handle, 0, None, 1, dr.extra.handle, 0, toks.ctypes.data, 3,
                                                4, 2, None, out.ctypes.data, None) == 1
    assert capi.lib().b200_generate_speculative(h, 2, tgt.extra.handle, 0, dh, 1, None, 0, toks.ctypes.data, 3,
                                                4, 2, None, out.ctypes.data, None) == 1
    assert (tgt.n_past(), dr.n_past()) == ([2 + 3 + 56 - 1] * 2, [2 + 3 + 56 - 1])
    for ch in (tgt, dr, vd):
        ch.close()
    # the refusals left the caches alone: the full-length call above gave the plain loop's ids
    twin = Chain(paths, extra_path, 64)
    x = twin.extra.embed([1, 2])
    for s in twin.slices:
        x = s.session_forward(0, x)
    assert ids.tolist() == capi.generate_greedy(twin.slices, twin.extra, [0], [prompt], len(ids))[:, 0].tolist()
    twin.close()


def _nan_extra(tmp_path, sh):
    """An extra-layers file whose norm.weight holds a NaN: every logit is NaN (as tests/test_gpu_stream.py builds it)."""
    path = str(tmp_path / "extra_nan.bin")
    ggjt.write_synth_extra(path, sh, ggjt.T_F16, seed=45)
    norm = next(raw for name, _, _, raw in ggjt.synth_extra_tensors(sh, ggjt.T_F16, 45) if name == "norm.weight")
    data = bytearray(open(path, "rb").read())
    at = bytes(data).index(norm) + 4 * 3
    data[at:at + 4] = np.array([np.nan], np.float32).tobytes()
    open(path, "wb").write(bytes(data))
    return path


def test_a_row_without_distribution_matches_generate_sample(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    nan_extra = capi.Extra(_nan_extra(tmp_path, sh), 0)
    tgt = [capi.Slice(p, 0, 64) for p in paths]
    dr = Chain(paths[:1], extra_path, 64)
    sp, keep = capi._sampling(1, 0.7, 1.1, [11], 0, None)
    toks = np.array([3, 4], np.int32)
    h = (C.c_void_p * 2)(*[s.handle for s in tgt])
    want = np.zeros(6, np.int32)
    sessions, counts = np.array([0], np.int32), np.array([2], np.int32)
    rc_plain = capi.lib().b200_generate_sample(h, 2, nan_extra.handle, sessions.ctypes.data, counts.ctypes.data, 1,
                                               toks.ctypes.data, 6, C.byref(sp), want.ctypes.data)
    msg_plain = capi.lib().b200_last_error()
    for s in tgt:
        s.clear_context()
    got = np.zeros(6, np.int32)
    dh = (C.c_void_p * 1)(dr.slices[0].handle)
    stats = capi.SpecStats()
    rc = capi.lib().b200_generate_speculative(h, 2, nan_extra.handle, 0, dh, 1, dr.extra.handle, 0, toks.ctypes.data, 2, 6, 3,
                                              C.byref(sp), got.ctypes.data, C.byref(stats))
    msg = capi.lib().b200_last_error()
    assert rc == rc_plain == 1 and msg == msg_plain and b"step 0" in msg
    assert got.tolist() == want.tolist() == [-1] * 6
    assert [s.n_past for s in tgt] == [2 + 6 - 1] * 2
    nan_extra.close()
    dr.close()
    for s in tgt:
        s.close()
    del keep


def test_local_pipeline_generate_speculative(tmp_path):
    from distributedllm_b200.client import LocalPipeline
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=0)
    sl, dsl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "draft.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.slice_model(full, dsl, 0, 0)
    ggjt.extract_extra_layers(full, extra)
    lp, dp = LocalPipeline([sl], [0]), LocalPipeline([dsl], [0])
    text = "the the a in"
    greedy = lp.generate_greedy(extra, text, 30)
    assert lp.generate_speculative(extra, text, dp, extra, 30, n_draft=3) == greedy
    for seed, tk, tp in ((4, None, None), (2 ** 63 + 1, 40, 0.95)):
        strings = list(lp.generate(extra, text, 25, temperature=0.8, repeat_penalty=1.1, seed=seed, top_k=tk, top_p=tp))
        ids = lp.generate_speculative(extra, text, dp, extra, 25, n_draft=4, temperature=0.8, repeat_penalty=1.1, seed=seed,
                                      top_k=tk, top_p=tp)
        assert [lp._extra[1].token_text(i) for i in ids] == strings
    n_prompt = len(lp._extra[1].tokenize(text))
    assert lp.slices[0].n_past == dp.slices[0].n_past == n_prompt + 25 - 1
    lp.close()
    dp.close()


def test_draft_context_limit_and_no_graph(tmp_path, monkeypatch):
    """B200_ECONTEXT raised by the draft chain alone (its n_ctx is smaller than the target's), and the loop with the
    decode graph off (B200_GRAPH=0: the draft's single steps are enqueued kernel by kernel)."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    tgt = Chain(paths, extra_path, 160)
    small = Chain(paths[:1], extra_path, 40)
    prompt = [9, 8, 7]
    with pytest.raises(capi.B200Error) as ei:
        capi.generate_speculative(tgt.slices, tgt.extra, 0, small.slices, small.extra, 0, prompt, 40 - 3 - 4 + 2, 4)
    assert ei.value.code == 5
    assert tgt.n_past() == [0, 0] and small.n_past() == [0]
    ids, _ = capi.generate_speculative(tgt.slices, tgt.extra, 0, small.slices, small.extra, 0, prompt, 40 - 3 - 4 + 1, 4)
    tgt.clear()
    want = capi.generate_greedy(tgt.slices, tgt.extra, [0], [prompt], len(ids))[:, 0]
    assert ids.tolist() == want.tolist()
    small.close()
    monkeypatch.setenv("B200_GRAPH", "0")
    nog_t = Chain(paths, extra_path, 160)
    nog_d = Chain(paths[:1], extra_path, 160)
    seed = 99
    tgt.clear()
    want_g = capi.generate_greedy(tgt.slices, tgt.extra, [0], [prompt], 40)[:, 0]
    tgt.clear()
    want_s = capi.generate_sample(tgt.slices, tgt.extra, [0], [prompt], 40, 0.7, 1.1, [seed])[:, 0]
    for k in (1, 3, 8):
        for temp in (None, 0.7):
            nog_t.clear()
            nog_d.clear()
            got, st = capi.generate_speculative(nog_t.slices, nog_t.extra, 0, nog_d.slices, nog_d.extra, 0, prompt, 40, k,
                                                temperature=temp, seed=seed)
            assert got.tolist() == (want_s if temp else want_g).tolist(), (k, temp)
            assert st["drafted"] == st["passes"] * k
    for ch in (tgt, nog_t, nog_d):
        ch.close()
