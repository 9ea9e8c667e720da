"""GPU: the client's perplexity on the device.  k_nll_rows (b200_extra_nll) against the host twin (tests/score_ref.py),
and b200_score against scoring each session alone, other pass packings, the host path (b200_extra_embed ->
session_forward on each slice -> b200_extra_logits -> twin), the compiled reference, and DistributedLLM.perplexity
through a node.

Between the device and the host twin the tolerance is score_ref.TOL (the last ulps of float64 exp and the summation
order); on the device itself there is none: a session's NLLs are the same bits however the call packs it."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import score_ref
from distributedllm_b200 import ggjt
from test_gpu_generate import REF, _model, _serve
from test_gpu_reference_python import needs_ref_py, ref_py  # noqa: F401  (ref_py is a fixture)

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _rows(rng, n_vocab):
    """(logit rows, targets): a wide spread, ties at the max, the target at the max, an underflowing target, -inf
    entries, then the rows numpy turns into NaN."""
    rows, targets = [], []

    def add(r, t):
        rows.append(np.asarray(r, np.float32))
        targets.append(int(t))

    for scale in (0.5, 3.0, 30.0):
        add(rng.standard_normal(n_vocab) * scale, rng.integers(0, n_vocab))
    r = np.round(rng.standard_normal(n_vocab) * 2) / 2
    top = np.flatnonzero(r == r.max())
    r[rng.integers(0, n_vocab, 5)] = r.max()
    add(r, top[0])                                                    # ties at the max, target among them
    add(r, np.argmin(r))
    r = rng.standard_normal(n_vocab) * 4
    add(r, np.argmax(r))                                              # target at the max
    add(np.full(n_vocab, 1.25), 3)                                    # all tied
    r = rng.standard_normal(n_vocab)
    r[7] = -1000.0
    add(r, 7)                                                         # e_t underflows: +inf
    r = rng.standard_normal(n_vocab) * 3
    r[rng.random(n_vocab) < 0.5] = -np.inf
    add(r, np.flatnonzero(np.isfinite(r))[0])                         # half -inf, finite target
    add(r, np.flatnonzero(np.isinf(r))[0])                            # -inf target: +inf
    for bad in (np.nan, np.inf):
        r = rng.standard_normal(n_vocab)
        r[11] = bad
        add(r, 2)                                                     # NaN
    add(np.full(n_vocab, -np.inf), 0)                                 # all -inf: NaN
    return np.asarray(rows), np.asarray(targets, np.int32)


@pytest.mark.parametrize("n_vocab", [512, 32000])
def test_extra_nll_equals_the_host_twin(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    path = str(tmp_path / "extra.bin")
    if n_vocab == 512:
        ggjt.write_synth_extra(path, ggjt.SHAPES["tiny128"], ggjt.T_Q4_0, seed=70)
    else:
        ggjt.write_fast_q4_extra(path, ggjt.SHAPES["3b"], seed=70)
    extra = capi.Extra(path, 0)
    assert extra.n_vocab == n_vocab
    rng = np.random.default_rng(n_vocab)
    rows, targets = _rows(rng, n_vocab)
    got = extra.nll(rows, targets)
    want = score_ref.nll_rows(rows, targets)
    assert score_ref.within(got, want).all(), [(k, got[k], want[k]) for k in np.flatnonzero(~score_ref.within(got, want))]
    assert np.isinf(want[7]) and np.isnan(want[-3:]).all() and np.isfinite(want[:7]).all()
    fin = np.isfinite(want)
    err = np.abs(got[fin] - want[fin]) / np.maximum(1, np.abs(want[fin]))
    print("n_vocab %d: largest relative difference from the twin %.3g" % (n_vocab, err.max()))
    # a row's value depends only on its logits and its target: any order, any batch, the same bits
    perm = rng.permutation(len(rows))
    assert (_bits(extra.nll(rows[perm], targets[perm])) == _bits(got[perm])).all()
    assert all(_bits(extra.nll(rows[k:k + 1], targets[k:k + 1]))[0] == _bits(got)[k] for k in range(len(rows)))
    many = np.repeat(rows[:4], 50, axis=0)
    assert (_bits(extra.nll(many, np.repeat(targets[:4], 50))) == _bits(np.repeat(got[:4], 50))).all()
    for bad in (-1, n_vocab):
        with pytest.raises(capi.B200Error) as ei:
            extra.nll(rows[:2], [0, bad])
        assert ei.value.code == 1
    extra.close()


def _host_nll(slices, extra, session, tokens):
    """The client's perplexity through the host: embed tokens[:-1], one session_forward per slice, all logits, twin."""
    x = extra.embed(tokens[:-1])
    for s in slices:
        x = s.session_forward(session, x)
    return score_ref.nll_rows(extra.logits(x), tokens[1:])


@pytest.mark.parametrize("kind", ["q4_0", "f16", "q4_K_M"])
def test_sessions_equal_alone_other_packings_and_the_host_path(tmp_path, kind):
    """5 sessions, two of them mid-context, whose fed rows (186) exceed n_ctx 128: one call packs them into passes
    [3, 0, 4] and [1, 2], the reversed list into [2, 1] and [4, 0, 3], each alone into a pass of its own."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    n_sess = 5
    gpu = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    twin = [capi.Slice(p, 0, 128, n_sessions=n_sess) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(9)
    for sess, n in ((1, 7), (3, 20)):                  # mid-context sessions: the same history on both handle sets
        pre = rng.integers(0, sh.n_vocab, n).tolist()
        for hs in (gpu, twin):
            x = extra.embed(pre)
            for s in hs:
                x = s.session_forward(sess, x)
    sessions = [3, 0, 4, 1, 2]
    lengths = [40, 2, 70, 25, 55]
    texts = [rng.integers(0, sh.n_vocab, n).tolist() for n in lengths]
    before = [s.session_n_past(k) for s in gpu for k in range(n_sess)]
    got = capi.score(gpu, extra, sessions, texts)
    assert [len(g) for g in got] == [n - 1 for n in lengths]
    for s in gpu:
        for j, k in enumerate(sessions):
            assert s.session_n_past(k) == before[k] + lengths[j] - 1
    start = {k: twin[0].session_n_past(k) for k in sessions}

    def rewind():
        for s in twin:
            for k in sessions:
                s.session_rewind(k, start[k])

    rev = capi.score(twin, extra, sessions[::-1], texts[::-1])[::-1]
    rewind()
    worst = 0.0
    for j, k in enumerate(sessions):
        assert (_bits(rev[j]) == _bits(got[j])).all(), (kind, k)
        alone = capi.score(twin, extra, [k], [texts[j]])[0]
        assert (_bits(alone) == _bits(got[j])).all(), (kind, k)
        rewind()
        host = _host_nll(twin, extra, k, texts[j])
        rewind()
        assert np.isfinite(host).all() and score_ref.within(got[j], host).all(), (kind, k)
        worst = max(worst, float((np.abs(got[j] - host) / np.maximum(1, np.abs(host))).max()))
    print("%s: largest relative difference from the host path %.3g" % (kind, worst))
    extra.close()
    for s in gpu + twin:
        s.close()


@pytest.mark.skipif(not os.path.isfile(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle",
                                                    "_ref", "libllmref.so")), reason="oracle/_ref not built")
def test_config1_3b_two_slices_against_the_reference(tmp_path):
    """BASELINE config 1 (OpenLLaMA-3B shapes, layers 0-16 / 17-25, Q4_0 output) on one GPU: b200_score of a 17-token
    text against the twin on the logits the compiled reference computes for it (one call per slice, as
    DistributedLLM.perplexity makes them)."""
    from distributedllm_b200 import capi
    from oracle import oracle
    sh = ggjt.SHAPES["3b"]
    pa, pb, extra_path = str(tmp_path / "a.bin"), str(tmp_path / "b.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(pa, sh, 0, 16, seed=3)
    ggjt.write_fast_q4_slice(pb, sh, 17, 25, seed=3)
    ggjt.write_fast_q4_extra(extra_path, sh, seed=3)
    tokens = [1 + (i * 7919) % 31999 for i in range(17)]
    threads = min(16, os.cpu_count() or 4)
    h = oracle.ref_embed(extra_path, tokens[:-1], sh.n_embd)
    for p in (pa, pb):
        ref = oracle.RefSlice(p, threads, 512)
        h = ref.forward(h)
        ref.close()
    want = score_ref.nll_rows(oracle.ref_logits(extra_path, h, sh.n_vocab, True), tokens[1:])
    gpu = [capi.Slice(pa, 0, 512), capi.Slice(pb, 0, 512)]
    extra = capi.Extra(extra_path, 0)
    got = capi.score(gpu, extra, [0], [tokens])[0]
    assert np.isfinite(want).all() and score_ref.within(got, want).all(), (got, want)
    assert [s.n_past for s in gpu] == [16, 16]
    # the device loop's first greedy id comes from the same rows: the reference's config-1 id
    for s in gpu:
        s.clear_context()
    assert capi.generate_greedy(gpu, extra, [0], [tokens[:16]], 1)[0, 0] == REF["config1"]["ids"][0]
    extra.close()
    for s in gpu:
        s.close()


def test_row_blocks_at_7b_shape(tmp_path):
    """A LLaMA-7B layer with a Q6_K lm_head (32000 x 4096) and a 150-token text: 149 rows, over two full row blocks and
    a partial one.  Every row's NLL is bit-identical to that row's logits computed and scored alone."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    sl, extra_path = str(tmp_path / "layer.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(sl, sh, 0, 0, seed=5)
    ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=5)
    gpu, twin = capi.Slice(sl, 0, 256), capi.Slice(sl, 0, 256)
    extra = capi.Extra(extra_path, 0)
    tokens = [1 + (i * 7919) % 31999 for i in range(150)]
    got = capi.score([gpu], extra, [0], [tokens])[0]
    x = twin.session_forward(0, extra.embed(tokens[:-1]))
    alone = np.array([extra.nll(extra.logits(x[i:i + 1]), [tokens[i + 1]])[0] for i in range(len(x))])
    assert np.isfinite(got).all()
    assert (_bits(got) == _bits(alone)).all(), np.flatnonzero(_bits(got) != _bits(alone))
    extra.close()
    gpu.close()
    twin.close()


def _raw_score(slices, extra, sessions, texts, nll=True):
    from distributedllm_b200 import capi
    ids = np.ascontiguousarray(sessions, dtype=np.int32)
    counts = np.array([len(t) for t in texts], np.int32)
    toks = np.ascontiguousarray([t for p in texts for t in p] or [0], dtype=np.int32)
    handles = (C.c_void_p * len(slices))(*[s.handle for s in slices])
    out = np.zeros(max(int(counts.sum()), 1), np.float64)
    return capi.lib().b200_score(handles, len(slices), extra.handle, capi._ptr(ids), capi._ptr(counts), len(ids),
                                 capi._ptr(toks), capi._ptr(out) if nll else None)


def test_errors_change_nothing(tmp_models, tmp_path):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=47), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=47)]
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=47)
    extra = capi.Extra(extra_path, 0)
    other_path = str(tmp_path / "other.bin")           # n_embd 256
    ggjt.write_synth_slice(other_path, ggjt.SHAPES["tiny"], 0, 0, ggjt.T_Q4_0, seed=47)
    other = capi.Slice(other_path, 0, 64)
    gap = capi.Slice(tmp_models("tiny128", ggjt.T_Q4_0, 2, 2, seed=47), 0, 64)
    x = extra.embed(list(range(3, 53)))                 # session 1 at n_past 50
    for s in gpu:
        x = s.session_forward(1, x)

    def positions():
        return [s.session_n_past(k) for s in gpu for k in range(3)]

    before = positions()
    V = sh.n_vocab
    cases = [
        ("slices out of layer order", [gpu[1], gpu[0]], [0], [[1, 2]], 1),
        ("a gap in the layers", [gpu[0], gap], [0], [[1, 2]], 1),
        ("another n_embd", [other], [0], [[1, 2]], 1),
        ("a handle listed twice", [gpu[0], gpu[0]], [0], [[1, 2]], 1),
        ("session out of range", gpu, [3], [[1, 2]], 1),
        ("negative session", gpu, [-1], [[1, 2]], 1),
        ("session listed twice", gpu, [0, 0], [[1, 2], [3, 4]], 1),
        ("session listed twice in other passes", gpu, [0, 2, 0], [[1] * 40, [3] * 40, [5, 6]], 1),
        ("one token", gpu, [0, 2], [[1, 2], [3]], 1),
        ("no tokens", gpu, [0, 2], [[1, 2], []], 1),
        ("negative token", gpu, [0], [[1, -1, 2]], 1),
        ("target past the vocabulary", gpu, [0], [[1, V]], 1),
        ("context overflow", gpu, [0, 1], [[1, 2], [5] * 16], 5),
        ("a text longer than n_ctx", gpu, [2], [[1] * 66], 5),
    ]
    for what, slices, sessions, texts, code in cases:
        with pytest.raises(capi.B200Error) as ei:
            capi.score(slices, extra, sessions, texts)
        assert ei.value.code == code, (what, str(ei.value))
        assert positions() == before, what
    assert _raw_score(gpu, extra, [0], [[1, 2]], nll=False) == 1
    assert positions() == before
    # the largest call that fits: session 1 ends exactly at n_ctx, session 2 fills a pass of its own
    got = capi.score(gpu, extra, [0, 1, 2], [[1, 2], [5] * 15, list(range(7, 72))])
    assert [len(g) for g in got] == [1, 14, 64] and all(np.isfinite(g).all() for g in got)
    assert [gpu[1].session_n_past(k) for k in range(3)] == [1, 64, 64]
    extra.close()
    for s in [other, gap] + gpu:
        s.close()


def test_handles_on_two_devices_or_in_a_pipeline_are_refused(tmp_models, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    paths = [tmp_models("tiny128", ggjt.T_Q4_0, 0, 0, seed=48), tmp_models("tiny128", ggjt.T_Q4_0, 1, 2, seed=48)]
    extra_path = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra_path, sh, ggjt.T_Q4_0, seed=48)
    extra = capi.Extra(extra_path, 0)
    split = [capi.Slice(paths[0], 0, 64), capi.Slice(paths[1], 1, 64)]
    with pytest.raises(capi.B200Error) as ei:
        capi.score(split, extra, [0], [[1, 2, 3]])
    assert ei.value.code == 1 and "device" in str(ei.value)
    assert [s.n_past for s in split] == [0, 0]
    lib = capi.lib()
    uid = np.zeros(128, np.uint8)
    capi.check(lib.b200_pipeline_unique_id(capi._ptr(uid)))
    rcs = [None, None]

    def join(r):
        rcs[r] = lib.b200_pipeline_init(split[r].handle, r, 2, capi._ptr(uid))

    threads = [threading.Thread(target=join, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert rcs == [0, 0]
    with pytest.raises(capi.B200Error) as ei:
        capi.score(split[:1], extra, [0], [[1, 2, 3]])
    assert ei.value.code == 1 and "pipeline" in str(ei.value)
    assert split[0].n_past == 0
    for s in split:
        capi.check(lib.b200_pipeline_destroy(s.handle))
    extra.close()
    for s in split:
        s.close()


TEXT = "the the a in the a the in a the the in in a the a a the in the"


def _full_model(tmp_path):
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=0)
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    return sh, sl, extra


def _local_perplexity(sl, extra):
    from distributedllm_b200.client import LocalPipeline
    lp = LocalPipeline([sl], [0])
    ppl = lp.perplexity(extra, TEXT)
    assert lp.perplexity(extra, TEXT) == ppl                            # clears the context first
    n_past = lp.slices[0].n_past
    lp.close()
    return ppl, n_past


def _node_perplexity(tmp_path, sh, sl, extra, client):
    """client([address], extra).perplexity(TEXT) through this repo's node server holding the whole model."""
    from distributedllm_b200.compute_node.slices import import_llm
    from distributedllm_b200.control_center import Connection
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        return float(client([addr], extra).perplexity(TEXT))
    finally:
        srv.shutdown()
        srv.server_close()
        import_llm().unload_slice()


def test_local_pipeline_perplexity_equals_the_node_path(tmp_path):
    """LocalPipeline.perplexity (device scoring) against DistributedLLM.perplexity through a node (host softmax)."""
    from distributedllm_b200.client import DistributedLLM
    from distributedllm_b200.compute_node.slices import import_llm
    sh, sl, extra = _full_model(tmp_path)
    want = _node_perplexity(tmp_path, sh, sl, extra, DistributedLLM)
    got, n_past = _local_perplexity(sl, extra)
    n = len(import_llm().tokenize_prompt(extra, TEXT))
    assert n > 16 and n_past == n - 1
    assert np.isfinite(want) and want > 1 and abs(got - want) <= 1e-12 * want, (got, want)


@needs_ref_py
def test_local_pipeline_perplexity_equals_the_reference_client(ref_py, tmp_path):  # noqa: F811
    """The reference's own DistributedLLM.perplexity, unmodified (its Connection, its scipy softmax and sequential sum),
    through a node on this repo's `llm` module, against LocalPipeline.perplexity."""
    from distllm.cli_api.common import DistributedLLM
    sh, sl, extra = _full_model(tmp_path)
    want = _node_perplexity(tmp_path, sh, sl, extra, DistributedLLM)
    got, _ = _local_perplexity(sl, extra)
    assert np.isfinite(want) and want > 1 and abs(got - want) <= 1e-12 * want, (got, want)
