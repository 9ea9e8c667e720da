"""GPU: llama.cpp's windowed perplexity on the device (b200_perplexity_windows, b200_extra_ppl_terms).

* k_ppl_rows (the door) against the host twin client.ppl_terms, bit for bit, at 512, 1031 and 32000 ids.
* The terms are the same bits however many windows share a pass (1, 2, 3 or 8 sessions), and equal the host loop on the
  same slices (b200_session_forward per segment, b200_extra_logits, the twin) for Q4_0, Q4_1, Q5_1, Q8_0, F16, Q4_K_M and
  Q6_K models, and for one LLaMA-7B layer at n_ctx 2048 with n_batch 512 and 2048.
* LocalPipeline.perplexity_windows prints what llama.cpp's `perplexity` printed for the fixture model
  (tests/golden/ppl_windows.json), and DistributedLLM.perplexity_windows through a node gives the same values.
* Fast mode stays near exact mode; exact mode launches no tensor-core kernel.
* Refusals change no position and no cache; handles an open stream owns are refused."""
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from distributedllm_b200.client import ppl_terms, running_perplexity, windowed_perplexity_terms

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import gen_golden_ppl_windows as gen  # noqa: E402
from test_perplexity_windows_ref import FIXTURE  # noqa: E402

pytestmark = pytest.mark.gpu

# Fast mode against exact mode on one LLaMA-7B Q4_0 layer (test_fast_mode_close_to_exact): the largest relative
# difference of a running perplexity measured on an H100 80GB HBM3 was 1.5e-3; the bound leaves room for other weights.
FAST_TOL = 1e-2


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    """Bit-equal, NaNs in the same places (any NaN payload)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return bool((nan == np.isnan(b)).all() and (_bits(a[~nan]) == _bits(b[~nan])).all())


def _rows(rng, n_vocab):
    """(logit rows, targets): spreads, ties at the max, target at the max, an underflowing target, -inf entries, the
    rows with no distribution, and a row whose prob underflows only in float."""
    rows, targets = [], []

    def add(r, t):
        rows.append(np.asarray(r, np.float32))
        targets.append(int(t))

    for scale in (0.5, 3.0, 30.0):
        for _ in range(4):
            add(rng.standard_normal(n_vocab) * scale, rng.integers(0, n_vocab))
    r = np.round(rng.standard_normal(n_vocab) * 2) / 2
    r[rng.integers(0, n_vocab, 5)] = r.max()
    add(r, np.flatnonzero(r == r.max())[0])
    add(r, np.argmin(r))
    r = rng.standard_normal(n_vocab) * 4
    add(r, np.argmax(r))
    add(np.full(n_vocab, 1.25), 3)
    r = rng.standard_normal(n_vocab)
    r[7] = -1000.0
    add(r, 7)                                                       # e_t underflows: +inf
    r = rng.standard_normal(n_vocab) * 0.1
    r[9] = r.max() - 101.0
    add(r, 9)                                                       # e_t a float denormal, e_t / S 0 in float: +inf
    r = rng.standard_normal(n_vocab) * 3
    r[rng.random(n_vocab) < 0.5] = -np.inf
    add(r, np.flatnonzero(np.isfinite(r))[0])
    add(r, np.flatnonzero(np.isinf(r))[0])
    for bad in (np.nan, np.inf):
        r = rng.standard_normal(n_vocab)
        r[11] = bad
        add(r, 2)
    add(np.full(n_vocab, -np.inf), 0)
    return np.asarray(rows), np.asarray(targets, np.int32)


@pytest.mark.parametrize("n_vocab", [512, 1031, 32000])
def test_door_equals_the_host_twin(tmp_path, n_vocab):
    from distributedllm_b200 import capi
    path = str(tmp_path / "extra.bin")
    if n_vocab == 32000:
        ggjt.write_fast_q4_extra(path, ggjt.SHAPES["3b"], seed=71)
    else:
        ggjt.write_synth_extra(path, ggjt.ModelShape(n_vocab, 256, 32, 4, 1), ggjt.T_Q4_0, seed=71)
    extra = capi.Extra(path, 0)
    assert extra.n_vocab == n_vocab
    rng = np.random.default_rng(n_vocab + 1)
    rows, targets = _rows(rng, n_vocab)
    got = extra.ppl_terms(rows, targets)
    want = ppl_terms(rows, targets)
    assert _same(got, want), [(k, got[k], want[k]) for k in range(len(got)) if not _same(got[k:k + 1], want[k:k + 1])]
    assert np.isinf(want[[-7, -6, -4]]).all() and np.isnan(want[-3:]).all() and np.isfinite(want[:8]).all()
    # any batch, any order: the same bits (one block takes 8 rows; 19 rows end part-way into a block)
    perm = rng.permutation(len(rows))
    assert _same(extra.ppl_terms(rows[perm], targets[perm]), got[perm])
    assert _same(extra.ppl_terms(rows[:19], targets[:19]), got[:19])
    assert all(_same(extra.ppl_terms(rows[k:k + 1], targets[k:k + 1]), got[k:k + 1]) for k in range(0, len(rows), 5))
    for bad in (-1, n_vocab):
        with pytest.raises(capi.B200Error) as ei:
            extra.ppl_terms(rows[:2], [0, bad])
        assert ei.value.code == 1
    extra.close()


def _model(tmp_path, kind):
    """Slices and extra layers of one small model of the given weight family: (slice paths, extra path, shape)."""
    d = tmp_path / kind
    d.mkdir()
    paths, extra = [str(d / "a.bin"), str(d / "b.bin")], str(d / "extra.bin")
    block = {"q4_0": ggjt.T_Q4_0, "q4_1": ggjt.T_Q4_1, "q5_1": ggjt.T_Q5_1, "q8_0": ggjt.T_Q8_0, "f16": ggjt.T_F16}
    if kind in block:
        sh = ggjt.SHAPES["tiny128"]
        ggjt.write_synth_slice(paths[0], sh, 0, 0, block[kind], seed=61)
        ggjt.write_synth_slice(paths[1], sh, 1, sh.n_layer - 1, block[kind], seed=61)
        ggjt.write_synth_extra(extra, sh, block[kind], seed=61)
    else:
        sh = ggjt.SHAPES["tinyk128"]
        ggjt.write_kquant_slice(paths[0], sh, 0, 3, kind, seed=62)
        ggjt.write_kquant_slice(paths[1], sh, 4, sh.n_layer - 1, kind, seed=62)
        ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=62)          # Q6_K output.weight, Q4_K tok_embeddings
    return paths, extra, sh


def _host_loop(slices, extra, tokens, n_ctx, n_batch, session=0):
    """perplexity.cpp's loop through the host: b200_session_forward per segment, b200_extra_logits, the twin."""
    def eval_segment(ids, n_past):
        if n_past == 0:
            for s in slices:
                s.session_clear(session)
        x = extra.embed(ids)
        for s in slices:
            x = s.session_forward(session, x)
        return extra.logits(x)

    terms = windowed_perplexity_terms(tokens, n_ctx, n_batch, eval_segment)
    for s in slices:
        s.session_clear(session)
    return terms


@pytest.mark.parametrize("kind", ["q4_0", "q4_1", "q5_1", "q8_0", "f16", "q4_K_M", "q6_K"])
def test_packings_and_the_host_loop(tmp_path, kind):
    """9 windows of 32 ids (and a partial one) in segments of 12, 12 and 8 rows; slice n_ctx 96 admits 8 segments per
    pass.  Waves of 1, 2, 3 and 8 windows give the same bits, equal to the host loop."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, kind)
    gpu = [capi.Slice(p, 0, 96, n_sessions=8) for p in paths]
    extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(3)
    tokens = rng.integers(0, sh.n_vocab, 9 * 32 + 17).tolist()
    x = extra.embed(tokens[:5])                         # sessions mid-context before the call
    for s in gpu:
        x = s.session_forward(6, x)
    got = {}
    for sessions in ([0], [5, 2], [7, 0, 3], [6, 1, 2, 3, 4, 5, 7, 0]):
        got[len(sessions)] = capi.perplexity_windows(gpu, extra, sessions, tokens, 32, 12)
        assert all(s.session_n_past(k) == 0 for s in gpu for k in sessions)
    ref = got[1]
    assert ref.shape == (9, 32 - 1 - 16) and np.isfinite(ref).all()
    for w, t in got.items():
        assert _same(t, ref), (kind, w)
    host = _host_loop(gpu, extra, tokens, 32, 12)
    assert _same(ref, host), (kind, np.flatnonzero(_bits(ref) != _bits(host)))
    # n_batch larger than n_ctx is cut to n_ctx: one 32-row segment per window, 3 windows per pass
    one = capi.perplexity_windows(gpu, extra, [0, 1, 2], tokens, 32, 500)
    assert _same(one, _host_loop(gpu, extra, tokens, 32, 32)), kind
    extra.close()
    for s in gpu:
        s.close()


@pytest.mark.parametrize("n_batch", [512, 2048])
def test_7b_layer_at_n_ctx_2048(tmp_path, n_batch):
    """One LLaMA-7B Q4_0 layer with a Q6_K lm_head, two windows of 2048 ids (first scored row 512)."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    sl, extra_path = str(tmp_path / "layer.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(sl, sh, 0, 0, seed=8)
    ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=8)
    gpu = capi.Slice(sl, 0, 2048, n_sessions=2)
    extra = capi.Extra(extra_path, 0)
    tokens = [(i * 7919 + 13) % sh.n_vocab for i in range(2 * 2048 + 100)]
    got = capi.perplexity_windows([gpu], extra, [0, 1], tokens, 2048, n_batch)
    assert got.shape == (2, 2048 - 1 - 512) and np.isfinite(got).all()
    host = _host_loop([gpu], extra, tokens, 2048, n_batch)
    assert _same(got, host), np.flatnonzero(_bits(got) != _bits(host))
    print("n_batch %d: running perplexity %s" % (n_batch, running_perplexity(got)))
    extra.close()
    gpu.close()


def test_local_pipeline_prints_what_llama_cpp_printed(tmp_path):
    from distributedllm_b200.client import LocalPipeline
    full = str(tmp_path / "full.bin")
    assert gen.write_model(full) == FIXTURE["model_sha256"]
    sh = ggjt.SHAPES[gen.SHAPE]
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    lp = LocalPipeline([sl], [0], n_ctx=64, n_sessions=4)
    for case in FIXTURE["cases"]:
        got = lp.perplexity_windows(extra, gen.text(), case["n_ctx"], case["n_batch"])
        assert ["%.4f" % v for v in got] == case["printed"], (case, got)
        assert lp.perplexity_windows(extra, gen.text(), case["n_ctx"], case["n_batch"], sessions=[2]) == got
    assert lp.slices[0].session_n_past(0) == 0
    lp.close()


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return {ev.key for ev in prof.key_averages()}


def test_fast_mode_close_to_exact(tmp_path):
    """One LLaMA-7B Q4_0 layer, 4 windows of 512: fast mode's running perplexities within FAST_TOL of exact mode's;
    exact mode launches no tensor-core matmul (k_gemm_tc2), fast mode does."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    sl, extra_path = str(tmp_path / "layer.bin"), str(tmp_path / "extra.bin")
    ggjt.write_fast_q4_slice(sl, sh, 0, 0, seed=9)
    ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=9)
    gpu = capi.Slice(sl, 0, 1024, n_sessions=2)
    extra = capi.Extra(extra_path, 0)
    tokens = [(i * 104729 + 7) % sh.n_vocab for i in range(4 * 512)]
    out = {}
    names = {}
    for fast in (False, True):
        names[fast] = _kernel_names(lambda: out.__setitem__(fast, capi.perplexity_windows([gpu], extra, [0, 1], tokens,
                                                                                          512, 512, fast=fast)))
    assert not any("k_gemm_tc2" in k for k in names[False]), sorted(names[False])
    assert any("k_gemm_tc2" in k for k in names[True]), sorted(names[True])
    assert any("k_ppl_rows" in k for k in names[False])
    a, b = np.asarray(running_perplexity(out[False])), np.asarray(running_perplexity(out[True]))
    rel = float(np.max(np.abs(b - a) / a))
    print("fast against exact: running perplexities %s / %s, largest relative difference %.3g" % (a, b, rel))
    assert np.isfinite(b).all() and rel <= FAST_TOL
    # the fast terms too are the same bits in any packing
    assert _same(capi.perplexity_windows([gpu], extra, [1], tokens, 512, 512, fast=True), out[True])
    extra.close()
    gpu.close()


def test_errors_change_nothing(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    twin = [capi.Slice(p, 0, 64, n_sessions=3) for p in paths]
    extra = capi.Extra(extra_path, 0)
    other_path = str(tmp_path / "other.bin")                 # n_embd 256
    ggjt.write_synth_slice(other_path, ggjt.SHAPES["tiny"], 0, 0, ggjt.T_Q4_0, seed=61)
    other = capi.Slice(other_path, 0, 64)
    pre = list(range(3, 43))
    for hs in (gpu, twin):                                   # session 1 at n_past 40 on both handle sets
        x = extra.embed(pre)
        for s in hs:
            x = s.session_forward(1, x)
    before = [s.session_n_past(k) for s in gpu for k in range(3)]
    V = sh.n_vocab
    toks = list(range(5, 5 + 70))
    lib = capi.lib()
    import ctypes as C

    def raw(slices, sessions, tokens, n_ctx, n_batch):
        ids = np.ascontiguousarray(sessions, np.int32)
        t = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(4096, np.float32)
        h = (C.c_void_p * len(slices))(*[s.handle for s in slices])
        return lib.b200_perplexity_windows(h, len(slices), extra.handle, capi._ptr(ids), len(ids), capi._ptr(t), len(t),
                                           n_ctx, n_batch, 0, capi._ptr(out))

    cases = [
        ("slices out of layer order", [gpu[1], gpu[0]], [0], toks, 16, 8, 1),
        ("another n_embd", [other], [0], toks, 16, 8, 1),
        ("a handle listed twice", [gpu[0], gpu[0]], [0], toks, 16, 8, 1),
        ("session out of range", gpu, [3], toks, 16, 8, 1),
        ("negative session", gpu, [-1], toks, 16, 8, 1),
        ("session listed twice", gpu, [0, 2, 0], toks, 16, 8, 1),
        ("n_ctx 1", gpu, [0], toks, 1, 1, 1),
        ("n_batch 0", gpu, [0], toks, 16, 0, 1),
        ("negative id", gpu, [0], toks[:40] + [-1], 16, 8, 1),
        ("id past the vocabulary", gpu, [0], toks + [V], 16, 8, 1),
        ("no sessions", gpu, [], toks, 16, 8, 1),
        ("n_ctx over the slices' n_ctx", gpu, [0], toks * 2, 65, 8, 5),
    ]
    for what, slices, sessions, tokens, n_ctx, n_batch, code in cases:
        assert raw(slices, sessions, tokens, n_ctx, n_batch) == code, (what, capi.lib().b200_last_error())
        assert [s.session_n_past(k) for s in gpu for k in range(3)] == before, what
    # session 1 continues exactly as on the handles that saw no error: its cache is untouched
    nxt = list(range(50, 60))
    outs = []
    for hs in (gpu, twin):
        x = extra.embed(nxt)
        for s in hs:
            x = s.session_forward(1, x)
        outs.append(x)
    assert (outs[0].view(np.uint32) == outs[1].view(np.uint32)).all()
    # fewer ids than one window: zero windows, no error, the listed sessions cleared
    got = capi.perplexity_windows(gpu, extra, [0, 1], toks[:15], 16, 8)
    assert got.shape == (0, 7) and [s.session_n_past(1) for s in gpu] == [0, 0]
    extra.close()
    for s in [other] + gpu + twin:
        s.close()


def test_stream_owned_handles_are_refused(tmp_path):
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 64, n_sessions=2) for p in paths]
    extra = capi.Extra(extra_path, 0)
    toks = list(range(5, 70))
    want = capi.perplexity_windows(gpu, extra, [0], toks, 32, 16)
    with capi.Stream(gpu, extra):
        with pytest.raises(capi.B200Error) as ei:
            capi.perplexity_windows(gpu, extra, [1], toks, 32, 16)
        assert ei.value.code == 1 and "stream" in str(ei.value)
        with pytest.raises(capi.B200Error):
            extra.ppl_terms(np.zeros((1, sh.n_vocab), np.float32), [0])
    assert _same(capi.perplexity_windows(gpu, extra, [1], toks, 32, 16), want)
    extra.close()
    for s in gpu:
        s.close()


def test_distributed_llm_through_a_node_equals_local_pipeline(tmp_path):
    """DistributedLLM.perplexity_windows (the host loop: segments through a node, get_logits(all), the twin) against
    LocalPipeline.perplexity_windows on the fixture model: the same running perplexities, float for float."""
    from distributedllm_b200.client import DistributedLLM, LocalPipeline
    from distributedllm_b200.compute_node.slices import import_llm
    from distributedllm_b200.control_center import Connection
    from test_gpu_generate import _serve
    full = str(tmp_path / "full.bin")
    gen.write_model(full)
    sh = ggjt.SHAPES[gen.SHAPE]
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    case = FIXTURE["cases"][0]
    srv = _serve(tmp_path)
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            name = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})["file_name"]
        conn.load_slice(name)
        host = DistributedLLM([addr], extra).perplexity_windows(gen.text(), case["n_ctx"], case["n_batch"])
    finally:
        srv.shutdown()
        srv.server_close()
        import_llm().unload_slice()
    lp = LocalPipeline([sl], [0], n_ctx=64, n_sessions=2)
    got = lp.perplexity_windows(extra, gen.text(), case["n_ctx"], case["n_batch"])
    lp.close()
    assert host == got and ["%.4f" % v for v in host] == case["printed"], (host, got)
