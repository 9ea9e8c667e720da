"""GPU: the wgmma "fast mode" prefill (csrc/fastgemm2.cuh, layer_fast) checked per matmul against the float64 bound of
tests/test_gpu_fast_prefill.py in every kind of call that reaches it, not only a one-layer prompt from position 0:
  * prompt calls of 1000 and 2047 rows at n_ctx 2048 (LLaMA-7B Q4_0 / Q8_0, 3B Q4_0): grids of more than 4 token tiles
    with a ragged last one;
  * Q8_0 at 3B (head size 100; w2's K = 8640 ends in a half-filled 128-wide quad) and at 13B;
  * a 700-row chunk at n_past 300 in session 2 of a 4-session slice, whose context passes the 512-row staged window;
  * the last layer of a 2-layer slice that starts at layer 5 (input read from xa);
  * the last fast pass of b200_perplexity_windows: two windows' segments in one mixed pass, rebuilt from the ids;
each with fast_ref.check_layer: xh == prep(gate) bit for bit, every matmul within TAU * sum_k |w16 * x16| on a row and
token sample, and one lost 32-wide K block in the reference moving >= LOST_BLOCK of the outputs outside the bound.
And what fast mode leaves exact:
  * decode after a fast prefill: single-token steps (graphed and not), decode rows, a batched step and a mixed pass
    carrying a prompt chunk give the same bits on the fast handle and on an exact handle restored from its caches;
  * calls below min_tokens and calls after the switch is turned off are exact mode's bits and run no fast-mode layer;
  * Q4_1 and F16 slices ignore the switch.
Which schedule a call ran is read from xh, not from a profiler: k_gemm_tc2 runs only in layer_fast, which writes w2's
fp16 input there with k_prep_q8_f16, and no exact-mode kernel touches xh.  So a call that leaves xh as it was ran no
fast layer, and a call after which xh == prep(gate) ran its last layer in fast mode.
TAU, TAU_LONG and the LOST_BLOCK floor are test_gpu_fast_prefill's; the largest values measured here are listed below."""
import time

import numpy as np
import pytest

import fast_ref
from distributedllm_b200 import ggjt
from test_gpu_fast_prefill import LOST_BLOCK, _n_sm, tau, tile_plan

pytestmark = pytest.mark.gpu

# Largest normalised error |y - y_ref| / sum_k |w16 * x16| per case (every time in w2, the longest K), measured on an
# NVIDIA H100 80GB HBM3 (700 W power limit):
#   7b q4_0 N=1000 1.44e-6   7b q4_0 N=2047 1.44e-6   7b q8_0 N=1000 1.44e-6   7b q8_0 N=2047 1.39e-6
#   3b q4_0 N=1000 1.26e-6   3b q8_0 N=300 1.23e-6    13b q8_0 N=300 1.60e-6
#   session 2, 700 rows at n_past 300 1.33e-6   layer 6 of 5-6 q4_0 1.45e-6, q8_0 1.46e-6
#   perplexity pass n_batch 512 1.43e-6, n_batch 256 1.43e-6
# All below the largest of test_gpu_fast_prefill (1.73e-6, 13b q4_0) and so inside TAU = 2^-17; the largest K here is
# 11008 <= LONG_K.  No constant is re-derived.
# The lost-block share is a property of the reference data, not of the kernel: which outputs stay inside the bound
# depends on how large the zeroed block's contribution is against sum_k |w16 * x16|.  Measured from one token's outputs
# (the ~736 sampled w2 rows), as test_gpu_fast_prefill does, it ranged 0.9872 .. 0.9999 over these cases and fell below
# LOST_BLOCK = 0.99 in w2 three times (3b q8_0 0.9872, layer 6 q4_0 0.9891, perplexity pass n_batch 256 0.9878): a
# 0.99 floor is within about two binomial standard deviations of such a 736-output estimate.  So these cases keep the
# floor and pool LOST_TOKENS tokens, spread from the first sampled token to the last, into one estimate.  Pooled, the
# smallest share was 0.9915 (perplexity pass n_batch 256, w2; its tokens one by one 0.9837 .. 0.9973), and 0.9926 ..
# 0.9956 in w2 of the other cases (same GPU, same power limit).
LOST_TOKENS = 8

def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _same_bits(a, b) -> int:
    """How many floats differ in their bits."""
    return int((_bits(a) != _bits(b)).sum())


def _xh(gpu, n: int, n_ff: int) -> np.ndarray:
    """The first n rows of xh as [n][n_ff] fp16 bits: where a fast-mode layer leaves w2's input (see the docstring)."""
    return gpu.debug_read(9, n * n_ff // 2, np.uint32).view(np.uint16).reshape(n, n_ff)


def _ran_fast(gpu, n: int, n_ff: int) -> bool:
    """Did the last n-row call run its last layer in fast mode: is xh that layer's prep(gate), bit for bit?"""
    gate = gpu.debug_read(3, n * n_ff).reshape(n, n_ff)
    return bool(np.array_equal(_xh(gpu, n, n_ff), fast_ref.prep(gate).view(np.uint16)))


def _without_fast_layer(gpu, n: int, n_ff: int, call):
    """call() -> its result; asserts that it left the first n rows of xh as they were, so ran no fast layer."""
    before = _xh(gpu, n, n_ff).copy()
    out = call()
    changed = int((_xh(gpu, n, n_ff) != before).sum())
    assert changed == 0, "the call wrote %d halves of xh: a fast-mode layer ran" % changed
    return out


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    """Slices at the real model shapes from the benchmark's block-pool writer: (shape, wtype, first, last) -> path."""
    root = tmp_path_factory.mktemp("big_calls")
    cache = {}

    def get(shape: str, wtype: int, first: int = 0, last: int = 0) -> str:
        key = (shape, wtype, first, last)
        if key not in cache:
            p = str(root / ("%s_%s_%d_%d.bin" % (shape, ggjt.TYPE_NAME[wtype], first, last)))
            ggjt.write_fast_q4_slice(p, ggjt.SHAPES[shape], first, last, seed=9, wtype=wtype)
            cache[key] = p
        return cache[key]

    return get


def _check(w, x, gpu, y, label, t0):
    n = x.shape[0]
    tokens = fast_ref.token_sample(n)
    worst, lost = fast_ref.check_layer(w, x, fast_ref.read_layer(gpu, n, w.E, w.FF), y, tau, LOST_BLOCK, label, tokens,
                                       lost_tokens=LOST_TOKENS)
    big_mat = max(worst, key=worst.get)
    print("[fast-calls] %s  largest %.3g (2^%.2f, %s)  smallest lost-block share %.4f  %d of %d tokens  %.1f s" % (
        label, worst[big_mat], np.log2(max(worst[big_mat], 1e-30)), big_mat, min(lost.values()), len(tokens), n,
        time.time() - t0))
    return worst


# ------------------------------------------------------------------------------------ one-layer prompt calls
PROMPT_CASES = [("7b", ggjt.T_Q4_0, 1000), ("7b", ggjt.T_Q4_0, 2047), ("7b", ggjt.T_Q8_0, 1000), ("7b", ggjt.T_Q8_0, 2047),
                ("3b", ggjt.T_Q4_0, 1000),
                ("3b", ggjt.T_Q8_0, 300),       # head size 100 (generic attention); w2: K = 8640, a half-filled last quad
                ("13b", ggjt.T_Q8_0, 300)]


@pytest.mark.parametrize("shape,wtype,n", PROMPT_CASES,
                         ids=["%s-%s-N%d" % (s, ggjt.TYPE_NAME[t], n) for s, t, n in PROMPT_CASES])
def test_prompt_call_within_the_float64_bound(big, shape, wtype, n):
    """One prompt call of n rows from position 0 through a one-layer slice at n_ctx 2048.  Calls of 1000 rows and more
    run grids of more than 4 token tiles, every one with a ragged last tile."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    t0 = time.time()
    path = big(shape, wtype)
    if n >= 1000:
        plan = tile_plan(shape, wtype, n, _n_sm())
        print("\n[fast-calls] %s %s N=%d tile plan %s" % (shape, ggjt.TYPE_NAME[wtype], n, plan))
        assert max(p[1] for p in plan.values()) > 4 and all(p[2] for p in plan.values()), plan
    w = fast_ref.LayerWeights(path, 0, sh.n_embd, sh.n_ff)
    gpu = capi.Slice(path, 0, 2048)
    try:
        gpu.set_fast_prefill(True, 32)
        x = np.random.default_rng([n, sh.n_embd, 3]).standard_normal((n, sh.n_embd), dtype=np.float32)
        y = gpu.forward(x)
        _check(w, x, gpu, y, "%s %s N=%d" % (shape, ggjt.TYPE_NAME[wtype], n), t0)
    finally:
        gpu.close()


# ------------------------------------------------------------------------------------ later chunks, other sessions
def test_later_chunk_in_another_session(big):
    """Session 2 of a 4-session LLaMA-7B Q4_0 slice at n_ctx 2048: a 300-row chunk, then a 700-row chunk at n_past 300,
    whose context (1000 rows) passes the 512-row staged window, so its attention runs the per-query cluster kernel on
    fast-made q / k / v.  The second chunk's matmuls are checked."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    t0 = time.time()
    path = big("7b", ggjt.T_Q4_0)
    w = fast_ref.LayerWeights(path, 0, sh.n_embd, sh.n_ff)
    gpu = capi.Slice(path, 0, 2048, n_sessions=4)
    try:
        gpu.set_fast_prefill(True, 32)
        rng = np.random.default_rng(31)
        gpu.session_forward(2, rng.standard_normal((300, sh.n_embd), dtype=np.float32))
        assert gpu.session_n_past(2) == 300 and gpu.session_n_past(0) == 0
        x = rng.standard_normal((700, sh.n_embd), dtype=np.float32)
        y = gpu.session_forward(2, x)
        assert gpu.session_n_past(2) == 1000
        _check(w, x, gpu, y, "7b q4_0 session 2 N=700 at n_past 300", t0)
    finally:
        gpu.close()


# ------------------------------------------------------------------------------------ several layers
@pytest.mark.parametrize("wtype", [ggjt.T_Q4_0, ggjt.T_Q8_0], ids=["q4_0", "q8_0"])
def test_last_of_two_layers(big, wtype):
    """A slice of LLaMA-7B layers 5 and 6: layer 5 writes xa, layer 6 reads it and writes the call's output, and both
    reuse xh.  Layer 6's matmuls are checked against its input read from xa."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    E, n = sh.n_embd, 300
    t0 = time.time()
    path = big("7b", wtype, 5, 6)
    w = fast_ref.LayerWeights(path, 6, E, sh.n_ff)
    gpu = capi.Slice(path, 0, 1024)
    try:
        gpu.set_fast_prefill(True, 32)
        x = np.random.default_rng(32).standard_normal((n, E), dtype=np.float32)
        y = gpu.forward(x)
        x6 = gpu.debug_read(4, n * E).reshape(n, E)
        assert np.isfinite(x6).all() and (_bits(x6) != _bits(x)).any(axis=1).all()     # layer 5 changed every row
        _check(w, x6, gpu, y, "7b %s layers 5-6, layer 6 N=%d" % (ggjt.TYPE_NAME[wtype], n), t0)
    finally:
        gpu.close()


# ------------------------------------------------------------------------------------ the windowed perplexity's passes
@pytest.fixture(scope="module")
def ppl_model(tmp_path_factory):
    """One LLaMA-7B Q4_0 layer and a Q4_K_M extra (Q6_K lm_head), as in test_gpu_perplexity_windows."""
    root = tmp_path_factory.mktemp("ppl_calls")
    sh = ggjt.SHAPES["7b"]
    sl, extra = str(root / "layer.bin"), str(root / "extra.bin")
    ggjt.write_fast_q4_slice(sl, sh, 0, 0, seed=9)
    ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=9)
    return sl, extra


@pytest.mark.parametrize("n_batch", [512, 256])
def test_perplexity_fast_pass(ppl_model, n_batch):
    """4 windows of 512 ids over 2 sessions of a slice at n_ctx 1024: 2 windows per wave.  The call's last pass holds
    the last segment of windows 2 and 3: two 512-row segments from n_past 0 (n_batch 512), or two 256-row segments at
    n_past 256 (n_batch 256).  Its input rows are rebuilt with Extra.embed from the ids the call feeds (BOS = 1 at each
    window's position 0), its output is read from the slice's d_out, and all four matmuls are checked over both
    segments.  Exact mode on the same call runs no fast-mode layer: it leaves xh as it was."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    E, FF, n_ctx = sh.n_embd, sh.n_ff, 512
    t0 = time.time()
    sl, extra_path = ppl_model
    w = fast_ref.LayerWeights(sl, 0, E, FF)
    gpu = capi.Slice(sl, 0, 1024, n_sessions=2)
    extra = capi.Extra(extra_path, 0)
    try:
        tokens = [(i * 104729 + 7) % sh.n_vocab for i in range(4 * n_ctx)]
        exact = _without_fast_layer(gpu, 1024, FF, lambda: capi.perplexity_windows(
            [gpu], extra, [0, 1], tokens, n_ctx, n_batch))
        fast = capi.perplexity_windows([gpu], extra, [0, 1], tokens, n_ctx, n_batch, fast=True)   # last: its buffers stay
        assert np.isfinite(exact).all() and np.isfinite(fast).all() and _same_bits(fast, exact) > 0
        j0 = n_ctx - n_batch
        ids = [1 if j == 0 else tokens[c * n_ctx + j] for c in (2, 3) for j in range(j0, n_ctx)]
        n = len(ids)
        x = extra.embed(ids)
        y = gpu.debug_read(10, n * E).reshape(n, E)
        _check(w, x, gpu, y, "7b q4_0 perplexity pass n_batch %d: 2 segments of %d at n_past %d" % (
            n_batch, n_batch, j0), t0)
    finally:
        extra.close()
        gpu.close()


# ------------------------------------------------------------------------------------ decode after a fast prefill
@pytest.mark.parametrize("shape", ["tiny128b", "7b"])
def test_decode_after_a_fast_prefill_is_exact(tmp_models, big, monkeypatch, shape):
    """A fast handle (min_tokens 32) prefills sessions with fast chunks; their caches are saved and restored into an
    exact handle of the same file.  Both then take the same continuation -- single-token steps, decode rows
    (session_forward_steps), a batched step and a mixed pass carrying a prompt chunk -- with the decode graph and
    without it (B200_GRAPH=0): every output float and the final caches are the same bits.  At 7B (one layer, n_ctx
    2048) both sessions are past position 512."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    E = sh.n_embd
    if shape == "tiny128b":
        path, n_ctx, chunks = tmp_models("tiny128b", ggjt.T_Q4_0, 0, 1, seed=25), 256, {0: (40, 72), 1: (100,)}
    else:
        path, n_ctx, chunks = big("7b", ggjt.T_Q4_0), 2048, {0: (300, 260), 1: (540,)}
    for graph in ("1", "0"):
        monkeypatch.setenv("B200_GRAPH", graph)
        rng = np.random.default_rng([33, int(graph)])
        fast, exact = capi.Slice(path, 0, n_ctx, n_sessions=3), capi.Slice(path, 0, n_ctx, n_sessions=3)
        try:
            fast.set_fast_prefill(True, 32)
            for k, ns in chunks.items():
                for n in ns:
                    fast.session_forward(k, rng.standard_normal((n, E), dtype=np.float32))
                    assert _ran_fast(fast, n, sh.n_ff), (shape, graph, k, n)
            for k in chunks:
                exact.session_restore(k, fast.session_save(k))
                assert exact.session_n_past(k) == fast.session_n_past(k) == sum(chunks[k])

            def both(what, call):
                a, b = call(fast), call(exact)
                assert np.isfinite(a).all()
                assert _same_bits(a, b) == 0, "%s graph=%s %s: %d of %d floats differ" % (
                    shape, graph, what, _same_bits(a, b), a.size)

            for step in range(3):
                for k in chunks:
                    x = rng.standard_normal((1, E), dtype=np.float32)
                    both("step %d session %d" % (step, k), lambda s: s.session_forward(k, x))
            x = rng.standard_normal((4, E), dtype=np.float32)
            both("decode rows", lambda s: s.forward_steps(0, x))
            x = rng.standard_normal((2, E), dtype=np.float32)
            both("batched step", lambda s: s.batch_forward([1, 0], x))
            x = rng.standard_normal((1 + 40 + 33, E), dtype=np.float32)
            both("mixed pass", lambda s: s.mixed_forward([0, 2, 1], [1, 40, 33], x))
            for k in (2, 1):
                x = rng.standard_normal((1, E), dtype=np.float32)
                both("step after the mixed pass, session %d" % k, lambda s: s.session_forward(k, x))
            for k in range(3):
                assert fast.session_save(k) == exact.session_save(k), (shape, graph, k)
        finally:
            fast.close()
            exact.close()


# ------------------------------------------------------------------------------------ threshold and switch
def test_min_tokens_and_the_switch(tmp_models):
    """min_tokens m = 40: a 39-row call gives the exact handle's bits and runs no fast-mode layer, a 40-row call runs
    fast mode; after set_fast_prefill(False) calls give exact bits again and run no fast-mode layer."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128b"]
    m, E, FF = 40, sh.n_embd, sh.n_ff
    path = tmp_models("tiny128b", ggjt.T_Q4_0, 0, 1, seed=26)
    fast, exact = capi.Slice(path, 0, 256), capi.Slice(path, 0, 256)
    try:
        fast.set_fast_prefill(True, m)
        rng = np.random.default_rng(34)
        x = rng.standard_normal((m - 1, E), dtype=np.float32)
        below = _without_fast_layer(fast, m, FF, lambda: fast.forward(x))
        assert _same_bits(below, exact.forward(x)) == 0
        for s in (fast, exact):
            s.clear_context()
        x = rng.standard_normal((m, E), dtype=np.float32)
        at = fast.forward(x)
        assert _ran_fast(fast, m, FF)
        assert _same_bits(at, exact.forward(x)) > 0                 # a different code path, at the same positions
        for s in (fast, exact):
            s.clear_context()
        fast.set_fast_prefill(False)
        for n in (64, m, 1):
            x = rng.standard_normal((n, E), dtype=np.float32)
            off = _without_fast_layer(fast, 64, FF, lambda: fast.forward(x))
            assert _same_bits(off, exact.forward(x)) == 0, n
    finally:
        fast.close()
        exact.close()


@pytest.mark.parametrize("wtype", [ggjt.T_Q4_1, ggjt.T_F16], ids=["q4_1", "f16"])
def test_q4_1_and_f16_ignore_the_switch(tmp_models, wtype):
    """Q4_1 and F16 slices with fast mode on (min_tokens 32) give exactly the bits of the switch off on prompts of 64
    and 100 rows and a step, and run no fast-mode layer."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128b"]
    path = tmp_models("tiny128b", wtype, 0, 1, seed=27)
    on, off = capi.Slice(path, 0, 256), capi.Slice(path, 0, 256)
    try:
        on.set_fast_prefill(True, 32)
        rng = np.random.default_rng(35)
        for n in (64, 100, 1):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            got = _without_fast_layer(on, 100, sh.n_ff, lambda: on.forward(x))
            assert np.isfinite(got).all() and _same_bits(got, off.forward(x)) == 0, n
    finally:
        on.close()
        off.close()
