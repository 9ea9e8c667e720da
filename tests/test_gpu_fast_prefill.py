"""GPU: the wgmma "fast mode" prefill (csrc/fastgemm2.cuh) against exact mode and against a float64
restatement of each matmul (tests/fast_ref.py).

Fast mode is NOT bit-exact by design: the weight matmuls run as fp16 x fp16 -> fp32 tensor-core MMAs on operands
that went through the reference's Q8_0 activation quantisation and one fp16 rounding each.  Stated tolerances:
  * each weight matmul (qkv, wo + residual, w1|w3 + SiLU gate, w2 + residual) against the float64 sum of the same fp16
    operands: |y - y_ref| <= TAU * sum_k |w16 * x16| (+ one fp32 ulp of |y| for a residual add), TAU below (TAU_LONG
    for K > 13824);
  * one weight matmul against exact mode (qkv of the first layer): relative RMS error <= 1e-3 (measured 2.7e-4: fp16
    operand rounding + fp32 accumulation order);
  * slice output (hidden states, 2 layers): relative RMS error <= 1.5e-2.  Most of it is not the tensor core: every
    following matmul re-quantises its input to Q8_0 like the reference does, and a 3e-4 perturbation flips ~5-10 %
    of the 8-bit codes by one step (measured 4.7e-3 after one layer, 8.7e-3 after two) -- the same order as the
    quantisation noise the reference itself carries relative to fp32 math.
Fast mode applies to prefill calls only: single-token and batched steps stay exact whatever min_tokens is.
Exact mode stays the default and is what every parity claim refers to."""
import time

import numpy as np
import pytest

import fast_ref
from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu

# Largest normalised error |y - y_ref| / sum_k |w16 * x16| of test_each_fast_matmul_is_within_the_float64_bound, measured
# on an NVIDIA H100 80GB HBM3 (400 W power limit), per case over all its token counts and matmuls (w2, the longest K,
# is the largest in every case):
#   7b q4_0 v2 1.53e-6   7b q8_0 v2 1.55e-6   13b q4_0 v2 1.73e-6   3b q4_0 v2 1.42e-6
#   tiny128b q4_0 v2 5.54e-7   tiny128b q8_0 v2 5.74e-7
# The error grows with K (2.5e-7 at K = 512, 7e-7 at 4096, 1.7e-6 at 13824): the tensor core adds each k16 product
# group into the fp32 accumulator with less than round-to-nearest accuracy (the same fp16 products summed in fp32
# by a CPU BLAS stay below 5e-8 at K = 11008).  TAU is 4x the largest, rounded up to a power of two.  At TAU, zeroing one 32-wide activation block puts >= 99.05 % of a token's outputs outside the bound.
# The longer K of LLaMA-30B / 65B (same GPU, same power limit), largest per case, every time in w2:
#   30b q4_0 v2 1.80e-6   30b q8_0 v2 1.95e-6   65b q4_0 v2 2.17e-6   65b q8_0 v2 1.99e-6
# The matmuls with K <= 6656 .. 8192 stay below 9.5e-7.  By the same rule the matmuls with K > LONG_K (w2 of 30B and
# 65B, K = 17920 and 22016) get TAU_LONG, the others keep TAU.  Zeroing one of the 560 / 688 activation blocks moves a
# smaller share of such a sum: at these shapes it put >= 96.78 % of a token's outputs outside the bound (30b q8_0 w2;
# >= 98.95 % for the matmuls with K <= 8192), so they are held to LOST_BLOCK_LARGE.
MEASURED = 1.73e-6
TAU = 2.0 ** -17
LONG_K = 13824
MEASURED_LONG = 2.17e-6
TAU_LONG = 2.0 ** -16
assert TAU <= 2.0 ** -16 and TAU == 2.0 ** np.ceil(np.log2(4 * MEASURED))
assert TAU_LONG <= 2.0 ** -16 and TAU_LONG == 2.0 ** np.ceil(np.log2(4 * MEASURED_LONG))
LOST_BLOCK = 0.99
LOST_BLOCK_LARGE = 0.95          # the 30b / 65b cases


def tau(k: int) -> float:
    return TAU if k <= LONG_K else TAU_LONG


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def big_models(tmp_path_factory):
    """One-layer slices at the real model shapes from the benchmark's block-pool writer (shape, wtype) -> path."""
    root = tmp_path_factory.mktemp("big")
    cache = {}

    def get(shape: str, wtype: int) -> str:
        if (shape, wtype) not in cache:
            p = str(root / ("%s_%s.bin" % (shape, ggjt.TYPE_NAME[wtype])))
            ggjt.write_fast_q4_slice(p, ggjt.SHAPES[shape], 0, 0, seed=9, wtype=wtype)
            cache[(shape, wtype)] = p
        return cache[(shape, wtype)]

    return get


_V = {ggjt.T_Q4_0: "v2-tma-n256-q4_0", ggjt.T_Q8_0: "v2-tma-n256-q8_0"}
_LAYER_CASES = [pytest.param("tiny128b", n, wt, id="%d-%s" % (n, _V[wt]))
                for wt in _V for n in (128, 200, 33, 300)]
_LAYER_CASES += [pytest.param(shape, 512, wt, id="%s-512-%s" % (shape, _V[wt]))
                 for shape in ("7b", "30b", "65b") for wt in (ggjt.T_Q4_0, ggjt.T_Q8_0)]


@pytest.mark.parametrize("shape,n_tokens,wtype", _LAYER_CASES)
def test_fast_prefill_close_to_exact(tmp_models, big_models, shape, n_tokens, wtype):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    path = tmp_models(shape, wtype, 0, 1) if shape.startswith("tiny") else big_models(shape, wtype)
    x = np.random.default_rng(4).standard_normal((n_tokens, sh.n_embd), dtype=np.float32)
    exact = capi.Slice(path, 0, 1024)
    fast = capi.Slice(path, 0, 1024)
    fast.set_fast_prefill(True, 32)
    launches0 = fast.launch_count()
    ye, yf = exact.forward(x), fast.forward(x)
    assert fast.launch_count() > launches0
    assert np.isfinite(yf).all()
    rel_rms = float(np.sqrt(np.mean((yf - ye) ** 2)) / np.sqrt(np.mean(ye ** 2)))
    max_rel = float(np.abs(yf - ye).max() / np.abs(ye).max())
    assert rel_rms <= 1.5e-2, rel_rms
    assert max_rel <= 1e-1, max_rel
    assert not np.array_equal(yf, ye) or n_tokens < 32       # it really is a different code path
    # decode after a fast prefill runs in exact mode on a (slightly different) KV cache: stays close
    x1 = np.random.default_rng(5).standard_normal((1, sh.n_embd), dtype=np.float32)
    de, df = exact.forward(x1), fast.forward(x1)
    assert float(np.sqrt(np.mean((df - de) ** 2)) / np.sqrt(np.mean(de ** 2))) <= 1.5e-2
    exact.close()
    fast.close()


@pytest.mark.parametrize("wtype", [pytest.param(ggjt.T_Q4_0, id="2-2"), pytest.param(ggjt.T_Q8_0, id="2-8")])
def test_tensor_core_matmul_alone_is_tight(tmp_models, wtype):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128b"]
    path = tmp_models("tiny128b", wtype, 0, 0)
    x = np.random.default_rng(4).standard_normal((128, sh.n_embd), dtype=np.float32)
    a, b = capi.Slice(path, 0, 512), capi.Slice(path, 0, 512)
    b.set_fast_prefill(True, 32)
    a.forward(x), b.forward(x)
    n = 128 * 3 * sh.n_embd
    qa, qb = a.debug_read(0, n), b.debug_read(0, n)            # the qkv matmul output [128][3E] of the only layer
    rel = float(np.sqrt(np.mean((qa - qb) ** 2)) / np.sqrt(np.mean(qa ** 2)))
    assert 0 < rel <= 1e-3, rel
    a.close()
    b.close()


def test_fast_mode_falls_back_when_shapes_do_not_tile(tmp_models):
    """tiny128 has n_ff = 1376 (not a multiple of 64): the request is honoured with the exact kernels."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1)
    x = np.random.default_rng(4).standard_normal((64, sh.n_embd), dtype=np.float32)
    a, b = capi.Slice(path, 0, 512), capi.Slice(path, 0, 512)
    b.set_fast_prefill(True, 32)
    assert np.array_equal(a.forward(x), b.forward(x))
    a.close()
    b.close()


def test_fast_prefill_keeps_greedy_ids_where_the_margin_allows(tmp_path):
    """Fast mode is tolerance-level, so a greedy id may legitimately flip only where the exact logits' top-1 / top-2 margin is
    within the perturbation fast mode causes.  For every prompt position: either the fast-prefill argmax equals the exact one,
    or the exact margin is smaller than twice the largest logit deviation observed on that row."""
    from distributedllm_b200 import capi
    from distributedllm_b200.compute_node.slices import import_llm
    llm = import_llm()
    sh = ggjt.SHAPES["tiny128b"]
    full, sl, extra = str(tmp_path / "full.bin"), str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=11)
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    tokens = [1 + (i * 37) % (sh.n_vocab - 1) for i in range(96)]
    emb = np.array(llm.prepare_embeddings(extra, tokens), np.float32).reshape(len(tokens), sh.n_embd)
    exact, fast = capi.Slice(sl, 0, 512), capi.Slice(sl, 0, 512)
    fast.set_fast_prefill(True, 32)
    he, hf = exact.forward(emb), fast.forward(emb)
    le = np.array(llm.get_logits(extra, he.ravel().tolist(), True), np.float32).reshape(len(tokens), -1)
    lf = np.array(llm.get_logits(extra, hf.ravel().tolist(), True), np.float32).reshape(len(tokens), -1)
    same = flips_ok = 0
    for r in range(len(tokens)):
        top = np.argsort(le[r])[-2:]
        margin = float(le[r, top[1]] - le[r, top[0]])
        dev = float(np.abs(lf[r] - le[r]).max())
        if int(np.argmax(lf[r])) == int(top[1]):
            same += 1
        else:
            assert margin <= 2 * dev, "row %d: argmax flipped with margin %.4g > 2 x deviation %.4g" % (r, margin, dev)
            flips_ok += 1
    assert same >= len(tokens) * 3 // 4, (same, flips_ok)
    exact.close()
    fast.close()


# ------------------------------------------------------------------------------------ each matmul against float64
# (shape, wtype, token counts).  One layer each, so every matmul's input and output can be read back.
MATMUL_CASES = [
    ("7b", ggjt.T_Q4_0, (512, 300, 129, 33)),
    ("7b", ggjt.T_Q8_0, (512, 300)),
    ("13b", ggjt.T_Q4_0, (300,)),
    ("3b", ggjt.T_Q4_0, (300,)),                # w2: K = 8640, 67.5 quads of 128
    ("30b", ggjt.T_Q4_0, (300,)),               # w2: K = 17920
    ("30b", ggjt.T_Q8_0, (300,)),
    ("65b", ggjt.T_Q4_0, (300,)),               # w2: K = 22016
    ("65b", ggjt.T_Q8_0, (300,)),
    ("tiny128b", ggjt.T_Q4_0, (128, 300)),
    ("tiny128b", ggjt.T_Q8_0, (128, 300)),
]
_CASE_IDS = ["%s-%s-v2" % (c[0], ggjt.TYPE_NAME[c[1]]) for c in MATMUL_CASES]


def _n_sm() -> int:
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_plan(shape: str, wtype: int, n: int, n_sm: int) -> dict:
    """matmul -> (kernel instantiation, token tiles, last tile ragged), restating launch_fast_gemm: a matrix takes 256-token
    tiles when (128-row tiles) x (256-token tiles) fills the SMs or when N <= 128, else 128-token tiles."""
    sh = ggjt.SHAPES[shape]
    plan = {}
    for mat, rows in (("qkv", 3 * sh.n_embd), ("wo", sh.n_embd), ("w13", 2 * sh.n_ff), ("w2", sh.n_embd)):
        wide = (rows // 128) * -(-n // 256) >= n_sm or n <= 128
        nt = 256 if wide else 128
        kern = "v2-%s-nt%d" % (ggjt.TYPE_NAME[wtype], nt)
        plan[mat] = (kern, -(-n // nt), n % nt != 0)
    return plan


def test_cases_run_every_instantiation_over_several_ragged_token_tiles():
    n_sm = _n_sm()
    covered = set()
    for shape, wtype, ns in MATMUL_CASES:
        for n in ns:
            for kern, tiles, ragged in tile_plan(shape, wtype, n, n_sm).values():
                if tiles >= 2 and ragged:
                    covered.add(kern)
    want = {"v2-q4_0-nt128", "v2-q4_0-nt256", "v2-q8_0-nt128", "v2-q8_0-nt256"}
    assert want <= covered, (n_sm, sorted(want - covered))


@pytest.mark.parametrize("shape,wtype,ns", MATMUL_CASES, ids=_CASE_IDS)
def test_each_fast_matmul_is_within_the_float64_bound(tmp_models, big_models, shape, wtype, ns):
    """Every token and a row sample (every row of the first and last tile, 1/8 of the others, every 8-row position) of
    the four matmuls of one layer, against fast_ref's float64 sum of the same fp16 operands (fast_ref.check_layer).
    The fp16 activations the kernels read are proven bit-exact through the w2 input left in xh.  Also checks, in numpy
    only, that the bound is tight enough to see one lost 32-wide K block: zeroing one activation block of one token in
    the reference must put >= 99 % (95 % at 30B / 65B) of that token's outputs outside it."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    E, FF = sh.n_embd, sh.n_ff
    path = tmp_models(shape, wtype, 0, 0) if shape.startswith("tiny") else big_models(shape, wtype)
    t0 = time.time()
    w = fast_ref.LayerWeights(path, 0, E, FF)
    floor = LOST_BLOCK_LARGE if shape in ("30b", "65b") else LOST_BLOCK
    gpu = capi.Slice(path, 0, 1024)
    gpu.set_fast_prefill(True, 32)
    worst = {}
    try:
        for n in ns:
            gpu.clear_context()
            x = np.random.default_rng([n, E]).standard_normal((n, E), dtype=np.float32)
            y = gpu.forward(x)
            label = "%s %s N=%d" % (shape, ggjt.TYPE_NAME[wtype], n)
            errs, _ = fast_ref.check_layer(w, x, fast_ref.read_layer(gpu, n, E, FF), y, tau, floor, label)
            for mat, e in errs.items():
                worst[(n, mat)] = e
    finally:
        gpu.close()
    print("[fast-matmul] %s %s  largest %.3g (2^%.2f)  %.1f s" % (
        shape, ggjt.TYPE_NAME[wtype], max(worst.values()), np.log2(max(worst.values())), time.time() - t0))


# ------------------------------------------------------------------------------------ fast mode is prefill-only
def test_fast_mode_never_applies_to_a_batched_step(tmp_models):
    """A batched step (one token of each of 4 sessions) with fast mode on and min_tokens 2 equals stepping each session
    alone, bit for bit: the batch is 4 independent single-token steps, not a 4-token prefill."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128b"]
    path = tmp_models("tiny128b", ggjt.T_Q4_0, 0, 1, seed=23)
    batched, alone = capi.Slice(path, 0, 128, n_sessions=4), capi.Slice(path, 0, 128, n_sessions=4)
    for s in (batched, alone):
        s.set_fast_prefill(True, 2)
    rng = np.random.default_rng(6)
    for k, n in enumerate([40, 3, 17, 2]):                  # prompts: fast-mode prefills, identical on both slices
        x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
        assert (_bits(batched.session_forward(k, x)) == _bits(alone.session_forward(k, x))).all()
    for step in range(3):
        x = rng.standard_normal((4, sh.n_embd), dtype=np.float32)
        got = batched.batch_forward([0, 1, 2, 3], x)
        for k in range(4):
            assert (_bits(got[k]) == _bits(alone.session_forward(k, x[k:k + 1])[0])).all(), (step, k)
    batched.close()
    alone.close()


@pytest.mark.parametrize("graph", ["1", "0"], ids=["graphed", "ungraphed"])
def test_fast_mode_never_applies_to_a_single_token_step(tmp_models, monkeypatch, graph):
    """With min_tokens 1 every single-token step (the captured decode graph, or the launches without it) stays exact."""
    from distributedllm_b200 import capi
    from oracle import oracle
    monkeypatch.setenv("B200_GRAPH", graph)
    sh = ggjt.SHAPES["tiny128b"]
    path = tmp_models("tiny128b", ggjt.T_Q4_0, 0, 1, seed=24)
    gpu, cpu = capi.Slice(path, 0, 64), oracle.PortSlice(path, 64)
    gpu.set_fast_prefill(True, 1)
    rng = np.random.default_rng(7)
    for step in range(4):
        x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
        assert (_bits(gpu.forward(x)) == _bits(cpu.forward(x))).all(), step
    gpu.close()
    cpu.close()


def test_q8_0_exact_mode_one_7b_layer_bit_exact(big_models):
    """Exact-mode Q8_0 at LLaMA-7B shape (K = 4096 and 11008): a 40-token call, then 3 decode steps, against the C
    restatement bit for bit."""
    from distributedllm_b200 import capi
    from oracle import oracle
    sh = ggjt.SHAPES["7b"]
    path = big_models("7b", ggjt.T_Q8_0)
    gpu, cpu = capi.Slice(path, 0, 64), oracle.PortSlice(path, 64)
    rng = np.random.default_rng(8)
    for n in (40, 1, 1, 1):
        x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
        a, b = cpu.forward(x), gpu.forward(x)
        assert np.isfinite(b).all()
        bad = int((_bits(a) != _bits(b)).sum())
        assert bad == 0, "N=%d: %d of %d floats differ" % (n, bad, a.size)
    gpu.close()
    cpu.close()
