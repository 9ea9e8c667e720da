"""GPU: attention over the whole context a slice accepts, bit for bit.  n_ctx is a load parameter here (the reference is
fixed at 512), so every attention path past position 512 and every prompt call over 1024 rows runs in production:

  * prompt calls of more than 1024 rows: the per-query cluster kernel runs in launches of 1024 queries (n0 > 0);
  * single-token steps past 512: each CTA of the cluster kernel mixes its 128 staged rows with rows read from global
    memory, and the V tail comes from its own staged block;
  * the generic kernel (head sizes 64 and 100) with score rows of thousands of positions;
  * the largest n_ctx the loader accepts per attention family, filled to its last position;
  * a k-quant slice, mixed passes, batched steps, scoring and a stream at distant positions of different sessions.

Hidden states are compared as uint32 views with the C restatement (oracle.PortSlice / tests/kq_port.py), which has no
position limit.  One-layer LLaMA-7B and LLaMA-13B slices at n_ctx 2048 are compared with the compiled reference's
digests (tests/golden/ref_digests_long.json, written by tests/golden/gen_golden_long.py)."""
import json
import os
import re
import sys

import numpy as np
import pytest

import score_ref
from distributedllm_b200 import ggjt
from test_gpu_generate import _model
from test_gpu_mixed_batch import _decode_rounds, _mixed_pass, _port

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import gen_golden_long as long_ref  # noqa: E402
LONG = json.load(open(os.path.join(HERE, "golden", "ref_digests_long.json")))

# One head of each attention family at the narrowest n_embd the loader accepts: the restatement's attention costs
# O(T^2 * n_embd), which keeps a context of tens of thousands of positions affordable.
ONE_HEAD = {128: ggjt.ModelShape(512, 128, 32, 1, 1), 64: ggjt.ModelShape(512, 64, 32, 1, 1)}

# Three contexts at n_ctx 4096, call sizes in rows.  Positions in the comments are those of the call's first row; a
# step at position p attends over T = p + 1 rows.
N_CTX = 4096
CONTEXT_1 = ([300, 211]             # query-tiled prompt calls up to position 511
             + [1, 1, 1]            # steps at 511 (T % 32 = 0), 512 (T % 32 = 1), 513
             + [28, 1, 1]           # cluster-kernel prompt call; steps at 542 (T % 32 = 31) and 543
             + [479, 1, 1]          # to 1023; steps at 1023 and 1024
             + [1024, 1025, 1, 1])  # one and two query launches; steps at 3074, 3075
CONTEXT_2 = ([300, 212]             # a prompt call ending exactly at 512, the last the tiled kernel takes
             + [2049, 1]            # three query launches; step at 2561
             + [1502] + [1] * 32)   # to 4064; steps at 4064..4095: T % 32 = 1 ... 31, 0, and the last position
CONTEXT_3 = [400, 113, 1]           # a prompt call ending at 513, the first the cluster kernel takes; step at 513
assert sum(CONTEXT_2) == N_CTX


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _replay(gpu, ref, schedule, rng, n_embd, where):
    """Each call of `schedule` on both sides (0: clear both contexts); every row must be the same bits."""
    for i, n in enumerate(schedule):
        if n == 0:
            gpu.clear_context()
            ref.clear_context()
            continue
        pos = gpu.n_past
        x = rng.standard_normal((n, n_embd), dtype=np.float32)
        g, r = gpu.forward(x), ref.forward(x)
        bad = int((_bits(g) != _bits(r)).sum())
        assert bad == 0, "%s: call %d (%d rows at position %d): %d of %d floats differ" % (where, i, n, pos, bad, g.size)
        assert gpu.n_past == pos + n


def _refuse_overflow(gpu, n_embd):
    """The context is full: one more row is refused and the position stays."""
    from distributedllm_b200 import capi
    full = gpu.n_past
    with pytest.raises(capi.B200Error):
        gpu.forward(np.ones((1, n_embd), np.float32))
    assert gpu.n_past == full


@pytest.mark.parametrize("shape,wtype,layers", [("tiny128", ggjt.T_Q4_0, 2), ("tiny128", ggjt.T_Q8_0, 1),
                                                ("tiny", ggjt.T_Q4_0, 1), ("tiny3b", ggjt.T_Q4_0, 1)],
                         ids=["d128-q4_0", "d128-q8_0", "d64-q4_0", "d100-q4_0"])
def test_every_boundary_up_to_n_ctx_4096(tmp_models, shape, wtype, layers):
    """Head size 128 (tiled and cluster kernels; Q8_0 quantises the attention output for wo in the kernel) and the
    generic kernel (head sizes 64 and 100) across 512, 1024, the query launches of long calls and the last position."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    path = tmp_models(shape, wtype, 0, layers - 1, seed=31)
    gpu, ref = capi.Slice(path, 0, N_CTX), _port(path, wtype, N_CTX)
    try:
        _replay(gpu, ref, CONTEXT_1, np.random.default_rng(1), sh.n_embd, "context 1")
        _replay(gpu, ref, [0] + CONTEXT_2, np.random.default_rng(2), sh.n_embd, "context 2")
        _refuse_overflow(gpu, sh.n_embd)
        _replay(gpu, ref, [0] + CONTEXT_3, np.random.default_rng(3), sh.n_embd, "context 3")
    finally:
        gpu.close()
        ref.close()


def _attn_smem_need(n_ctx, d_head):
    """(bytes, limit) of the attention kernels' worst-case dynamic shared memory at n_ctx: f32 scores and f16
    probabilities of every position, then for head size 128 the cluster kernel's 128 staged K / V rows of 272 B, the V
    tail, the reduction and the exp table's 64 KB (opt-in limit 200 KB); for other head sizes k_attention's partial sums
    (226 KB)."""
    sc = ((n_ctx + 3) & ~3) * 4 + ((n_ctx + 7) & ~7) * 2
    if d_head == 128:
        return ((sc + 15) & ~15) + 2 * 128 * 272 + 32 * 64 + 64 + 65536, 200 * 1024
    return sc + 4 * d_head * 32 + 64, 226 * 1024


@pytest.mark.parametrize("d_head", [128, 64])
def test_the_largest_context_the_loader_accepts(tmp_path, d_head):
    """The n_ctx the load error names is loaded, filled to its last position in long prompt calls and single steps,
    and checked call by call; the first n_ctx whose attention does not fit is refused at load, the one below it is not."""
    from distributedllm_b200 import capi
    from oracle import oracle
    sh = ONE_HEAD[d_head]
    path = str(tmp_path / "one_head.bin")
    ggjt.write_synth_slice(path, sh, 0, 0, ggjt.T_Q4_0, seed=32)
    with pytest.raises(capi.B200Error) as ei:
        capi.Slice(path, 0, 1 << 17)
    assert ei.value.code == 1
    m = re.search(r"largest supported n_ctx for head size %d is (\d+)" % d_head, str(ei.value))
    assert m, str(ei.value)
    named = int(m.group(1))
    need, limit = _attn_smem_need(named, d_head)
    assert need <= limit and named > (11000 if d_head == 128 else 37000)
    first_bad = named
    while _attn_smem_need(first_bad, d_head)[0] <= limit:
        first_bad += 1
    with pytest.raises(capi.B200Error) as ei:
        capi.Slice(path, 0, first_bad)
    assert ei.value.code == 1 and "n_ctx %d" % first_bad in str(ei.value)
    capi.Slice(path, 0, first_bad - 1).close()

    chunk = 3000 if d_head == 128 else 6000
    calls = [512] + [chunk] * ((named - 512 - 3) // chunk)
    calls += [named - 3 - sum(calls), 1, 1, 1]
    gpu, ref = capi.Slice(path, 0, named), oracle.PortSlice(path, named)
    try:
        _replay(gpu, ref, calls, np.random.default_rng(d_head), sh.n_embd, "n_ctx %d" % named)
        assert gpu.n_past == named
        _refuse_overflow(gpu, sh.n_embd)
    finally:
        gpu.close()
        ref.close()


def test_kquant_slice_past_1024(tmp_path):
    """A Q4_K_M layer (wv and w2 in Q6_K) feeds wo through k_quant_q8k, not through the attention epilogue: a call of
    1100 rows, steps past 1024, and the last position of n_ctx 2048."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tinyk128"]
    path = str(tmp_path / "kq.bin")
    ggjt.write_kquant_slice(path, sh, 0, 0, "q4_K_M", seed=33)
    gpu, ref = capi.Slice(path, 0, 2048), _port(path, ggjt.T_Q4_K, 2048)
    try:
        _replay(gpu, ref, [700, 1100, 1, 1, 203] + [1] * 43, np.random.default_rng(4), sh.n_embd, "q4_K_M")
        assert gpu.n_past == 2048
        _refuse_overflow(gpu, sh.n_embd)
    finally:
        gpu.close()
        ref.close()


def test_sessions_at_distant_positions(tmp_models):
    """One mixed pass at n_ctx 4096: a 1500-row segment starting at 600 (two query launches), query-tiled segments,
    single tokens at positions 5, 700 and 3999; then a batched step over sessions at 4000, 6, 701 and 2100, and graph
    replays.  Each session against its own restatement and a twin handle's per-session calls."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=34)
    S = 6
    gpu, twin = capi.Slice(path, 0, N_CTX, n_sessions=S), capi.Slice(path, 0, N_CTX, n_sessions=S)
    refs = {}
    rng = np.random.default_rng(5)
    try:
        for k, n in zip(range(S), (600, 100, 5, 700, 3999, 0)):
            refs[k] = _port(path, ggjt.T_Q4_0, N_CTX)
            if n:
                x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
                want = refs[k].forward(x)
                assert (_bits(gpu.session_forward(k, x)) == _bits(want)).all()
                assert (_bits(twin.session_forward(k, x)) == _bits(want)).all()
        _mixed_pass(gpu, twin, refs, [2, 0, 3, 1, 4, 5], [1, 1500, 1, 50, 1, 20], rng, sh.n_embd, "mixed")
        assert [gpu.session_n_past(k) for k in range(S)] == [2100, 150, 6, 701, 4000, 20]
        ids = [4, 2, 3, 0]
        x = rng.standard_normal((len(ids), sh.n_embd), dtype=np.float32)
        got = gpu.batch_forward(ids, x)
        for j, k in enumerate(ids):
            assert (_bits(got[j]) == _bits(refs[k].forward(x[j:j + 1])[0])).all(), ("batched step", k)
            twin.session_forward(k, x[j:j + 1])
        _decode_rounds(gpu, twin, refs, [5, 0, 4, 1], rng, sh.n_embd, 1, "replays")
        assert [gpu.session_n_past(k) for k in range(S)] == [twin.session_n_past(k) for k in range(S)]
    finally:
        for r in refs.values():
            r.close()
        gpu.close()
        twin.close()


def test_score_of_a_text_that_fills_n_ctx(tmp_path):
    """capi.score of a 2047-token text at n_ctx 2048: one session, one segment of 2046 rows (two query launches), against
    the host path (forward, all logits, the client's float64 softmax)."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 2048) for p in paths]
    twin = [capi.Slice(p, 0, 2048) for p in paths]
    extra = capi.Extra(extra_path, 0)
    tokens = np.random.default_rng(6).integers(0, sh.n_vocab, 2047).tolist()
    got = capi.score(gpu, extra, [0], [tokens])[0]
    x = extra.embed(tokens[:-1])
    for s in twin:
        x = s.session_forward(0, x)
    want = score_ref.nll_rows(extra.logits(x), tokens[1:])
    assert len(got) == 2046 and np.isfinite(want).all()
    ok = score_ref.within(got, want)
    assert ok.all(), [(j, got[j], want[j]) for j in np.flatnonzero(~ok)[:8]]
    assert [s.n_past for s in gpu] == [2046, 2046]
    extra.close()
    for s in gpu + twin:
        s.close()


def test_stream_with_a_prompt_over_1024_ids(tmp_path):
    """A one-session stream whose 1100-id prompt is one segment of a mixed pass equals generate_greedy on a twin."""
    from distributedllm_b200 import capi
    paths, extra_path, sh = _model(tmp_path, "q4_0")
    gpu = [capi.Slice(p, 0, 1280) for p in paths]
    twin = [capi.Slice(p, 0, 1280) for p in paths]
    extra = capi.Extra(extra_path, 0)
    prompt = np.random.default_rng(7).integers(0, sh.n_vocab, 1100).tolist()
    want = capi.generate_greedy(twin, extra, [0], [prompt], 24)[:, 0].tolist()
    with capi.Stream(gpu, extra) as st:
        st.add(0, prompt, 24)
        got = [t for _, t in st]
    assert got == want and len(set(want)) > 3
    assert [s.n_past for s in gpu] == [s.n_past for s in twin] == [1100 + 23] * 2
    extra.close()
    for s in gpu + twin:
        s.close()


def replay_long_case(tmp_path, name):
    """Replay case `name` of ref_digests_long.json on a fresh slice: -> [(call, first row's position)] that differ."""
    from distributedllm_b200 import capi
    case = LONG[name]
    path = str(tmp_path / ("%s.bin" % name))
    long_ref.write_slice(path, case["shape"], case["wtype"], case["seed"])
    gpu = capi.Slice(path, 0, case["n_ctx"])
    bad = []
    try:
        for i, (x, want) in enumerate(zip(long_ref.case_inputs(case), case["digests"])):
            pos = gpu.n_past
            if long_ref.digest(gpu.forward(x)) != want:
                bad.append((i, pos))
        assert gpu.n_past == case["n_ctx"]
    finally:
        gpu.close()
    os.remove(path)
    return bad


@pytest.mark.parametrize("name", ["7b_q4_0", "13b_q4_0"])
def test_full_size_layers_against_the_reference_at_n_ctx_2048(tmp_path, name):
    """One LLaMA-7B / LLaMA-13B Q4_0 layer prefilled in the reference's chunks to 2000, then stepped to 2047."""
    bad = replay_long_case(tmp_path, name)
    assert not bad, "%s: calls (index, position) %s differ from the reference" % (name, bad)
