"""GPU: the multi-session passes -- mixed passes (b200_mixed_forward), batched steps (b200_batch_forward) and decode
rows (b200_session_forward_steps) -- at LLaMA-13B, 30B and 65B layer shapes, bit for bit against the reference's
digests in tests/golden/ref_digests_passes_large.json (written by tests/golden/gen_golden_passes_large.py, which also
defines the files, the operations and their inputs).  Every case runs on one slice with n_ctx 1024 and 12 sessions.

What each operation of the script reaches at 40, 52 and 64 heads of size 128:

  mixed pass of 12 prompts   the query-tiled attention kernel over the pass's tile table (every segment ends at or
                             before position 512), the fused single-token kernel for session 2's one-row segment;
                             148 columns: matmul column groups of 8 with a remainder of 4
  batched steps              the fused single-token kernel, one cluster row per column at per-session cache offsets;
                             12 columns = 8 + 4, 9 columns = 8 + 1; at 65B the w2 launch of Q8_0, Q4_1 and Q5_1 falls
                             back to 4 columns (eight do not fit in shared memory), so 12 columns run as 4 + 4 + 4
  32-row session_forward     a prompt chunk of one session (query-tiled up to position 512, per-query cluster kernel
                             past it)
  mixed pass past 512        A's 29 rows at 515..543 take the per-query cluster kernel with per-row lengths (col_T:
                             T = 544, a multiple of 32, so a wrong length moves the float / double split of the V sum),
                             session 0's 20 rows the query-tiled kernel, two single tokens the fused kernel, each alone
  decode rows                k_steps_table builds the pass on the device; the per-query cluster kernel with T = position
                             + 1 per row: B's 24 rows across 512, A's 16 rows at 544..559, session 2's 40 rows at 5..44
  final batched step         the fused kernel over 12 sessions at positions 6 to 560

Every multi-column F16 matmul at these shapes (K >= 5120) takes the one-column kernel; k-quant slices quantise each
column's activations to Q8_K.  The 65B Q4_0 and Q4_K_M cases are replayed under the runtime switches that select
between exact schedules (column groups, attention kernels, rings, PDL and graphs, one CTA per SM).

Long decode rows (tiny shapes, against the C restatement): passes of up to 1500 rows at n_ctx 4096, where the head-size-
128 cluster kernel runs in launches of 1024 queries, ending exactly at n_ctx.  End to end at 13B: greedy generation and
speculative decoding on the two-layer Q4_K_M file with the k-quant fixture's extra layers give the reference's ids.

Each weight file is written once per module and deleted after its last run: the 65B F16 layer is about 1.6 GB."""
import collections
import contextlib
import json
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle
from test_gpu_large_shapes import _bits, _checker, _checker_name

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLD)
import gen_golden_kquant_large as klarge  # noqa: E402
import gen_golden_passes_large as passes  # noqa: E402
import gen_golden_vocab as vocab  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(GOLD, "ref_digests_passes_large.json")))
PASSES = [n for n, c in CASES.items() if c["kind"] == "passes"]

SWITCHES = [{"B200_NC": "8"}, {"B200_NC": "4"}, {"B200_NC": "2"}, {"B200_TILED_ATTN": "0"}, {"B200_RING": "0"},
            {"B200_PDL": "0", "B200_GRAPH": "0"}, {"B200_CTA_PER_SM": "1"}]
SWEEPS = {"65b_q4_0": SWITCHES, "65b_q4_K_M": SWITCHES}
RUNS = [(n, env) for n in PASSES for env in [{}] + SWEEPS.get(n, [])]
USES = collections.Counter(n for n, _ in RUNS)


def _run_id(name, env):
    return name + "".join("-%s%s" % (k[5:].lower(), v) for k, v in env.items())


def _port(case):
    """The C restatement that covers the case's weight family."""
    if case["family"] in passes.KQUANT:
        from kq_port import KQPortSlice
        return KQPortSlice
    if case["family"] in ("q5_0", "q5_1"):
        from q5_port import Q5PortSlice
        return Q5PortSlice
    return oracle.PortSlice


@pytest.fixture(scope="module")
def case_file(tmp_path_factory):
    """Context manager name -> path of the case's weight file; a file is deleted once its last run in RUNS is done."""
    root = tmp_path_factory.mktemp("passes_large")
    files, left = {}, collections.Counter(USES)

    @contextlib.contextmanager
    def use(name):
        if name not in files:
            files[name] = str(root / ("%s.bin" % name))
            passes.write_case_file(files[name], CASES[name])
            assert vocab.file_sha256(files[name]) == CASES[name]["file_sha256"], \
                "the writer changed: regenerate the fixture"
        try:
            yield files[name]
        finally:
            left[name] -= 1
            if left[name] == 0:
                os.remove(files.pop(name))

    yield use
    for p in files.values():
        os.remove(p)


def _replay_passes(path, case):
    from distributedllm_b200 import capi
    xs, ops = passes.inputs(case), case["ops"]
    gpu = capi.Slice(path, 0, case["n_ctx"], n_sessions=case["n_sessions"])
    got = []
    try:
        for op, x in zip(ops, xs):
            if op["op"] == "mixed":
                y = gpu.mixed_forward(op["sessions"], op["counts"], x)
            elif op["op"] == "batch":
                y = gpu.batch_forward(op["sessions"], x)
            elif op["op"] == "session":
                y = gpu.session_forward(op["session"], x)
            else:
                y = gpu.forward_steps(op["session"], x)
            got.append(passes.split(op, y))
        n_past = [gpu.session_n_past(s) for s in range(case["n_sessions"])]
    finally:
        gpu.close()
    pos, _ = passes.positions(case)
    wrong = [(i, k) for i, op in enumerate(ops) for k in range(len(got[i]))
             if passes.digest(got[i][k]) != case["digests"][i][k]]
    assert all(np.isfinite(y).all() for g in got for y in g)
    if wrong:
        port = _port(case)
        cpu = _checker(path, case["n_ctx"], port)
        try:
            want = passes.replay(cpu, case, xs, sorted({passes.op_sessions(ops[i])[k][0] for i, k in wrong}))
        finally:
            cpu.close()
        report = []
        for i, k in wrong:
            s, n = passes.op_sessions(ops[i])[k]
            report.append("operation %d (%s), session %d at position %d, %d rows: %d of %d floats differ" % (
                i, ops[i]["op"], s, pos[i][k], n, int((_bits(got[i][k]) != _bits(want[(i, s)])).sum()), got[i][k].size))
        pytest.fail("%d outputs differ from the reference (recomputed with %s): %s" % (
            len(wrong), _checker_name(port), "; ".join(report)))
    assert n_past == case["n_past"]


@pytest.mark.parametrize("name,env", [pytest.param(n, e, id=_run_id(n, e)) for n, e in RUNS])
def test_passes_match_reference(case_file, monkeypatch, name, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    with case_file(name) as path:
        _replay_passes(path, CASES[name])


# ---------------------------------------------------------------- long decode rows

LONG_N_CTX = 4096
LONG_ROWS = [17, 100, 1024, 1025, 1500]      # one, two and three 1024-query launches of the cluster kernel


@pytest.mark.parametrize("shape", ["tiny128", "tiny"], ids=["d128", "d64"])
def test_long_decode_rows_equal_single_steps_up_to_n_ctx(tmp_models, shape):
    """Decode rows of session 1 from position 430 (session 0 holds another context) to exactly n_ctx 4096, each pass
    against one-row calls of the C restatement; then one more row is refused and the position stays.  One layer: its
    K / V rows depend on the inputs alone, so every pass is checked on a correct cache even after one differs."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    path = tmp_models(shape, ggjt.T_Q4_0, 0, 0, seed=23)
    rng = np.random.default_rng(9)
    gpu, ref = capi.Slice(path, 0, LONG_N_CTX, n_sessions=2), oracle.PortSlice(path, LONG_N_CTX)
    try:
        gpu.session_forward(0, rng.standard_normal((37, sh.n_embd), dtype=np.float32))
        x = rng.standard_normal((LONG_N_CTX - sum(LONG_ROWS), sh.n_embd), dtype=np.float32)
        assert (_bits(gpu.session_forward(1, x)) == _bits(ref.forward(x))).all()
        report = []
        for n in LONG_ROWS:
            pos = gpu.session_n_past(1)
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            got = gpu.forward_steps(1, x)
            want = np.concatenate([ref.forward(x[j:j + 1]) for j in range(n)])
            bad = _bits(got) != _bits(want)
            if bad.any():
                report.append("%d decode rows at position %d: %d of %d floats differ, first in row %d" % (
                    n, pos, int(bad.sum()), got.size, int(np.argmax(bad.any(axis=1)))))
            assert gpu.session_n_past(1) == pos + n
        assert not report, "; ".join(report)
        assert gpu.session_n_past(1) == LONG_N_CTX
        with pytest.raises(capi.B200Error) as ei:
            gpu.forward_steps(1, np.ones((1, sh.n_embd), np.float32))
        assert ei.value.code == 5
        assert gpu.session_n_past(1) == LONG_N_CTX and gpu.session_n_past(0) == 37
    finally:
        gpu.close()
        ref.close()


# ---------------------------------------------------------------- end to end at 13B

def test_13b_greedy_and_speculative_give_the_reference_ids(tmp_path):
    """generate_greedy over 3 sessions on the 13B Q4_K_M two-layer file with the k-quant fixture's 13B extra layers:
    the reference's own greedy ids.  Then generate_speculative, one session at a time, with n_draft 4 and 15 and the
    file's first layer alone as the draft: the same ids."""
    from distributedllm_b200 import capi
    case = CASES["13b_generate"]
    sh = ggjt.SHAPES[case["shape"]]
    path, dpath, epath = (str(tmp_path / n) for n in ("t.bin", "d.bin", "extra.bin"))
    klarge.write_layers(path, case)
    klarge.write_layers(dpath, dict(case, layers=[case["layers"][0]] * 2))
    ggjt.write_kquant_extra(epath, sh, case["mix"], seed=case["seed"])
    assert (vocab.file_sha256(path), vocab.file_sha256(epath)) == (case["file_sha256"], case["extra_sha256"]), \
        "the writer changed: regenerate the fixture"
    prompts, n_steps = case["prompts"], case["n_steps"]
    tgt = capi.Slice(path, 0, 128, n_sessions=len(prompts))
    drf = capi.Slice(dpath, 0, 128)
    ext, dext = capi.Extra(epath, 0), capi.Extra(epath, 0)
    try:
        ids = capi.generate_greedy([tgt], ext, list(range(len(prompts))), prompts, n_steps)
        assert ids.tolist() == case["ids"]
        assert [tgt.session_n_past(k) for k in range(len(prompts))] == [len(p) + n_steps - 1 for p in prompts]
        for n_draft in (4, 15):
            for k, p in enumerate(prompts):
                tgt.session_clear(k)
                drf.session_clear(0)
                got, st = capi.generate_speculative([tgt], ext, k, [drf], dext, 0, p, n_steps, n_draft)
                assert got.tolist() == [r[k] for r in case["ids"]], (n_draft, k)
                assert st["drafted"] == st["passes"] * n_draft
                assert tgt.session_n_past(k) == drf.session_n_past(0) == len(p) + n_steps - 1
    finally:
        for h in (ext, dext, tgt, drf):
            h.close()
