"""GPU: one layer of LLaMA-30B (n_embd 6656, 52 heads, n_ff 17920) and LLaMA-65B (8192, 64 heads, 22016) for every weight
type, bit for bit against the reference's hidden states, kept as digests in tests/golden/ref_digests_large.json (written
by tests/golden/gen_golden_large.py, which also defines the inputs).

These shapes reach host-side choices the 3B / 7B / 13B tests never make: at 65B the eight-column w2 launch of Q8_0,
Q4_1 and Q5_1 slices does not fit in shared memory (the launcher takes four columns instead), wo has 256 tiles (the most
the B200_NQ epilogue accepts), attention runs 208 / 256 four-CTA clusters, and every multi-token F16 matmul takes the
one-column kernel (the activations of K >= 6656 do not fit the multi-column one).  The 65B Q4_0 schedule is replayed
under every runtime switch that selects between exact schedules; each must reproduce the reference's digests.

Each weight file is written once per module (tmp_path_factory) and deleted after its last case: the 65B F16 layer is
about 1.6 GB."""
import collections
import contextlib
import json
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLD)
import gen_golden_large as large  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(GOLD, "ref_digests_large.json")))
HAVE_REF = oracle.have_ref()

# runtime switches replayed on a case's file right after its default run (every one selects a bit-identical schedule)
SWEEPS = {
    "65b_q4_0": [{"B200_RING": "0"}, {"B200_NQ": "1"}, {"B200_PDL": "0", "B200_GRAPH": "0"}, {"B200_TILED_ATTN": "0"},
                 {"B200_NC": "8"}, {"B200_NC": "4"}, {"B200_NC": "2"}],
    "65b_q8_0": [{"B200_NC": "8"}],          # a forced group is an upper bound: w2 still takes four columns
}


def _file_key(case):
    return case["shape"], case["wtype"], case["seed"]


def _runs():
    """(case, environment) in file order: every run on one weight file next to the others."""
    runs, names = [], list(CASES)
    for i, name in enumerate(names):
        runs.append((name, {}))
        last = i + 1 == len(names) or _file_key(CASES[names[i + 1]]) != _file_key(CASES[name])
        if last:
            for n in names[:i + 1]:
                if _file_key(CASES[n]) == _file_key(CASES[name]):
                    runs += [(n, env) for env in SWEEPS.get(n, [])]
    return runs


RUNS = _runs()
USES = collections.Counter(_file_key(CASES[name]) for name, _ in RUNS)


def _run_id(name, env):
    return name + "".join("-%s%s" % (k[5:].lower(), v) for k, v in env.items())


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def layer_file(tmp_path_factory):
    """Context manager case -> path of its one-layer file; a file is deleted once its last run in RUNS is done."""
    root = tmp_path_factory.mktemp("large")
    files, left = {}, collections.Counter(USES)

    @contextlib.contextmanager
    def use(case):
        key = _file_key(case)
        if key not in files:
            files[key] = str(root / ("%s_%s_s%d.bin" % (key[0], ggjt.TYPE_NAME[key[1]], key[2])))
            large.write_slice(files[key], *key)
        try:
            yield files[key]
        finally:
            left[key] -= 1
            if left[key] == 0:
                os.remove(files.pop(key))

    yield use
    for p in files.values():
        os.remove(p)


def _checker(path, n_ctx, port=oracle.PortSlice):
    """The CPU computation a mismatch is counted against: the compiled reference where it was built, else the C port
    `port` (a class with PortSlice's forward / clear_context / close)."""
    return oracle.RefSlice(path, min(16, os.cpu_count() or 4), n_ctx) if HAVE_REF else port(path, n_ctx)


def _checker_name(port=oracle.PortSlice):
    return "RefSlice" if HAVE_REF else port.__name__


def _replay_schedule(path, case, port=oracle.PortSlice):
    from distributedllm_b200 import capi
    xs = large.case_inputs(case)
    gpu = capi.Slice(path, 0, case["n_ctx"])
    try:
        ys = [gpu.forward(x) for x in xs]
    finally:
        gpu.close()
    wrong = [i for i, y in enumerate(ys) if large.digest(y) != case["digests"][i]]
    for i, y in enumerate(ys):
        assert np.isfinite(y).all(), "call %d (N=%d): non-finite output" % (i, len(xs[i]))
    if wrong:
        cpu = _checker(path, case["n_ctx"], port)
        try:
            want = [cpu.forward(x) for x in xs[:wrong[-1] + 1]]
        finally:
            cpu.close()
        report = ["call %d (N=%d): %d of %d floats differ" % (i, len(xs[i]), int((_bits(ys[i]) != _bits(want[i])).sum()),
                                                              ys[i].size) for i in wrong]
        pytest.fail("%d of %d calls differ from the reference (recomputed with %s): %s" % (
            len(wrong), len(xs), _checker_name(port), "; ".join(report)))


def _replay_batch(path, case, port=oracle.PortSlice):
    from distributedllm_b200 import capi
    prompts, steps = large.batch_inputs(case)
    sessions = case["sessions"]
    gpu = capi.Slice(path, 0, case["n_ctx"], n_sessions=len(sessions))
    try:
        got_p = [gpu.session_forward(s, prompts[b]) for b, s in enumerate(sessions)]
        got_s = [gpu.batch_forward(sessions, x) for x in steps]
    finally:
        gpu.close()
    wrong = [("prompt", b) for b in range(len(sessions)) if large.digest(got_p[b]) != case["prompt_digests"][b]]
    wrong += [("step %d" % i, b) for i in range(len(steps)) for b in range(len(sessions))
              if large.digest(got_s[i][b]) != case["step_digests"][i][b]]
    assert all(np.isfinite(y).all() for y in got_p + got_s)
    if wrong:
        cpu = _checker(path, case["n_ctx"], port)
        want_p, want_s = [], [[None] * len(sessions) for _ in steps]
        try:
            for b in range(len(sessions)):
                cpu.clear_context()
                want_p.append(cpu.forward(prompts[b]))
                for i, x in enumerate(steps):
                    want_s[i][b] = cpu.forward(x[b:b + 1])[0]
        finally:
            cpu.close()
        report = []
        for what, b in wrong:
            g, w = (got_p[b], want_p[b]) if what == "prompt" else (got_s[int(what[5:])][b], want_s[int(what[5:])][b])
            report.append("%s, column %d (session %d): %d of %d floats differ" % (
                what, b, sessions[b], int((_bits(g) != _bits(w)).sum()), g.size))
        pytest.fail("%d outputs differ from the reference (recomputed with %s): %s" % (
            len(wrong), _checker_name(port), "; ".join(report)))


@pytest.mark.parametrize("name,env", [pytest.param(n, e, id=_run_id(n, e)) for n, e in RUNS])
def test_large_shape_layer_matches_reference(layer_file, monkeypatch, name, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    case = CASES[name]
    with layer_file(case) as path:
        if case["kind"] == "batch":
            _replay_batch(path, case)
        else:
            _replay_schedule(path, case)
