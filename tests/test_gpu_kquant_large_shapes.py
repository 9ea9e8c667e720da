"""GPU: Q4_K_S, Q4_K_M and Q6_K slices at LLaMA-13B (n_embd 5120, n_ff 13824), 30B (6656, 17920) and 65B (8192, 22016)
shapes, bit for bit against the reference's digests in tests/golden/ref_digests_kquant_large.json (written by
tests/golden/gen_golden_kquant_large.py, which also defines the files and inputs).

These shapes reach what the tinyk / 7B k-quant tests do not: w2 has 54 / 70 / 86 super-blocks per row, so a tile is an
odd number of ring stages (27 / 35 / 43), and launches have more tiles than co-resident CTAs: w1|w3 from 5 columns on
at every shape (65B already at one), 30B / 65B qkv from 5, w2 from 17 (13B) and 9 (30B) or 5 (65B) columns on, and
every 32000-row lm_head.  A CTA's second tile then starts mid-ring, on the other mbarrier phase.  The 65B Q6_K w2
launch at 8 columns (201 296 B of activations + two 13 440-B ring stages) is the one closest to the shared-memory limit in
the runtime.  Q4_K_M files hold two adjacent layers, the first all Q4_K and the second with Q6_K
wv / w2 at the model's real layer count, so one slice runs both qkv packings.

The 65B Q4_K_M schedule is replayed under every runtime switch that selects between exact schedules, and must reproduce
the same digests: among them B200_CTA_PER_SM=1 (every matmul of the case walks two or more tiles per CTA), B200_NS=3 (the
ring wraps at a different stage of every tile), and B200_NQ=1 / B200_FAST_PREFILL=1, which k-quant slices ignore.  The
extra-layers files (Q4_K tok_embeddings, Q6_K output.weight of 32000 ids) go through capi.Extra: embedding rows, every
row's logits and the device argmax.

Each weight file is written once per module and deleted after its last run: the largest, the two-layer 65B Q4_K_M file,
is about 1 GB."""
import collections
import contextlib
import json
import os
import sys

import numpy as np
import pytest

from oracle import oracle
from test_gpu_large_shapes import _bits, _replay_batch, _replay_schedule

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLD)
import gen_golden_kquant_large as klarge  # noqa: E402
import gen_golden_vocab as vocab  # noqa: E402

pytestmark = pytest.mark.gpu
CASES = json.load(open(os.path.join(GOLD, "ref_digests_kquant_large.json")))
HAVE_REF = oracle.have_ref()

# runtime switches replayed on a case's file right after its default run (every one selects a bit-identical schedule)
SWEEPS = {
    "65b_q4_K_M": [{"B200_RING": "0"}, {"B200_PDL": "0", "B200_GRAPH": "0"}, {"B200_TILED_ATTN": "0"},
                   {"B200_NC": "8"}, {"B200_NC": "4"}, {"B200_NC": "2"}, {"B200_CTA_PER_SM": "1"}, {"B200_NS": "3"},
                   {"B200_NQ": "1"}, {"B200_FAST_PREFILL": "1"}],
}


def _runs():
    """(case, environment) in file order: every run on one weight file next to the others."""
    runs, names = [], list(CASES)
    key = lambda n: klarge.file_key(CASES[n])  # noqa: E731
    for i, name in enumerate(names):
        runs.append((name, {}))
        if i + 1 == len(names) or key(names[i + 1]) != key(name):
            runs += [(n, env) for n in names[:i + 1] if key(n) == key(name) for env in SWEEPS.get(n, [])]
    return runs


RUNS = _runs()
USES = collections.Counter(klarge.file_key(CASES[name]) for name, _ in RUNS)


def _run_id(name, env):
    return name + "".join("-%s%s" % (k[5:].lower(), v) for k, v in env.items())


@pytest.fixture(scope="module")
def case_file(tmp_path_factory):
    """Context manager case -> path of its weight file; a file is deleted once its last run in RUNS is done."""
    root = tmp_path_factory.mktemp("kquant_large")
    files, left = {}, collections.Counter(USES)

    @contextlib.contextmanager
    def use(name):
        case = CASES[name]
        key = klarge.file_key(case)
        if key not in files:
            files[key] = str(root / ("%s.bin" % name))
            klarge.write_case_file(files[key], case)
            assert vocab.file_sha256(files[key]) == case["file_sha256"], "the writer changed: regenerate the fixture"
        try:
            yield files[key]
        finally:
            left[key] -= 1
            if left[key] == 0:
                os.remove(files.pop(key))

    yield use
    for p in files.values():
        os.remove(p)


def _replay_extra(path, case):
    from distributedllm_b200 import capi
    from kq_port import KQPortExtra
    extra = capi.Extra(path, 0)
    try:
        assert (extra.n_vocab, extra.n_embd) == (case["n_vocab"], case["n_embd"])
        xs = [vocab.hidden(case, n) for n in case["rows"]]
        ys = [extra.logits(x) for x in xs]
        ids = [extra.next_token(x) for x in xs]
        emb = extra.embed(case["embed_ids"])
    finally:
        extra.close()
    for y in ys + [emb]:
        assert np.isfinite(y).all()
    wrong = [(i, j) for i, y in enumerate(ys) for j, r in enumerate(y) if klarge.digest(r) != case["logits"][i][j]]
    wrong_emb = [j for j, r in enumerate(emb) if klarge.digest(r) != case["embed"][j]]
    if wrong or wrong_emb:
        port = KQPortExtra(path)
        want = {i: oracle.ref_logits(path, xs[i], case["n_vocab"], True) if HAVE_REF else port.logits(xs[i])
                for i in sorted({i for i, _ in wrong})}
        want_emb = oracle.ref_embed(path, case["embed_ids"], case["n_embd"]) if HAVE_REF else port.embed(case["embed_ids"])
        report = ["call %d (N=%d), row %d: %d of %d logits differ" % (
            i, len(xs[i]), j, int((_bits(ys[i][j]) != _bits(want[i][j])).sum()), case["n_vocab"]) for i, j in wrong]
        report += ["embedding of id %d: %d of %d floats differ" % (
            case["embed_ids"][j], int((_bits(emb[j]) != _bits(want_emb[j])).sum()), case["n_embd"]) for j in wrong_emb]
        pytest.fail("%d outputs differ from the reference (recomputed with %s): %s" % (
            len(report), "the reference" if HAVE_REF else "KQPortExtra", "; ".join(report)))
    assert ids == [a[-1] for a in case["argmax"]]


@pytest.mark.parametrize("name,env", [pytest.param(n, e, id=_run_id(n, e)) for n, e in RUNS])
def test_kquant_large_shape_matches_reference(case_file, monkeypatch, name, env):
    from kq_port import KQPortSlice
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    case = CASES[name]
    with case_file(name) as path:
        if case["kind"] == "extra":
            _replay_extra(path, case)
        elif case["kind"] == "batch":
            _replay_batch(path, case, KQPortSlice)
        else:
            _replay_schedule(path, case, KQPortSlice)
