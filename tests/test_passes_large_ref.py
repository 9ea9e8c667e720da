"""CPU: the multi-session pass fixture at LLaMA-13B, 30B and 65B shapes (tests/golden/ref_digests_passes_large.json,
written by tests/golden/gen_golden_passes_large.py) -- what its operations cover, and the C restatements
(oracle.PortSlice, tests/q5_port.py, tests/kq_port.py) reproducing the 13B digests and greedy ids.  The restatements
replay each session alone, so a match shows that the digests encode per-session semantics (a segment is a call of its
rows, a batched-step column or a decode row a one-row call), which is what tests/test_gpu_passes_large_shapes.py holds
the GPU passes to."""
import json
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import gen_golden_kquant_large as klarge  # noqa: E402
import gen_golden_passes_large as passes  # noqa: E402
import gen_golden_vocab as vocab  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "ref_digests_passes_large.json")))
PASSES = {n: c for n, c in CASES.items() if c["kind"] == "passes"}
WINDOW = 512                                   # the attention kernels' staged window (kAttnTMax)


def _port(family):
    """The C restatement of a weight family, or None."""
    if family in passes.KQUANT:
        from kq_port import KQPortSlice
        return KQPortSlice
    if family in ("q5_0", "q5_1"):
        from q5_port import Q5PortSlice
        return Q5PortSlice
    return oracle.PortSlice if family in ("q4_0", "q4_1", "q8_0", "f16") else None


def test_fixture_covers_every_family_and_the_kernels_of_each_pass():
    assert {(c["shape"], c["family"]) for c in PASSES.values()} == {
        (sh, f) for sh, fams in passes.FAMILIES.items() for f in fams}
    assert len(passes.FAMILIES["65b"]) == 9
    ops = passes.ops()
    for name, c in PASSES.items():
        assert (c["ops"], c["n_ctx"], c["n_sessions"]) == (ops, 1024, 12), name
        assert [len(d) for d in c["digests"]] == [len(passes.op_sessions(op)) for op in ops], name
        assert c["n_past"] == passes.positions(c)[1], name
    pos, n_past = passes.positions(next(iter(PASSES.values())))
    kinds = [op["op"] for op in ops]
    # every call the reference makes is at most RefSlice.MAX_CHUNK rows
    assert max(n for op in ops for _, n in passes.op_sessions(op) if op["op"] != "steps") == oracle.RefSlice.MAX_CHUNK
    # 1: 12 ragged prompts, 1..32 rows, not in session order, all inside the staged window
    first = ops[0]
    assert first["op"] == "mixed" and sorted(first["sessions"]) == list(range(12))
    assert first["sessions"] != list(range(12))
    assert min(first["counts"]) == 1 and max(first["counts"]) == 32 and sum(first["counts"]) == 148
    # 2: batched steps over 12 and 9 sessions
    assert [len(op["sessions"]) for op in ops if op["op"] == "batch"] == [12, 12, 12, 9, 12]
    # 4: A's segment past 512 (per-query kernel), another below it (tiled), two single tokens
    i = kinds.index("mixed", 1)
    segs = list(zip(passes.op_sessions(ops[i]), pos[i]))
    assert [(s, n) for (s, n), _ in segs] == [(7, 1), (passes.A, 29), (0, 20), (9, 1)]
    assert segs[1][1] > WINDOW and segs[2][1] + 20 <= WINDOW
    assert (segs[1][1] + 29) % 32 == 0           # where the row length decides the V sum's float / double split
    # 5: decode rows across 512, the speculative maximum past it, 40 rows near the start
    steps = [(op["session"], op["count"], pos[j][0]) for j, op in enumerate(ops) if op["op"] == "steps"]
    assert steps[0][:2] == (passes.B, 24) and steps[0][2] < WINDOW < steps[0][2] + 24
    assert steps[1][:2] == (passes.A, 16) and steps[1][2] > WINDOW
    assert steps[2][1] == 40 and steps[2][2] < 10
    # 6: the last batched step spans distant positions
    assert min(pos[-1]) < 10 and max(pos[-1]) == 560 and n_past[passes.A] == 561
    # the digests are of distinct outputs (a repeated digest would mean a constant output)
    every = [d for c in PASSES.values() for op in c["digests"] for d in op]
    assert len(set(every)) == len(every)
    gen = CASES["13b_generate"]
    assert len(gen["ids"]) == gen["n_steps"] == 24 and all(len(r) == len(gen["prompts"]) == 3 for r in gen["ids"])


@pytest.mark.parametrize("name", [n for n in PASSES if n.startswith("13b_")])
def test_port_reproduces_13b_digests(tmp_path, name):
    case = PASSES[name]
    port = _port(case["family"])
    if port is None:
        pytest.skip("no C restatement of %s slices" % case["family"])
    path = str(tmp_path / "w.bin")
    passes.write_case_file(path, case)
    assert vocab.file_sha256(path) == case["file_sha256"], "the writer changed: regenerate the fixture"
    cpu = port(path, case["n_ctx"])
    try:
        got = passes.case_digests(case, passes.replay(cpu, case, passes.inputs(case)))
    finally:
        cpu.close()
    wrong = [(i, s) for i, op in enumerate(case["ops"]) for k, (s, _) in enumerate(passes.op_sessions(op))
             if got[i][k] != case["digests"][i][k]]
    assert not wrong, "(operation, session) %s differ from the reference" % wrong


def test_port_greedy_loop_gives_the_13b_reference_ids(tmp_path):
    from kq_port import KQPortExtra, KQPortSlice
    case = CASES["13b_generate"]
    path, epath = str(tmp_path / "w.bin"), str(tmp_path / "extra.bin")
    klarge.write_layers(path, case)
    ggjt.write_kquant_extra(epath, ggjt.SHAPES["13b"], case["mix"], seed=case["seed"])
    assert (vocab.file_sha256(path), vocab.file_sha256(epath)) == (case["file_sha256"], case["extra_sha256"])
    cpu, extra = KQPortSlice(path, 128), KQPortExtra(epath)
    try:
        ids = [passes.greedy(cpu, extra.embed, extra.logits, p, case["n_steps"]) for p in case["prompts"]]
    finally:
        cpu.close()
    assert [list(r) for r in zip(*ids)] == case["ids"]
    assert len({i for r in ids for i in r}) > 3            # not one id over and over


def test_replay_splits_each_operation_per_session():
    """replay's mapping from a pass to calls, on a stand-in checker that records the calls it receives."""
    case = dict(next(iter(PASSES.values())), shape="tiny")

    class Recorder:
        def __init__(self):
            self.calls = []

        def clear_context(self):
            self.calls.append("clear")

        def forward(self, x):
            self.calls.append(len(x))
            return x + 1

    xs = passes.inputs(case)
    rec = Recorder()
    out = passes.replay(rec, case, xs, [passes.A])
    ops = case["ops"]
    want = ["clear"] + [n if op["op"] != "steps" else 1 for op in ops for s, n in passes.op_sessions(op)
                        if s == passes.A for _ in range(n if op["op"] == "steps" else 1)]
    assert rec.calls == want
    for (i, s), y in out.items():
        k = [t for t, _ in passes.op_sessions(ops[i])].index(s)
        assert (y == passes.split(ops[i], xs[i])[k] + 1).all()
