"""CPU: the k-quant fixtures at LLaMA-13B, 30B and 65B shapes (tests/golden/ref_digests_kquant_large.json and
ref_kquant_types_deep.json, written by tests/golden/gen_golden_kquant_large.py) -- the writer's per-tensor types against
the reference's `quantize` at the real 40, 60 and 80 layer counts, what the digest fixture covers, and the C restatement
(tests/kq_port.c) reproducing the 13B digests, so that the GPU tests' fallback checker is pinned at a second shape."""
import itertools
import json
import os
import sys

import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
import gen_golden_kquant_large as klarge  # noqa: E402
import gen_golden_large as large  # noqa: E402
import gen_golden_vocab as vocab  # noqa: E402

CASES = json.load(open(os.path.join(GOLD, "ref_digests_kquant_large.json")))
TYPES = json.load(open(os.path.join(GOLD, "ref_kquant_types_deep.json")))
SHAPES = ("13b", "30b", "65b")
WV_W2 = ("attention.wv.weight", "feed_forward.w2.weight")


def test_writer_types_equal_reference_quantize_at_40_60_80_layers():
    """ggjt.kquant_tensor_type against the types the reference's `quantize` wrote on 40-, 60- and 80-layer models, for
    the full file and a slice_model cut across 7 n_layer / 8; the cut keeps the full model's types."""
    assert sorted(TYPES["n_layer"].values()) == [40, 60, 80]
    assert len(TYPES["types"]) == 3 * 3 * 2
    for key, types in TYPES["types"].items():
        label, mix, what = key.split("/")
        n_layer = TYPES["n_layer"][label]
        a, b = TYPES["cuts"][label]
        layers = range(n_layer) if what == "full" else range(a, b + 1)
        assert what in ("full", "slice_%d_%d" % (a, b)), key
        assert {n for n in types if n.startswith("layers.")} == {"layers.%d.%s" % (i, m) for i in layers
                                                                 for m in ggjt.LAYER_TENSORS}, key
        for name, tname in types.items():
            if tname == "f32":
                assert name.endswith("norm.weight"), (key, name)
                continue
            assert ggjt.TYPE_NAME[ggjt.kquant_tensor_type(name, mix, n_layer)] == tname, (key, name)
        if mix == "q4_K_M":
            q6 = {n for n, t in types.items() if t == "q6_K" and n.startswith("layers.")}
            assert q6 == {"layers.%d.%s" % (i, m) for i in layers if ggjt.use_more_bits(i, n_layer) for m in WV_W2}, key
    # where n_layer / 8 and 7 n_layer / 8 are rounded: 60 layers switch at 7 and 52, not 8 and 53
    assert [ggjt.use_more_bits(i, 60) for i in (6, 7, 8, 9, 51, 52)] == [True, False, False, True, True, True]
    assert TYPES["types"]["deep60/q4_K_M/full"]["layers.52.feed_forward.w2.weight"] == "q6_K"
    assert TYPES["types"]["deep60/q4_K_M/full"]["layers.50.feed_forward.w2.weight"] == "q4_K"


def test_digest_fixture_covers_every_shape_and_mix():
    sched = {(c["shape"], c["mix"]) for c in CASES.values() if c["kind"] == "schedule" and c["n_ctx"] == 512}
    assert sched == set(itertools.product(SHAPES, ("q4_K_S", "q4_K_M", "q6_K")))
    for name, c in CASES.items():
        if c["kind"] == "schedule":
            assert len(c["digests"]) == len(c["schedule"]), name
            assert c["schedule"] == (large.SCHEDULE if c["n_ctx"] == 512 else klarge.DEEP_SCHEDULE), name
    deep = CASES["13b_q4_K_M_deep"]
    assert (deep["n_ctx"], sum(deep["schedule"]), max(deep["schedule"])) == (2048, 2048, 32)
    assert sum(deep["schedule"][:deep["schedule"].index(1)]) == 2000
    batch = CASES["65b_q4_K_M_batch"]
    assert (batch["prompt_len"], batch["sessions"]) == (large.BATCH_PROMPTS, large.BATCH_SESSIONS)
    assert len(batch["step_digests"]) == batch["n_steps"] and all(len(s) == 12 for s in batch["step_digests"])
    for shape in SHAPES:
        e = CASES[shape + "_extra"]
        assert (e["n_vocab"], e["rows"]) == (32000, [1, 8, 9, 13])
        assert {0, 31999} <= set(e["embed_ids"]) and len(e["embed"]) == 7
        assert [len(d) for d in e["logits"]] == e["rows"] == [len(a) for a in e["argmax"]]
    # the digests are of distinct outputs (a digest repeated across calls would mean a constant output)
    every = [d for c in CASES.values() for d in c.get("digests", [])]
    assert len(set(every)) == len(every)


@pytest.mark.parametrize("shape", SHAPES)
def test_q4_K_M_file_holds_an_all_q4_K_layer_and_a_q6_K_wv_w2_layer(tmp_path, shape):
    """The Q4_K_M file every Q4_K_M case of the shape runs on, written as the GPU tests write it: the first layer's
    matrices are all Q4_K, the second's wv and w2 are Q6_K and the rest Q4_K; the bytes are the fixture's."""
    case = CASES["%s_q4_K_M" % shape]
    path = str(tmp_path / "w.bin")
    klarge.write_case_file(path, case)
    assert vocab.file_sha256(path) == case["file_sha256"], "the writer changed: regenerate the fixture"
    f = ggjt.read_file(path, sliced=True)
    a, b = case["layers"]
    assert (f.hparams.first_layer, f.hparams.n_layer, b) == (a, 2, a + 1)
    assert ggjt.use_more_bits(b, ggjt.SHAPES[shape].n_layer) and not ggjt.use_more_bits(a, ggjt.SHAPES[shape].n_layer)
    for m in ggjt.LAYER_MATRICES:
        assert f.tensors["layers.%d.%s" % (a, m)].ttype == ggjt.T_Q4_K, m
        assert f.tensors["layers.%d.%s" % (b, m)].ttype == (ggjt.T_Q6_K if m in WV_W2 else ggjt.T_Q4_K), m
    os.remove(path)


@pytest.mark.parametrize("name", ["13b_q4_K_S", "13b_q6_K", "13b_q4_K_M", "13b_extra"])
def test_port_reproduces_13b_digests(tmp_path, name):
    """tests/kq_port.c against the reference's 13B digests: every call of the schedules, and the extra layers'
    embedding rows and logits.  (It reproduces 13b_q4_K_M_deep too, but that takes about 5 minutes on 8 cores.)"""
    from kq_port import KQPortExtra, KQPortSlice
    case = CASES[name]
    path = str(tmp_path / "w.bin")
    klarge.write_case_file(path, case)
    assert vocab.file_sha256(path) == case["file_sha256"], "the writer changed: regenerate the fixture"
    if case["kind"] == "extra":
        port = KQPortExtra(path)
        for n, want in zip(case["rows"], case["logits"]):
            assert [klarge.digest(r) for r in port.logits(vocab.hidden(case, n))] == want, n
        assert [klarge.digest(r) for r in port.embed(case["embed_ids"])] == case["embed"]
        return
    port = KQPortSlice(path, case["n_ctx"])
    try:
        got = [klarge.digest(port.forward(x)) for x in large.case_inputs(case)]
    finally:
        port.close()
    wrong = [i for i, (g, w) in enumerate(zip(got, case["digests"])) if g != w]
    assert not wrong, "calls %s differ from the reference" % wrong


@pytest.mark.skipif(not oracle.have_ref(), reason="oracle/_ref not built")
def test_reference_replays_13b_q4_K_M_live(tmp_path):
    """The compiled reference itself, on the 13B Q4_K_M file: the fixture is what it computes today."""
    case = CASES["13b_q4_K_M"]
    path = str(tmp_path / "w.bin")
    klarge.write_case_file(path, case)
    got = large.ref_schedule(path, case, min(16, os.cpu_count() or 4))
    assert [klarge.digest(y) for y in got] == case["digests"]
