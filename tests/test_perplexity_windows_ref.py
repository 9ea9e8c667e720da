"""CPU: llama.cpp's windowed perplexity (examples/perplexity/perplexity.cpp) and its host twin.

* The compiled `perplexity` program (oracle/_ref/perplexity) on a tiny Q4_0 model against the twin (client.ppl_terms,
  windowed_perplexity_terms, running_perplexity) on the logits of the reference's own `llm` module path (get_inputs,
  TransformerSlice fed segment by segment, get_llm_output), to the 4 decimals the program prints; and against the
  fixture tests/golden/ppl_windows.json the GPU tests read.
* The twin's window rules and term arithmetic, and the arguments capi.perplexity_windows refuses before it reaches a
  device."""
import json
import math
import os
import sys
import tempfile
import types

import numpy as np
import pytest

from distributedllm_b200 import capi, ggjt
from distributedllm_b200.client import ppl_terms, running_perplexity, windowed_perplexity_terms

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import gen_golden_ppl_windows as gen  # noqa: E402

with open(os.path.join(HERE, "golden", "ppl_windows.json")) as _f:
    FIXTURE = json.load(_f)

needs_binary = pytest.mark.skipif(not (os.path.isfile(gen.BINARY) and os.path.isfile(os.path.join(ROOT, "oracle", "_ref",
                                                                                                  "libllmref.so"))),
                                  reason="oracle/_ref (perplexity, libllmref.so) not built")


def _llm_module_terms(model, extra, tokens, n_ctx, n_batch):
    """The twin on the reference llm module's logits: each window from a cleared slice, one forward per segment."""
    from oracle import oracle
    sh = ggjt.SHAPES[gen.SHAPE]
    ref = oracle.RefSlice(model, 1, n_ctx)

    def eval_segment(ids, n_past):
        assert len(ids) <= oracle.RefSlice.MAX_CHUNK
        if n_past == 0:
            ref.clear_context()
        h = ref.forward(oracle.ref_embed(extra, ids, sh.n_embd))
        return oracle.ref_logits(extra, h, sh.n_vocab, True)

    try:
        return windowed_perplexity_terms(tokens, n_ctx, n_batch, eval_segment)
    finally:
        ref.close()


@needs_binary
def test_binary_equals_the_twin_on_llm_module_logits():
    from oracle import oracle
    with tempfile.TemporaryDirectory() as d:
        full, text_path = os.path.join(d, "full.bin"), os.path.join(d, "text.txt")
        assert gen.write_model(full) == FIXTURE["model_sha256"]
        sl, extra = os.path.join(d, "slice.bin"), os.path.join(d, "extra.bin")
        ggjt.slice_model(full, sl, 0, ggjt.SHAPES[gen.SHAPE].n_layer - 1)
        ggjt.extract_extra_layers(full, extra)
        with open(text_path, "w") as f:
            f.write(gen.text())
        tokens = oracle.ref_tokenize(extra, gen.text())
        assert len(tokens) == FIXTURE["n_ids"]
        for case in FIXTURE["cases"]:
            n_ctx, n_batch = case["n_ctx"], case["n_batch"]
            printed = gen.run_binary(full, text_path, n_ctx, n_batch)
            assert printed == case["printed"], (n_ctx, n_batch)
            assert len(printed) == len(tokens) // n_ctx >= 4
            twin = running_perplexity(_llm_module_terms(sl, extra, tokens, n_ctx, n_batch))
            assert ["%.4f" % v for v in twin] == printed, (n_ctx, n_batch, twin, printed)


def _fake_logits(n_vocab):
    """eval_segment for the window rules: logits that depend on each row's id and position, and a log of the calls."""
    calls = []

    def eval_segment(ids, n_past):
        calls.append((list(ids), n_past))
        pos = np.arange(n_past, n_past + len(ids))[:, None]
        v = np.arange(n_vocab)[None, :]
        return (np.sin(0.37 * v + 0.11 * pos + 0.05 * np.asarray(ids)[:, None]) * 3).astype(np.float32)

    return eval_segment, calls


@pytest.mark.parametrize("n_ctx,n_batch,segments", [(64, 24, [24, 24, 16]), (64, 64, [64]), (64, 512, [64]),
                                                    (50, 7, [7] * 7 + [1])])
def test_window_segments_and_bos(n_ctx, n_batch, segments):
    """perplexity.cpp:44-76: each window from n_past 0 in segments of min(n_batch, n_ctx) rows, its id 0 BOS, the
    other ids (and every target) as tokenized; a trailing partial window is dropped."""
    V = 40
    rng = np.random.default_rng(n_ctx + n_batch)
    tokens = rng.integers(3, V, 3 * n_ctx + n_ctx // 2).tolist()
    ev, calls = _fake_logits(V)
    terms = windowed_perplexity_terms(tokens, n_ctx, n_batch, ev)
    first = min(512, n_ctx // 2)
    assert terms.shape == (3, n_ctx - 1 - first)
    assert [len(ids) for ids, _ in calls] == segments * 3
    assert [p for _, p in calls] == list(np.cumsum([0] + segments[:-1])) * 3
    for i in range(3):
        window = [t for ids, _ in calls[i * len(segments):(i + 1) * len(segments)] for t in ids]
        assert window == [1] + tokens[i * n_ctx + 1:(i + 1) * n_ctx]
    # each term is the twin on that row's logits and the next id of the text (never replaced by BOS)
    ev2, _ = _fake_logits(V)
    i, j = 2, n_ctx - 2
    row = ev2([1] + tokens[i * n_ctx + 1:(i + 1) * n_ctx], 0)[j]
    assert terms[i, j - first] == ppl_terms(row[None], [tokens[i * n_ctx + j + 1]])[0]


@pytest.mark.parametrize("n_ctx,first", [(2, 1), (3, 1), (100, 50), (1024, 512), (1025, 512), (2048, 512)])
def test_first_scored_row(n_ctx, first):
    """perplexity.cpp:103: rows from min(512, n_ctx / 2) to n_ctx - 2 are scored."""
    n_chunk, n_batch, f, n_scored = capi.ppl_window_rows(5 * n_ctx + 1, n_ctx, 512)
    assert (n_chunk, n_batch, f, n_scored) == (5, min(512, n_ctx), first, n_ctx - 1 - first)


def test_fewer_ids_than_a_window():
    ev, calls = _fake_logits(16)
    terms = windowed_perplexity_terms(list(range(3, 13)), 11, 4, ev)
    assert terms.shape == (0, 11 - 1 - 5) and calls == []
    assert running_perplexity(terms) == []


def _plain_term(row, t):
    """perplexity.cpp's softmax + -log(prob) restated one value at a time with Python floats."""
    f32 = lambda v: float(np.float32(v))
    m = max(f32(v) for v in row)
    e = [f32(math.exp(f32(f32(v) - m))) for v in row]
    S = 0.0
    for v in e:
        S += v
    return f32(-f32(math.log(f32(e[t] / S)))) if e[t] / S > 0 else math.inf


def test_twin_term_arithmetic():
    rng = np.random.default_rng(5)
    rows = [rng.standard_normal(1000) * s for s in (0.5, 4.0, 25.0)] + [np.full(37, 2.5)]
    targets = [3, 999, 500, 36]
    rows.append(np.r_[0.0, -200.0, rng.standard_normal(50)])      # e_1 underflows in float: +inf
    targets.append(1)
    for row, t in zip(rows, targets):
        got = ppl_terms(np.asarray(row, np.float32)[None], [t])[0]
        assert got == np.float32(_plain_term(np.asarray(row, np.float32), t)), (got, _plain_term(row, t))
    assert np.isinf(ppl_terms(np.asarray(rows[-1], np.float32)[None], [1])[0])
    # the sum runs in index order: a row where pairwise summation would round differently still matches the loop
    row = np.r_[np.zeros(1, np.float32), np.full(4097, -17.0, np.float32), np.float32(-0.5)]
    assert ppl_terms(row[None], [0])[0] == np.float32(_plain_term(row, 0))


def test_twin_rows_without_a_distribution():
    r = np.random.default_rng(1).standard_normal((4, 33)).astype(np.float32)
    r[0, 5] = np.nan
    r[1, 7] = np.inf
    r[2] = -np.inf
    got = ppl_terms(r, [0, 0, 0, 0])
    assert np.isnan(got[:3]).all() and np.isfinite(got[3])


def test_running_perplexity_order():
    terms = np.array([[0.5, 1.5], [2.0, 0.25]], np.float32)
    assert running_perplexity(terms) == [math.exp(2.0 / 2), math.exp(4.25 / 4)]


def test_capi_refusals_without_a_device():
    """What capi.perplexity_windows refuses before it touches a handle."""
    extra = types.SimpleNamespace(n_vocab=100, handle=None)
    toks = list(range(1, 50))
    for kw, err in (({"n_ctx": 1}, ValueError), ({"n_ctx": 0}, ValueError), ({"n_ctx": 8, "n_batch": 0}, ValueError),
                    ({"n_ctx": 8, "n_batch": -3}, ValueError), ({"n_ctx": 8.0}, TypeError), ({"n_ctx": True}, TypeError)):
        with pytest.raises(err):
            capi.perplexity_windows([], extra, [0], toks, **kw)
    with pytest.raises(ValueError, match="twice"):
        capi.perplexity_windows([], extra, [0, 1, 0], toks, 8)
    with pytest.raises(ValueError, match="at least one session"):
        capi.perplexity_windows([], extra, [], toks, 8)
    for bad in (-1, 100):
        with pytest.raises(ValueError, match="token ids"):
            capi.perplexity_windows([], extra, [0], toks + [bad], 8)


def test_fixture_is_what_the_generator_writes():
    """The fixture's model is the writer's output byte for byte (so the GPU test rebuilds the same model)."""
    with tempfile.TemporaryDirectory() as d:
        assert gen.write_model(os.path.join(d, "m.bin")) == FIXTURE["model_sha256"]
    assert [(c["n_ctx"], c["n_batch"]) for c in FIXTURE["cases"]] == list(gen.CASES)
    for c in FIXTURE["cases"]:
        assert len(c["printed"]) == FIXTURE["n_ids"] // c["n_ctx"]
