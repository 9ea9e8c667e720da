"""GPU at numeric edges (tests/edge_cases.py): every weight family x slice recipe x input class, bit for bit against the C
restatement and, where oracle/_ref is built, the reference itself.  Prompt chunks, single-token graph replays, batched
steps and mixed passes, the switches that move activation quantisation to another site, one LLaMA-7B layer, and the
extra layers (embedding rows, lm_head).  NaN counts as equal to NaN, though none is expected."""
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import edge_cases as ec  # noqa: E402
from test_oracle_edges import FAMILIES, SCHEDULE, _fid, layers_of, port_slice  # noqa: E402

pytestmark = pytest.mark.gpu


def _bad(a, b):
    """Floats of a and b that differ in their bits (two NaNs are equal)."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return int(((a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))).sum())


class _Checkers:
    """The C restatement, and the compiled reference when it is built, fed the same calls."""

    def __init__(self, path, wtype, n_ctx):
        self.cs = [port_slice(path, wtype, n_ctx)]
        if oracle.have_ref():
            self.cs.append(oracle.RefSlice(path, 3, n_ctx))

    def forward(self, x):
        return [c.forward(x) for c in self.cs]

    def clear_context(self):
        for c in self.cs:
            c.clear_context()

    def close(self):
        for c in self.cs:
            c.close()


def _run_classes(path, wtype, n_embd, rng, classes=ec.CLASSES, schedule=SCHEDULE, n_ctx=64):
    """For each class: a fresh context, a prompt chunk, then single-token steps; returns [(class, call, bad)]."""
    from distributedllm_b200 import capi
    gpu, chk = capi.Slice(path, 0, n_ctx), _Checkers(path, wtype, n_ctx)
    out = []
    try:
        for cls in classes:
            gpu.clear_context()
            chk.clear_context()
            for i, n in enumerate(schedule):
                x = ec.inputs(cls, n, n_embd, rng)
                y = gpu.forward(x)
                for w in chk.forward(x):
                    out.append((cls, i, _bad(y, w)))
    finally:
        gpu.close()
        chk.close()
    return out


def _assert_exact(res, where):
    bad = [r for r in res if r[2]]
    assert not bad, "%s: (class, call, floats differing): %s" % (where, bad)


@pytest.mark.parametrize("recipe", ec.RECIPES)
@pytest.mark.parametrize("family", FAMILIES, ids=_fid)
def test_edges_prompt_then_single_token_steps(tmp_path, family, recipe):
    shape, wtype = family
    path = ec.make_slice(str(tmp_path), shape, wtype, recipe, layers_of(wtype))
    rng = np.random.default_rng([7, ec.RECIPES.index(recipe)])
    _assert_exact(_run_classes(path, wtype, ggjt.SHAPES[shape].n_embd, rng), (family, recipe))


SWITCHES = [{"B200_NQ": "1"}, {"B200_RING": "0"}, {"B200_TILED_ATTN": "0"}, {"B200_F16_MC": "0"}, {"B200_F16_MC": "8"},
            {"B200_NC": "2"}]
SWITCH_FAMILIES = [("tiny128", ggjt.T_Q4_0), ("tiny3b", ggjt.T_Q4_1), ("tiny128", ggjt.T_Q5_1), ("tiny", ggjt.T_Q8_0),
                   ("tiny128", ggjt.T_F16), ("tiny3b", ggjt.T_F16), ("tinyk128", "q4_K_M"), ("tinyk", "q6_K")]


@pytest.mark.parametrize("env", SWITCHES, ids=lambda e: "-".join("%s=%s" % kv for kv in e.items()))
@pytest.mark.parametrize("family", SWITCH_FAMILIES, ids=_fid)
def test_edges_under_quantisation_site_switches(tmp_path, monkeypatch, family, env):
    """The fused RMSNorm prologue, the grid-barrier norm+quant epilogue (B200_NQ=1), the ring-less kernels, the per-query
    prompt attention, the F16 column counts and 2 columns per CTA quantise the same blocks elsewhere."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    shape, wtype = family
    sh = ggjt.SHAPES[shape]
    for recipe in ("zeros", "unit_norm"):
        path = ec.make_slice(str(tmp_path), shape, wtype, recipe, layers_of(wtype))
        rng = np.random.default_rng(17)
        _assert_exact(_run_classes(path, wtype, sh.n_embd, rng, schedule=(20, 1, 1, 7, 1)), (family, env, recipe))


@pytest.mark.parametrize("family", [("tiny128", ggjt.T_Q4_0), ("tiny3b", ggjt.T_Q4_1), ("tiny", ggjt.T_F16),
                                    ("tiny128", ggjt.T_Q5_0), ("tinyk128", "q4_K_M")], ids=_fid)
def test_edges_batched_step_and_mixed_pass(tmp_path, family):
    """Three sessions holding different classes: prompts, a mixed pass (a chunk beside single tokens), batched steps,
    then single-token steps; each session against its own restatement."""
    from distributedllm_b200 import capi
    shape, wtype = family
    sh = ggjt.SHAPES[shape]
    path = ec.make_slice(str(tmp_path), shape, wtype, "zeros", layers_of(wtype))
    classes = ("lattice", "outlier", "tiny40")
    rng = np.random.default_rng(23)
    gpu = capi.Slice(path, 0, 96, n_sessions=4)
    chk = [_Checkers(path, wtype, 96) for _ in classes]
    ids = [2, 0, 3]
    try:
        for k, cls, n in zip(ids, classes, (9, 1, 14)):
            x = ec.inputs(cls, n, sh.n_embd, rng)
            y = gpu.session_forward(k, x)
            assert all(_bad(y, w) == 0 for w in chk[ids.index(k)].forward(x)), ("prompt", cls)
        for counts in ([1, 12, 3], [5, 1, 1]):
            xs = [ec.inputs(cls, c, sh.n_embd, rng) for cls, c in zip(classes, counts)]
            y = gpu.mixed_forward(ids, counts, np.concatenate(xs))
            r0 = 0
            for j, (cls, c) in enumerate(zip(classes, counts)):
                assert all(_bad(y[r0:r0 + c], w) == 0 for w in chk[j].forward(xs[j])), ("mixed", counts, cls)
                r0 += c
        for step in range(3):
            xs = [ec.inputs(cls, 1, sh.n_embd, rng) for cls in classes]
            y = gpu.batch_forward(ids, np.concatenate(xs))
            for j, cls in enumerate(classes):
                assert all(_bad(y[j:j + 1], w) == 0 for w in chk[j].forward(xs[j])), ("batch", step, cls)
        for j, (k, cls) in enumerate(zip(ids, classes)):
            x = ec.inputs(cls, 1, sh.n_embd, rng)
            y = gpu.session_forward(k, x)
            assert all(_bad(y, w) == 0 for w in chk[j].forward(x)), ("step", cls)
    finally:
        gpu.close()
        for c in chk:
            c.close()


@pytest.mark.parametrize("wtype", [ggjt.T_Q4_0, "q4_K_M"], ids=["q4_0", "q4_K_M"])
def test_edges_one_7b_layer(tmp_path, wtype):
    """One LLaMA-7B layer (real tile counts and ring wrap) with unit norm weights, outlier and lattice rows."""
    sh = ggjt.SHAPES["7b"]
    src = str(tmp_path / "l.bin")
    if wtype == "q4_K_M":
        ggjt.write_kquant_slice(src, sh, 0, 0, "q4_K_M", seed=3)       # layer 0: Q6_K wv / w2
    else:
        ggjt.write_fast_q4_slice(src, sh, 0, 0, seed=3)
    path = ec.rewrite(src, str(tmp_path / "u.bin"), "unit_norm")
    rng = np.random.default_rng(31)
    _assert_exact(_run_classes(path, wtype, sh.n_embd, rng, classes=("outlier", "lattice"), schedule=(20, 1, 1)),
                  ("7b", wtype))


EMBED_TYPES = [ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0, ggjt.T_F16, ggjt.T_F32, ggjt.T_Q4_K]
REF_EMBEDS = (ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q4_K)


@pytest.mark.parametrize("wtype", EMBED_TYPES, ids=lambda t: ggjt.TYPE_NAME[t])
def test_edges_embedding_rows(tmp_path, wtype):
    """k_embed_rows on tok_embeddings blocks with scales of 0, 2^-20, powers of two, negative minima, Q4_K scales and
    minima of 0 / 63 and subnormal d / dmin, F16 subnormals and +-65504-range values."""
    from distributedllm_b200 import capi
    path = ec.make_extra(str(tmp_path), wtype)
    f = ggjt.read_file(path, sliced=True)
    toks = ec.embed_tokens(f.hparams.n_vocab)
    extra = capi.Extra(path, 0)
    try:
        got = extra.embed(toks)
    finally:
        extra.close()
    want = [ec.dequant_rows(f, "tok_embeddings.weight", toks)]
    if oracle.have_ref() and wtype in REF_EMBEDS:
        want.append(oracle.ref_embed(path, toks, f.hparams.n_embd))
    for w in want:
        assert np.isfinite(w).all() and _bad(got, w) == 0, _bad(got, w)


@pytest.mark.parametrize("out", ["q4_0", "q6_K"])
def test_edges_logits(tmp_path, out):
    """The lm_head (RMSNorm with unit weights, Q8_0 / Q8_K, Q4_0 / Q6_K with edge block scales) on outlier, zero and
    lattice rows, one and several rows per call."""
    from distributedllm_b200 import capi
    path = ec.make_extra(str(tmp_path), ggjt.T_Q4_0 if out == "q4_0" else ggjt.T_Q4_K)
    f = ggjt.read_file(path, sliced=True)
    rng = np.random.default_rng(4)
    extra = capi.Extra(path, 0)
    try:
        for cls in ("outlier", "zeros", "lattice", "alternating"):
            x = ec.inputs(cls, 6, f.hparams.n_embd, rng)
            want = [ec.port_logits(path, x)]
            if oracle.have_ref():
                want.append(oracle.ref_logits(path, x, f.hparams.n_vocab, True))
            for got in (extra.logits(x), np.concatenate([extra.logits(x[i:i + 1]) for i in range(len(x))])):
                for w in want:
                    assert np.isfinite(w).all() and _bad(got, w) == 0, (cls, _bad(got, w))
    finally:
        extra.close()
