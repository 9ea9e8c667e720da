"""The C restatements against the compiled reference at numeric edges (tests/edge_cases.py): every slice recipe x input
class, bit for bit, so that they can stand in for the reference in the GPU edge tests.  Also the witness: the edge
classes must actually reach the quantiser branches they are meant for (zero blocks, exact ties, fp16-zero scales,
id = inf blocks, Q8_K magnitude ties with either sign first)."""
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import edge_cases as ec  # noqa: E402

needs_ref = pytest.mark.skipif(not oracle.have_ref(), reason="oracle/_ref is not built (it needs the reference sources)")

FAMILIES = [(s, t) for t in (ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0, ggjt.T_F16)
            for s in ("tiny", "tiny3b", "tiny128")] + [(s, m) for m in ("q4_K_S", "q4_K_M", "q6_K") for s in ("tinyk", "tinyk128")]
SCHEDULE = (20, 1, 1, 1)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _fid(f):
    return "%s-%s" % (f[0], f[1] if isinstance(f[1], str) else ggjt.TYPE_NAME[f[1]])


def port_slice(path, wtype, n_ctx):
    """The C restatement that covers this slice's weight type."""
    if isinstance(wtype, str) or wtype in (ggjt.T_Q4_K, ggjt.T_Q6_K):
        from kq_port import KQPortSlice
        return KQPortSlice(path, n_ctx)
    if wtype in (ggjt.T_Q5_0, ggjt.T_Q5_1):
        from q5_port import Q5PortSlice
        return Q5PortSlice(path, n_ctx)
    return oracle.PortSlice(path, n_ctx)


def layers_of(wtype):
    return (2, 3) if isinstance(wtype, str) else (0, 1)      # Q4_K_M: layer 3's wv / w2 are Q6_K, layer 2's Q4_K


@needs_ref
@pytest.mark.parametrize("recipe", ec.RECIPES)
@pytest.mark.parametrize("family", FAMILIES, ids=_fid)
def test_port_matches_reference_at_edges(tmp_path, family, recipe):
    shape, wtype = family
    sh = ggjt.SHAPES[shape]
    path = ec.make_slice(str(tmp_path), shape, wtype, recipe, layers_of(wtype))
    port, ref = port_slice(path, wtype, 64), oracle.RefSlice(path, 3, 64)
    rng = np.random.default_rng([7, ec.RECIPES.index(recipe)])
    try:
        for cls in ec.CLASSES:
            port.clear_context()
            ref.clear_context()
            for i, n in enumerate(SCHEDULE):
                x = ec.inputs(cls, n, sh.n_embd, rng)
                a, b = port.forward(x), ref.forward(x)
                assert np.isfinite(b).all(), (cls, i, "the reference's output is not finite")
                bad = int((_bits(a) != _bits(b)).sum())
                assert bad == 0, "%s call %d (N=%d): %d floats differ" % (cls, i, n, bad)
    finally:
        port.close()
        ref.close()


@pytest.mark.parametrize("shape", ["tiny", "tiny3b", "tinyk128"])
def test_witness_reaches_every_quantiser_edge(tmp_path, shape):
    """Counted on the first layer's qkv input of a unit-norm slice, over the rows the edge tests feed."""
    from kq_port import lib as kq_lib
    sh = ggjt.SHAPES[shape]
    path = ec.make_slice(str(tmp_path), shape, "q4_K_M" if shape == "tinyk128" else ggjt.T_Q4_0, "unit_norm",
                         (2, 3) if shape == "tinyk128" else (0, 1))
    w = ec.slice_norm(path)
    assert (w == 1).all()
    rng = np.random.default_rng(11)
    per = {}
    for cls in ec.CLASSES:
        per[cls] = ec.witness(oracle.port_lib(), kq_lib(), ec.inputs(cls, 20, sh.n_embd, rng), w)
    tot = {k: sum(p[k] for p in per.values()) for k in per["gauss"]}
    nb = sh.n_embd // 32
    assert per["lattice"]["ties"] >= 20 * nb * 8, per["lattice"]               # ~half of every block's odd entries
    assert per["zeros"]["zero_blocks"] >= 7 * nb, per["zeros"]
    assert per["tiny40"]["id_inf"] == 20 * nb, per["tiny40"]                   # 127 / amax overflows in every block
    # 1e-30 rows: x * x underflows, RMSNorm scales by 1/sqrt(eps), fp16(amax / 127) = 0 while id stays finite
    assert per["tiny40"]["d16_zero"] == 20 * nb and per["tiny30"]["d16_zero"] == 20 * nb, (per["tiny40"], per["tiny30"])
    assert per["tiny30"]["id_inf"] == 0, per["tiny30"]
    assert per["gauss"]["ties"] == 0 and per["gauss"]["zero_blocks"] == 0 and tot["id_inf"] == per["tiny40"]["id_inf"]
    if sh.n_embd % 256 == 0:
        nbk = sh.n_embd // 256
        assert per["alternating"]["q8k_ties_neg_first"] == 10 * nbk, per["alternating"]
        assert per["alternating"]["q8k_ties_pos_first"] == 10 * nbk, per["alternating"]
        assert per["zeros"]["q8k_zero"] >= 7 * nbk, per["zeros"]
        # the lattice rows with a 256 per super-block (every other row): iscale = -32, every odd entry lands on k + 1/2
        assert per["lattice"]["q8k_ties"] >= 10 * sh.n_embd * 9 // 10, per["lattice"]
        assert per["gauss"]["q8k_ties"] == 0, per["gauss"]
        assert per["constant"]["q8k_ties_neg_first"] + per["constant"]["q8k_ties_pos_first"] == 0


@needs_ref
@pytest.mark.parametrize("wtype", [ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q4_K],
                         ids=lambda t: ggjt.TYPE_NAME[t])
def test_embedding_rows_with_edge_scales_match_reference(tmp_path, wtype):
    """numpy's dequantisers (the GPU embed tests' fallback checker) against the reference's ggml_get_rows, for the
    quantised types the reference embeds (its Q8_0, F16 and F32 embedding paths crash on these files)."""
    path = ec.make_extra(str(tmp_path), wtype)
    f = ggjt.read_file(path, sliced=True)
    toks = ec.embed_tokens(f.hparams.n_vocab)
    want = oracle.ref_embed(path, toks, f.hparams.n_embd)
    assert np.isfinite(want).all()
    got = ec.dequant_rows(f, "tok_embeddings.weight", toks)
    assert (_bits(got) == _bits(want)).all(), int((_bits(got) != _bits(want)).sum())


@needs_ref
@pytest.mark.parametrize("out", ["q4_0", "q6_K"])
def test_logits_at_edges_match_reference(tmp_path, out):
    """The restated lm_head (RMSNorm, Q8_0 / Q8_K, the Q4_0 / Q6_K dot) against the reference's get_logits on outlier,
    zero and lattice rows with unit norm weights and edge block scales."""
    path = ec.make_extra(str(tmp_path), ggjt.T_Q4_0 if out == "q4_0" else ggjt.T_Q4_K)
    f = ggjt.read_file(path, sliced=True)
    rng = np.random.default_rng(4)
    for cls in ("outlier", "zeros", "lattice", "alternating", "gauss"):
        x = ec.inputs(cls, 6, f.hparams.n_embd, rng)
        want = oracle.ref_logits(path, x, f.hparams.n_vocab, True)
        assert np.isfinite(want).all(), cls
        got = ec.port_logits(path, x)
        assert (_bits(got) == _bits(want)).all(), (cls, int((_bits(got) != _bits(want)).sum()))
