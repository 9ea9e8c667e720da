"""RMSNorm rows whose scale depends on the order of the float64 sum of squares (tests/norm_order.py), without a GPU:

* every constructed row is a witness: the sequential and the exact sum give different scales, and the family's
  activation quantiser turns those into different activations;
* the C restatement's orc_rmsnorm is the sequential sum, bit for bit;
* the compiled reference, fed witness rows, equals the restatement and differs from it fed the exact sum's scale;
* the kernels' certification (rms_scale in kernels.cuh), restated: wherever it accepts a tree sum, its float mean is the
  sequential one, over 10^5 rows of several kinds summed in several orders.
"""
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import edge_cases as ec  # noqa: E402
import norm_order as no  # noqa: E402

needs_ref = pytest.mark.skipif(not oracle.have_ref(), reason="oracle/_ref is not built (it needs the reference sources)")


def _norm_w(k: int) -> np.ndarray:
    rng = np.random.default_rng(k)
    return (1.0 + 0.1 * rng.standard_normal(k)).astype(np.float32)


@pytest.mark.parametrize("k", no.WIDTHS)
def test_witness_rows_change_scale_and_activations(k):
    w = _norm_w(k)
    n = 0
    for fam in no.FAMILIES:
        if fam == "q8_k" and k % 256:
            continue
        for d in no.DIRECTIONS:
            for where in no.PLACES:
                x = no.witness_row(k, fam, w, d, where)
                t = no.squares(x)
                s_seq, s_exact = no.scales(x)
                assert s_seq != s_exact, (fam, d, where)
                assert no.activations_differ(fam, x, s_seq, s_exact, w), (fam, d, where)
                # the sequential sum sits on a float32 tie of the mean; the exact one on the side given by `d`
                mean = np.float64(no.sequential_sum(t)) / k
                assert np.float64(np.float32(mean)) != mean
                assert (no.fsum(t) > no.sequential_sum(t)) == (d == "down")
                n += 1
    assert n >= 18


@pytest.mark.parametrize("k", no.WIDTHS)
def test_port_rmsnorm_is_the_sequential_sum(k):
    """orc_rmsnorm (the order the GPU is checked against) equals sequential_sum -> ref_scale bit for bit."""
    w = _norm_w(k)
    L = oracle.port_lib()
    for fam in ("q8_0", "f16"):
        for d in no.DIRECTIONS:
            for where in no.PLACES:
                x = no.witness_row(k, fam, w, d, where)
                got = np.empty(k, np.float32)
                L.orc_rmsnorm(ec.ptr(x), ec.ptr(w), k, ec.ptr(got))
                s = no.ref_scale(no.sequential_sum(no.squares(x)), k)
                want = (x * s).astype(np.float32) * w
                assert (got.view(np.uint32) == want.view(np.uint32)).all(), (fam, d, where)


REF_FAMILIES = [("tiny", ggjt.T_Q4_0), ("tiny", ggjt.T_Q4_1), ("tiny128", ggjt.T_Q5_0), ("tiny128", ggjt.T_Q5_1),
                ("tiny", ggjt.T_Q8_0), ("tiny", ggjt.T_F16), ("tinyk", "q4_K_M"), ("tinyk128", "q6_K")]


def _fid(f):
    return "%s-%s" % (f[0], f[1] if isinstance(f[1], str) else ggjt.TYPE_NAME[f[1]])


@needs_ref
@pytest.mark.parametrize("family", REF_FAMILIES, ids=_fid)
def test_reference_sums_in_index_order(tmp_path, family):
    """One-layer slices fed witness rows: the compiled reference equals the restatement bit for bit, and the rows are
    chosen so that a restatement using the exact sum's scale would differ (checked on the first activation quantiser)."""
    from test_oracle_edges import port_slice
    shape, wtype = family
    sh = ggjt.SHAPES[shape]
    src = str(tmp_path / "s.bin")
    layers = (3, 3) if isinstance(wtype, str) else (0, 0)
    if isinstance(wtype, str):
        ggjt.write_kquant_slice(src, sh, layers[0], layers[1], wtype, seed=2)
    else:
        ggjt.write_synth_slice(src, sh, layers[0], layers[1], wtype, seed=2)
    w = ec.slice_norm(src)
    fam = no.family_of(wtype)
    x = np.stack([no.witness_row(sh.n_embd, fam, w, d, where) for d in no.DIRECTIONS for where in no.PLACES])
    for r in x:
        s_seq, s_exact = no.scales(r)
        assert no.activations_differ(fam, r, s_seq, s_exact, w)
    port, ref = port_slice(src, wtype, 64), oracle.RefSlice(src, 3, 64)
    try:
        for rows in (x, x[:1], x[1:2]):
            a, b = port.forward(rows), ref.forward(rows)
            assert np.isfinite(b).all()
            assert (a.view(np.uint32) == b.view(np.uint32)).all(), int((a.view(np.uint32) != b.view(np.uint32)).sum())
    finally:
        port.close()
        ref.close()


def _rows(kind: str, n: int, k: int, rng) -> np.ndarray:
    if kind == "gauss":
        return rng.standard_normal((n, k), dtype=np.float32)
    if kind == "outlier":
        x = rng.standard_normal((n, k), dtype=np.float32)
        for i, f in enumerate((1e3, 1e4, 1e5, 1e6)):
            x[i::4, rng.integers(0, k, 3)] *= np.float32(f)
        return x
    if kind == "huge":
        return ec.inputs("huge", n, k, rng)
    raise ValueError(kind)


def _tree_sums(t: np.ndarray) -> list:
    """Sums of each row of t in orders other than index order: numpy's pairwise sum, a 128-thread strided sum with a
    reduce tree (the plain prologue's shape), and per-32 block sums added as a tree."""
    out = [t.sum(axis=1)]
    n, k = t.shape
    if k % 128 == 0:
        s = t.reshape(n, k // 128, 128)
        part = np.zeros((n, 128))
        for j in range(k // 128):
            part = part + s[:, j, :]
        while part.shape[1] > 1:
            part = part[:, 0::2] + part[:, 1::2]
        out.append(part[:, 0])
    b = t.reshape(n, -1, 32).sum(axis=2)
    while b.shape[1] > 1:
        if b.shape[1] % 2:
            b = np.concatenate([b, np.zeros((n, 1))], axis=1)
        b = b[:, 0::2] + b[:, 1::2]
    out.append(b[:, 0])
    return out


def test_certification_is_sound():
    """Wherever the certified interval maps to one float, that float is the sequential sum's mean; it accepts almost
    every ordinary row and rejects the witness rows."""
    rng = np.random.default_rng(99)
    accepted = rejected = 0
    for k, n in ((256, 30000), (800, 20000), (4096, 4000)):
        for kind in ("gauss", "outlier", "huge"):
            x = _rows(kind, n, k, rng)
            t = no.squares(x)
            want = (no.sequential_sum(t) / k).astype(np.float32)
            for s in _tree_sums(t):
                m = no.certified_mean(s, k)
                ok = ~np.isnan(m)
                assert (m[ok].view(np.uint32) == want[ok].view(np.uint32)).all(), (k, kind)
                accepted += int(ok.sum())
                rejected += int((~ok).sum())
    for k in no.WIDTHS:
        for d in no.DIRECTIONS:
            for where in no.PLACES:
                x = no.witness_row(k, "q8_1", _norm_w(k), d, where)[None]
                t = no.squares(x)
                want = (no.sequential_sum(t) / k).astype(np.float32)
                for s in _tree_sums(t):
                    m = no.certified_mean(s, k)
                    assert np.isnan(m[0]) or m[0] == want[0]
                    rejected += int(np.isnan(m[0]))
    assert accepted > 0.99 * (accepted + rejected) and rejected > 0, (accepted, rejected)
