"""LoRA merge on the host: the numpy twin (tests/lora_ref.py) against llama.cpp's merge, the ggla format, and the
binding's argument checks (no GPU)."""
from __future__ import annotations

import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import lora_ref
from distributedllm_b200 import capi, ggjt

HERE = os.path.dirname(os.path.abspath(__file__))
TOOL = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "lora_merge")
GOLD = json.load(open(os.path.join(HERE, "golden", "ref_digests_lora.json")))
CASES = lora_ref.cases() + lora_ref.edges()
TOOL_CASES = [c for c in CASES if c[1] in (1, 32, 40) or c in lora_ref.edges()]


@pytest.mark.parametrize("case", CASES, ids=[lora_ref.case_id(c) for c in CASES])
def test_twin_matches_golden_digests(case, tmp_path):
    m, a, b = lora_ref.write_case(str(tmp_path), case)
    out = str(tmp_path / "twin.bin")
    lora_ref.merge_file(m, out, a, b)
    f = ggjt.read_file(out, sliced=False)
    got = {n: hashlib.sha256(f.read_raw(n)).hexdigest() for n in f.tensors if n.startswith("layers.")}
    assert got == GOLD[lora_ref.case_id(case)]


@pytest.mark.skipif(not os.path.isfile(TOOL), reason="oracle/_ref/lora_merge not built")
@pytest.mark.parametrize("case", TOOL_CASES, ids=[lora_ref.case_id(c) for c in TOOL_CASES])
def test_twin_matches_llama_cpp_byte_for_byte(case, tmp_path):
    m, a, b = lora_ref.write_case(str(tmp_path), case)
    ref, twin = str(tmp_path / "ref.bin"), str(tmp_path / "twin.bin")
    subprocess.run([TOOL, m, a, b or "-", ref, "2"], check=True, capture_output=True)
    lora_ref.merge_file(m, twin, a, b)
    assert open(ref, "rb").read() == open(twin, "rb").read()


def test_cases_hit_ties_and_zero_blocks(tmp_path):
    """The F32-base cases put Q8_0 values half-way between integers and Q4_0 values on x*id + 8.5 integers."""
    x = lora_ref._matrix(np.random.default_rng(0), 4, 64)
    assert not x[0].any()
    q8 = np.frombuffer(lora_ref.quantize(x[2:3], ggjt.T_Q8_0), np.uint8).reshape(2, 34)
    q = q8[0, 2:].view(np.int8)
    assert q[0] == 127 and q[1] == -30 and q[2] == -30     # -30.5 and -29.5: half to even (roundf gives -31, -30)
    assert lora_ref.quantize(x[0:1], ggjt.T_Q4_0)[:2] == np.float16(-0.0).tobytes()


def test_edge_cases_cover_the_rank_paths_and_scales():
    e = lora_ref.edges()
    for fam in lora_ref.FAMILIES:
        ranks = {c[1] for c in e if c[0] == fam and len(c) == 4}
        assert set(lora_ref.EDGE_RANKS) <= ranks
        for c in e:                                     # the rank sweep's scales are not powers of two
            if c[0] == fam and c[1] in lora_ref.EDGE_RANKS and c[2] == 2 * c[1] + 1:
                s = np.float32(c[2]) / np.float32(c[1])
                assert np.frexp(s)[0] != 0.5
        for r in (8, 64):
            alphas = {c[2] for c in lora_ref.cases() + e if c[0] == fam and c[1] == r and c[3] is None and len(c) == 4}
            assert {1, r + 3, 3 * r, 0, -r, -(r + 3)} <= alphas
    # one job of stacked sources with two ranks (wq | wk | wv and w1 | w3), none equal to the header's r = 16 there
    assert lora_ref.MIXED_RANKS["attention.wq.weight"] != lora_ref.MIXED_RANKS["attention.wk.weight"]
    assert lora_ref.MIXED_RANKS["feed_forward.w1.weight"] != lora_ref.MIXED_RANKS["feed_forward.w3.weight"]
    assert {8, 16, 40, 64} == set(lora_ref.MIXED_RANKS.values())


def _signs(x):
    return np.signbit(np.asarray(x, np.float32))


@pytest.mark.parametrize("fam", list(lora_ref.FAMILIES))
def test_designed_blocks_reach_their_edges(fam):
    """Each designed block of the "designed" cases sits on its edge once base + BA is formed: a check of the values the
    merge quantises, so a block that misses its edge fails here rather than checking nothing."""
    F = np.float32
    base, A, B, target, place = lora_ref.designed_matrix(fam)
    d = lora_ref.ba(A, B, -4, 2)
    assert np.array_equal(A, np.exp2(np.round(np.log2(np.abs(A)))) * np.sign(A))      # powers of two
    nz = B != 0
    assert np.array_equal(B[nz], (np.exp2(np.round(np.log2(np.abs(B[nz])))) * np.sign(B[nz])).astype(F))
    blk = {n: target[j, 32 * b:32 * b + 32] for n, (j, b) in place.items()}
    bas = {n: base[j, 32 * b:32 * b + 32] for n, (j, b) in place.items()}
    ba_ = {n: d[j, 32 * b:32 * b + 32] for n, (j, b) in place.items()}
    for n in blk:
        assert np.array_equal((bas[n] + ba_[n]).astype(F).view(np.uint32), blk[n].view(np.uint32)), n
        if n.startswith("z_"):
            assert np.all((ba_[n] == 0) & _signs(ba_[n])), n                       # BA == -0 (negative scale)
        else:
            assert np.all(ba_[n] != 0), n                                          # the edge is made by adding BA
    z = blk["zero_from_base"]
    assert np.all(z == 0) and not _signs(z).any() and np.all(bas["zero_from_base"] != 0)
    wtype = lora_ref.FAMILIES[fam]
    if wtype == ggjt.T_Q8_0:
        for n in ("half", "half_id2"):
            x = blk[n]
            amax = np.abs(x).max()
            p = (x * (F(127) / amax)).astype(F)
            ties = (p - np.floor(p)) == 0.5
            away = np.sign(p) * np.floor(np.abs(p) + 0.5)
            assert ties.sum() >= 16 and (np.rint(p) != away).sum() >= 8, n       # half to even differs from roundf
    elif wtype in (ggjt.T_Q4_0, ggjt.T_Q5_0):
        half = F(8 if wtype == ggjt.T_Q4_0 else 16)
        for n, first in (("pm_tie", 1), ("mp_tie", -1)):
            a = np.abs(blk[n])
            top = np.flatnonzero(a == a.max())
            assert len(top) == 2 and np.sign(blk[n][top[0]]) == first and np.sign(blk[n][top[1]]) == -first, n
        x = blk["on_int"]
        mx = x[np.argmax(np.abs(x))]
        idv = F(1) / F(mx / -half)
        v = ((x * idv).astype(F) + (half + F(0.5))).astype(F)
        assert (v == np.trunc(v)).sum() == 31 and mx == -half                       # all but the max itself
    elif wtype in (ggjt.T_Q4_1, ggjt.T_Q5_1):
        div = F(15 if wtype == ggjt.T_Q4_1 else 31)
        x = blk["min_eq_max"]
        assert x.min() == x.max() != 0
        x = blk["on_int"]
        idv = F(1) / F((x.max() - x.min()) / div)
        v = (((x - x.min()).astype(F) * idv).astype(F) + F(0.5)).astype(F)
        assert (v == np.trunc(v)).sum() == 30                                       # all but min and max
        x = blk["fma_split"]
        m, idv = x.min(), F(1) / F((x.max() - x.min()) / div)
        two = np.trunc((((x - m).astype(F) * idv).astype(F) + F(0.5)).astype(F))
        one = np.trunc(lora_ref._fma((x - m).astype(F), np.full(32, idv, F), np.full(32, F(0.5), F)))
        assert (two != one).sum() == 1                                              # one product rounded, or not
        x = blk["z_zero_tie"]                                                       # minimum: +0 first, -0 later
        zi = np.flatnonzero(x == 0)
        assert x.min() == 0 and len(zi) == 2 and not _signs(x[zi[0]]) and _signs(x[zi[1]])
        x = blk["z_all_zero_signs"]
        assert np.all(x == 0) and not _signs(x[0]) and _signs(x[31])
    else:
        x = blk["ties"]
        h = x.astype(np.float16)
        toward = np.where(h.astype(F) > x, np.float16(-np.inf), np.float16(np.inf)).astype(np.float16)
        other = np.nextafter(h, toward)                                             # the fp16 neighbour across x
        assert np.array_equal(h.astype(np.float64) + other.astype(np.float64), 2 * x.astype(np.float64))   # half-way
        up = np.abs(h.astype(F)) > np.abs(x)                                        # half to even, away from zero
        assert up.sum() >= 8 and (~up).sum() >= 8
        x = blk["subnormal"]
        h = x.astype(np.float16)
        sub = (h != 0) & (np.abs(h) < np.float16(2.0 ** -14))
        assert sub.sum() >= 20
        assert (h == 0).any() and _signs(h.astype(F)[x < 0]).all()                  # -2^-25 rounds to -0
        x = blk["z_signed_zero"]
        assert np.all(x == 0) and _signs(x).sum() == 16


def test_designed_cases_merge_their_edge_blocks():
    """The twin's merged wq of a designed case is the quantised target: BA is exact, so the file holds exactly the
    designed blocks' requantisation."""
    for fam, wtype in lora_ref.FAMILIES.items():
        base, A, B, target, place = lora_ref.designed_matrix(fam)
        raw = lora_ref.merge_tensor(b"", wtype, 64, 64, A, B, -4, 2, base.tobytes(), ggjt.T_F32)
        assert raw == lora_ref.quantize(target, wtype), fam


def test_zero_b_rows_give_plus_zero():
    """A row of loraB that is zero gives BA == +0 in every column at every rank path, and -0 under a negative scale:
    the large-shape GPU tests compute BA only on the rows where loraB is nonzero."""
    rng = np.random.default_rng(3)
    for r in (1, 31, 32, 33, 64, 65, 308):
        A = rng.standard_normal((96, r), dtype=np.float32)
        B = rng.standard_normal((4, r), dtype=np.float32)
        B[1] = 0
        for alpha, neg in ((r, False), (2 * r + 1, False), (0, False), (-r - 3, True)):
            z = lora_ref.ba(A, B, alpha, r)[1]
            assert np.all(z == 0) and np.all(np.signbit(z) == neg), (r, alpha)


def test_fma_is_exact():
    rng = np.random.default_rng(1)
    a, b, c = (rng.standard_normal(100000).astype(np.float32) for _ in range(3))
    from fractions import Fraction
    got = lora_ref._fma(a, b, c)
    for i in range(0, 100000, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.array(v).view(np.uint32)) & 1))
        assert got[i] == best


def test_ggla_round_trip(tmp_path):
    rng = np.random.default_rng(2)
    ts = [("layers.3.attention.wq.weight.loraA", rng.standard_normal((64, 8), dtype=np.float32)),
          ("layers.3.attention.wq.weight.loraB", rng.standard_normal((64, 8), dtype=np.float32)),
          ("layers.3.attention.wv.weight.loraA", rng.standard_normal((64, 5)).astype(np.float16))]
    p = str(tmp_path / "a.bin")
    ggjt.write_lora(p, 8, 16, ts)
    r, alpha, got = ggjt.read_lora(p)
    assert (r, alpha) == (8, 16) and list(got) == [n for n, _ in ts]
    for n, a in ts:
        assert got[n].dtype == a.dtype and np.array_equal(got[n], a)
    raw = open(p, "rb").read()
    assert raw[:4] == b"algg" and raw[16:20] == (2).to_bytes(4, "little")
    assert raw[16 + 12:16 + 20] == (8).to_bytes(4, "little") + (64).to_bytes(4, "little")   # ne = shape reversed


def test_capi_lora_argument_checks():
    with pytest.raises(ValueError, match="lora_base needs lora"):
        capi.Slice("x.bin", 0, 0, lora=None, lora_base="b.bin")


def test_capi_calls_the_lora_entry_only_with_an_adapter(monkeypatch):
    calls = []

    class Fake:
        def b200_slice_load_ex(self, *a):
            calls.append(("ex", a[0]))
            return 2

        def b200_slice_load_lora(self, *a):
            calls.append(("lora", a[0], a[4], a[5]))
            return 2

        def b200_last_error(self):
            return b"refused"

    monkeypatch.setattr(capi, "lib", lambda: Fake())
    for kw in ({}, {"lora": "a.bin"}, {"lora": "a.bin", "lora_base": "b.bin"}):
        with pytest.raises(capi.B200Error):
            capi.Slice("s.bin", 0, 0, **kw)
    assert calls == [("ex", b"s.bin"), ("lora", b"s.bin", b"a.bin", None), ("lora", b"s.bin", b"a.bin", b"b.bin")]
