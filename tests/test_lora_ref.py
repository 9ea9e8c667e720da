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
CASES = lora_ref.cases()


@pytest.mark.parametrize("case", CASES, ids=[lora_ref.case_id(c) for c in CASES])
def test_twin_matches_golden_digests(case, tmp_path):
    m, a, b = lora_ref.write_case(str(tmp_path), case)
    out = str(tmp_path / "twin.bin")
    lora_ref.merge_file(m, out, a, b)
    f = ggjt.read_file(out, sliced=False)
    got = {n: hashlib.sha256(f.read_raw(n)).hexdigest() for n in f.tensors if n.startswith("layers.")}
    assert got == GOLD[lora_ref.case_id(case)]


@pytest.mark.skipif(not os.path.isfile(TOOL), reason="oracle/_ref/lora_merge not built")
@pytest.mark.parametrize("case", [c for c in CASES if c[1] in (1, 32, 40)],
                         ids=[lora_ref.case_id(c) for c in CASES if c[1] in (1, 32, 40)])
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
