"""b200_slice_load_lora on the GPU: a slice loaded with an adapter gives the same bits as the slice merged on the host
(tests/lora_ref.py, which equals llama.cpp's merge byte for byte) loaded plainly, in every kind of call."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lora_ref
from distributedllm_b200 import capi, ggjt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "oracle", "_ref", "lora_merge")
FAMS = {"q4_0": ggjt.T_Q4_0, "q4_1": ggjt.T_Q4_1, "q5_0": ggjt.T_Q5_0, "q5_1": ggjt.T_Q5_1, "q8_0": ggjt.T_Q8_0,
        "f16": ggjt.T_F16}


def adapter_for(slice_path: str, out: str, r: int, alpha: int, mats=lora_ref.MATS, layers=None, seed: int = 0,
                extra=()) -> str:
    f = ggjt.read_file(slice_path)
    rng = np.random.default_rng([seed, r])
    ts = []
    for name, t in f.tensors.items():
        layer = int(name.split(".")[1])
        if not name.endswith(tuple(mats)) or (layers is not None and layer not in layers):
            continue
        k, rows = t.ne
        ts.append((name + ".loraA", (rng.standard_normal((k, r), dtype=np.float32) * np.float32(0.05)).astype(np.float32)))
        ts.append((name + ".loraB", (rng.standard_normal((rows, r), dtype=np.float32) * np.float32(0.05)).astype(np.float32)))
    ggjt.write_lora(out, r, alpha, list(ts) + list(extra))
    return out


def bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_same_calls(a: capi.Slice, b: capi.Slice, E: int, seed: int = 0) -> None:
    """prompt call, single-token steps, a batched step of two sessions, a mixed pass"""
    rng = np.random.default_rng(seed)
    x = lambda n: rng.standard_normal((n, E), dtype=np.float32)   # noqa: E731
    for fn, args in ((lambda s, v: s.session_forward(0, v), (x(7),)), (lambda s, v: s.session_forward(0, v), (x(1),)),
                     (lambda s, v: s.session_forward(0, v), (x(1),)), (lambda s, v: s.session_forward(1, v), (x(3),)),
                     (lambda s, v: s.batch_forward([0, 1], v), (x(2),)),
                     (lambda s, v: s.mixed_forward([0, 1], [4, 1], v), (x(5),))):
        ga, gb = fn(a, *args), fn(b, *args)
        assert np.array_equal(bits(ga), bits(gb))


def load_pair(plain_path, lora_path, merged_path, base=None, n_ctx=128):
    a = capi.Slice(plain_path, 0, n_ctx, n_sessions=2, lora=lora_path, lora_base=base)
    b = capi.Slice(merged_path, 0, n_ctx, n_sessions=2)
    return a, b


@pytest.mark.parametrize("shape", ["tiny", "tiny128"])
@pytest.mark.parametrize("fam", list(FAMS))
@pytest.mark.parametrize("r,alpha", [(16, 32), (40, 40)])
def test_adapted_slice_equals_merged_slice(tmp_path, shape, fam, r, alpha):
    sh = ggjt.SHAPES[shape]
    p = str(tmp_path / "s.bin")
    ggjt.write_synth_slice(p, sh, 0, 1, FAMS[fam], seed=3)
    ad = adapter_for(p, str(tmp_path / "a.bin"), r, alpha)
    m = str(tmp_path / "m.bin")
    lora_ref.merge_file(p, m, ad)
    a, b = load_pair(p, ad, m)
    try:
        assert_same_calls(a, b, sh.n_embd)
    finally:
        a.close(), b.close()


def test_llama7b_layer_rank16_all_seven(tmp_path):
    sh = ggjt.SHAPES["7b"]
    p = str(tmp_path / "s.bin")
    ggjt.write_fast_q4_slice(p, sh, 0, 0, seed=1)
    ad = adapter_for(p, str(tmp_path / "a.bin"), 16, 32)
    m = str(tmp_path / "m.bin")
    lora_ref.merge_file(p, m, ad)
    a, b = load_pair(p, ad, m, n_ctx=256)
    try:
        assert_same_calls(a, b, sh.n_embd)
    finally:
        a.close(), b.close()


@pytest.mark.parametrize("btype", [ggjt.T_F16, ggjt.T_F32])
@pytest.mark.parametrize("fam", ["q4_0", "q8_0", "f16"])
def test_lora_base(tmp_path, fam, btype):
    sh = ggjt.SHAPES["tiny"]
    p, bp = str(tmp_path / "s.bin"), str(tmp_path / "base.bin")
    ggjt.write_synth_slice(p, sh, 0, 1, FAMS[fam], seed=3)
    ggjt.write_synth_slice(bp, sh, 0, 1, btype, seed=4)
    ad = adapter_for(p, str(tmp_path / "a.bin"), 8, 16, mats=lora_ref.MATS[:2] + lora_ref.MATS[4:6])
    m = str(tmp_path / "m.bin")
    lora_ref.merge_file(p, m, ad, bp)
    a, b = load_pair(p, ad, m, base=bp)
    try:
        assert_same_calls(a, b, sh.n_embd)
    finally:
        a.close(), b.close()


def _four_layer_model(d, wtype=ggjt.T_Q4_0):
    sh = ggjt.SHAPES["tiny"]
    full = os.path.join(d, "full.bin")
    ggjt.write_synth_full(full, sh, wtype, seed=5)
    return sh, full


def test_two_slices_one_adapter_and_greedy_ids(tmp_path):
    d = str(tmp_path)
    sh, full = _four_layer_model(d)
    ad = str(tmp_path / "a.bin")
    # rank 8 on wq / wv of every layer, written against the full model
    f = ggjt.read_file(full, sliced=False)
    rng = np.random.default_rng(9)
    ts = []
    for name, t in f.tensors.items():
        if name.endswith(("wq.weight", "wv.weight")):
            k, rows = t.ne
            ts += [(name + ".loraA", rng.standard_normal((k, 8), dtype=np.float32) * np.float32(0.05)),
                   (name + ".loraB", rng.standard_normal((rows, 8), dtype=np.float32) * np.float32(0.05))]
    ggjt.write_lora(ad, 8, 16, [(n, a.astype(np.float32)) for n, a in ts])
    merged = str(tmp_path / "merged_full.bin")
    lora_ref.merge_file(full, merged, ad)
    paths, mpaths = [], []
    for lo, hi in ((0, 1), (2, 3)):
        sp, mp = str(tmp_path / ("s%d.bin" % lo)), str(tmp_path / ("m%d.bin" % lo))
        ggjt.slice_model(full, sp, lo, hi)
        ggjt.slice_model(merged, mp, lo, hi)
        paths.append(sp), mpaths.append(mp)
    for sp, mp in zip(paths, mpaths):
        a, b = load_pair(sp, ad, mp)
        try:
            assert_same_calls(a, b, sh.n_embd)
        finally:
            a.close(), b.close()
    extra = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra, sh, ggjt.T_Q4_0, seed=5)
    from distributedllm_b200.client import LocalPipeline
    ids = []
    for kw, ps in (({"lora": ad}, paths), ({}, mpaths)):
        lp = LocalPipeline(ps, devices=[0, 0], n_ctx=128, **kw)
        ex = capi.Extra(extra, 0)
        try:
            ids.append(capi.generate_greedy(lp.slices, ex, [0], [[1, 17, 33, 5]], 12))
        finally:
            ex.close()
            for s in lp.slices:
                s.close()
    assert np.array_equal(ids[0], ids[1])


def test_adapter_that_misses_the_slice_loads_as_plain(tmp_path):
    sh = ggjt.SHAPES["tiny"]
    p, other = str(tmp_path / "s.bin"), str(tmp_path / "o.bin")
    ggjt.write_synth_slice(p, sh, 0, 1, ggjt.T_Q4_0, seed=3)
    ggjt.write_synth_slice(other, sh, 2, 3, ggjt.T_Q4_0, seed=3)
    ad = adapter_for(other, str(tmp_path / "a.bin"), 8, 16)
    a, b = load_pair(p, ad, p)
    try:
        assert_same_calls(a, b, sh.n_embd)
    finally:
        a.close(), b.close()


@pytest.mark.skipif(not os.path.isfile(TOOL), reason="oracle/_ref/lora_merge not built")
@pytest.mark.parametrize("fam", ["q4_0", "q8_0", "f16"])
def test_against_llama_cpp_merge_and_reference_path(tmp_path, fam):
    """llama.cpp merges the full model; its slice equals the host twin's file, and the adapted slice's hidden states
    equal both the GPU plain load of it and the reference CPU path on it."""
    from oracle import oracle
    d = str(tmp_path)
    sh, full = _four_layer_model(d, FAMS[fam])
    f = ggjt.read_file(full, sliced=False)
    rng = np.random.default_rng(11)
    ts = []
    for name, t in f.tensors.items():
        if name.startswith("layers.") and not name.endswith("norm.weight"):
            k, rows = t.ne
            ts += [(name + ".loraA", (rng.standard_normal((k, 16), dtype=np.float32) * np.float32(0.05)).astype(np.float32)),
                   (name + ".loraB", (rng.standard_normal((rows, 16), dtype=np.float32) * np.float32(0.05)).astype(np.float32))]
    ad = str(tmp_path / "a.bin")
    ggjt.write_lora(ad, 16, 32, ts)
    ref_full = str(tmp_path / "ref_full.bin")
    subprocess.run([TOOL, full, ad, "-", ref_full, "4"], check=True, capture_output=True)
    sp, rp, tp = str(tmp_path / "s.bin"), str(tmp_path / "r.bin"), str(tmp_path / "t.bin")
    ggjt.slice_model(full, sp, 0, 1)
    ggjt.slice_model(ref_full, rp, 0, 1)
    lora_ref.merge_file(sp, tp, ad)
    assert open(rp, "rb").read() == open(tp, "rb").read()
    a, b = load_pair(sp, ad, rp)
    try:
        assert_same_calls(a, b, sh.n_embd)
        if oracle.have_ref():
            ref = oracle.RefSlice(rp, n_threads=4, n_ctx=128)
            a.clear_context()
            x = np.random.default_rng(1).standard_normal((6, sh.n_embd), dtype=np.float32)
            for part in (x[:5], x[5:]):
                assert np.array_equal(bits(a.forward(part)), bits(ref.forward(part)))
            ref.close()
    finally:
        a.close(), b.close()


# ----------------------------------------------------------------------------------------------- refusals
def _raw_load(path, lora, base=None):
    h = C.c_void_p(12345)
    rc = capi.lib().b200_slice_load_lora(os.fsencode(path), 0, 128, 1, os.fsencode(lora),
                                         None if base is None else os.fsencode(base), C.byref(h))
    return rc, h.value, capi.lib().b200_last_error().decode()


def test_refusals_name_the_tensor_and_leave_nothing(tmp_path):
    import torch
    sh = ggjt.SHAPES["tiny"]
    p = str(tmp_path / "s.bin")
    ggjt.write_synth_slice(p, sh, 0, 1, ggjt.T_Q4_0, seed=3)
    E, FF = sh.n_embd, sh.n_ff
    wq = "layers.0.attention.wq.weight"
    A = lambda k, r=4: np.zeros((k, r), np.float32)          # noqa: E731
    good = [(wq + ".loraA", A(E)), (wq + ".loraB", A(E))]
    cases = []

    def add(what, name, tensors, r=4, alpha=8, base=None, **kw):
        fp = str(tmp_path / ("bad%d.bin" % len(cases)))
        ggjt.write_lora(fp, r, alpha, tensors, **kw)
        cases.append((what, name, fp, base))
        return fp

    add("magic", "magic", good, magic=0x12345678)
    add("version", "version", good, version=2)
    add("rank", "rank", good, r=0)
    tp = add("truncated", wq + ".loraB", good)
    with open(tp, "r+b") as f:
        f.truncate(os.path.getsize(tp) - 8)
    add("suffix", wq + ".lora", [(wq + ".lora", A(E))])
    add("not a layer matrix", "output.weight.loraA", [("output.weight.loraA", A(E))])
    add("not a layer matrix", "layers.0.attention_norm.weight.loraA", [("layers.0.attention_norm.weight.loraA", A(E))])
    add("3-D", wq + ".loraA", [(wq + ".loraA", np.zeros((2, E, 4), np.float32))])
    add("F16", wq + ".loraA", [(wq + ".loraA", A(E).astype(np.float16)), (wq + ".loraB", A(E))])
    add("rank mismatch", wq, [(wq + ".loraA", A(E, 8)), (wq + ".loraB", A(E, 4))])
    add("rank 1025", wq, [(wq + ".loraA", A(E, 1025)), (wq + ".loraB", A(E, 1025))], r=1025)
    add("shape", wq, [(wq + ".loraA", A(E + 32)), (wq + ".loraB", A(E))])
    add("shape", "layers.0.feed_forward.w2.weight", [("layers.0.feed_forward.w2.weight.loraA", A(E)),
                                                      ("layers.0.feed_forward.w2.weight.loraB", A(E))])
    add("lone A", wq, [(wq + ".loraA", A(E))])
    add("lone B", "layers.1.attention.wo.weight", good + [("layers.1.attention.wo.weight.loraB", A(E))])
    nobase = str(tmp_path / "nb.bin")
    ggjt.write_synth_slice(nobase, ggjt.SHAPES["tiny"], 2, 3, ggjt.T_F16, seed=0)
    add("base lacks", wq, good, base=nobase)
    wrong = str(tmp_path / "wrong.bin")
    ggjt.write_synth_slice(wrong, ggjt.SHAPES["tiny128"], 0, 1, ggjt.T_F16, seed=0)
    add("base shape", wq, good, base=wrong)
    qbase = str(tmp_path / "qb.bin")
    ggjt.write_synth_slice(qbase, sh, 0, 1, ggjt.T_Q8_0, seed=0)
    add("base type", wq, good, base=qbase)
    # a k-quant slice's matrix
    kp = str(tmp_path / "k.bin")
    ggjt.write_kquant_slice(kp, ggjt.SHAPES["tinyk"], 0, 0, mix="q4_K_M")
    ek = ggjt.SHAPES["tinyk"].n_embd
    kfile = str(tmp_path / "kq.bin")
    ggjt.write_lora(kfile, 4, 8, [(wq + ".loraA", A(ek)), (wq + ".loraB", A(ek))])

    gp = str(tmp_path / "good.bin")
    ggjt.write_lora(gp, 4, 8, good)
    capi.Slice(p, 0, 128, lora=gp).close()               # the first load brings in the library's modules
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    seen = []
    for what, name, fp, base in cases:
        rc, h, msg = _raw_load(p, fp, base)
        assert rc == 2, (what, rc, msg)
        assert h is None, what
        assert name in msg, (what, msg)
        seen.append(what)
    rc, h, msg = _raw_load(kp, kfile)
    assert rc == 2 and h is None and wq in msg and "k-quant" in msg, msg
    rc, h, msg = _raw_load(p, str(tmp_path / "missing.bin"))
    assert rc == 2 and h is None
    h = C.c_void_p()
    assert capi.lib().b200_slice_load_lora(os.fsencode(p), 0, 128, 1, None, os.fsencode(qbase), C.byref(h)) == 1
    free1 = torch.cuda.mem_get_info(0)[0]
    assert abs(free1 - free0) <= 2 << 20, (free0, free1)
    capi.Slice(p, 0, 128, lora=gp).close()               # a good adapter still loads after all of them
