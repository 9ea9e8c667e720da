"""Q5_0 / Q5_1 on the CPU: the Python quantisers against the reference `quantize` tool, the benchmark writer's files,
and the C restatement (tests/q5_port.c on oracle/slice_oracle.c) against hidden states dumped from the compiled reference."""
import hashlib
import json
import os

import numpy as np
import pytest

from distributedllm_b200 import ggjt

GOLD = os.path.join(os.path.dirname(__file__), "golden")
Q5 = [ggjt.T_Q5_0, ggjt.T_Q5_1]


def _digests():
    return json.load(open(os.path.join(GOLD, "ref_digests_q5.json")))


def _digest(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


@pytest.mark.parametrize("wt", Q5, ids=["q5_0", "q5_1"])
def test_q5_quantizer_is_the_reference_quantize_tool(tmp_path, wt):
    """Every Q5 tensor `quantize <f32 model> <out> q5_x` writes for tiny3b (output.weight and tok_embeddings included:
    n_embd 800 is not a multiple of 256) is byte-identical to ggjt.quantize_q5_x of the same f32 tensor."""
    want = _digests()["quantize_" + ggjt.TYPE_NAME[wt]]
    sh = ggjt.SHAPES["tiny3b"]
    full = str(tmp_path / "f32.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=0)
    f = ggjt.read_file(full)
    assert "output.weight" in want and "tok_embeddings.weight" in want and len(want) == 2 + 7 * sh.n_layer
    quant = ggjt.quantize_q5_0 if wt == ggjt.T_Q5_0 else ggjt.quantize_q5_1
    for name, h in want.items():
        t = f.tensors[name]
        x = np.frombuffer(f.read_raw(name), np.float32).reshape(t.ne[1], t.ne[0])
        assert hashlib.sha256(quant(x).tobytes()).hexdigest() == h, name


@pytest.mark.parametrize("wt", Q5, ids=["q5_0", "q5_1"])
def test_q5_dequantize_round_trip(wt):
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((64, 256)) * rng.uniform(0.01, 10, (64, 1))).astype(np.float32)
    x[3] = 0.0                                             # all-zero blocks: d = 0, every weight decodes to (q - 16) * 0 or m
    x[5, :32] = 2.5                                        # constant block
    if wt == ggjt.T_Q5_0:
        b = ggjt.quantize_q5_0(x)
        y = ggjt.dequantize_q5_0(b)
        d = np.abs(b[..., 0:2].copy().view(np.float16).astype(np.float32))
        m = np.zeros_like(d)
        assert b.shape == (64, 8, 22)
    else:
        b = ggjt.quantize_q5_1(x)
        y = ggjt.dequantize_q5_1(b)
        d = b[..., 0:2].copy().view(np.float16).astype(np.float32)
        m = np.abs(b[..., 2:4].copy().view(np.float16).astype(np.float32))
        assert b.shape == (64, 8, 24) and (d >= 0).all()
    err = np.abs(y - x).reshape(64, 8, 32).max(axis=2)
    # half a step (a whole one for Q5_0: d = max / -16 maps the opposite extreme to 16.5, clamped to 15), plus the fp16
    # rounding of d (times |q| <= 32) and of m
    step = 1.0 if wt == ggjt.T_Q5_0 else 0.5
    bound = step * d * (1 + 2.0 ** -8) + 32 * d * 2.0 ** -11 + m * 2.0 ** -10 + 1e-7
    assert (err <= bound[..., 0]).all(), float((err - bound[..., 0]).max())
    assert (y[3] == 0).all()
    assert np.allclose(y[5, :32], 2.5, rtol=1e-3)


@pytest.mark.parametrize("wt", Q5, ids=["q5_0", "q5_1"])
def test_fast_q5_writer_files_are_valid_for_the_reference(tmp_path, wt):
    """bench.py's Q5 model files: the reference loads them and computes finite states; the recorded digests of its outputs
    are what the C restatement computes on the same file."""
    from q5_port import Q5PortSlice
    sh = ggjt.SHAPES["tiny128"]
    path = str(tmp_path / "fast.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 1, 0, wtype=wt)
    f = ggjt.read_file(path, sliced=True)
    assert all(t.ttype == wt for n, t in f.tensors.items() if not n.endswith("norm.weight"))
    port, rng = Q5PortSlice(path, 512), np.random.default_rng(11)
    got = []
    for n in (20, 1, 1):
        y = port.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32))
        assert np.isfinite(y).all()
        got.append(_digest(y))
    port.close()
    assert got == _digests()["fast_%s_writer" % ggjt.TYPE_NAME[wt]]


@pytest.mark.parametrize("wt", Q5, ids=["q5_0", "q5_1"])
def test_port_matches_q5_reference_goldens(tmp_path, wt):
    """tiny / tiny128 / tiny3b (n_ff 2144 = 67 blocks: odd block counts), prefill + decode schedules."""
    from q5_port import Q5PortSlice
    stem = "slices_" + ggjt.TYPE_NAME[wt]
    meta = json.load(open(os.path.join(GOLD, stem + ".json")))
    gold = np.load(os.path.join(GOLD, stem + ".npz"))
    assert sorted(v["shape"] for v in meta.values()) == ["tiny", "tiny128", "tiny3b"]
    for name, m in meta.items():
        path = str(tmp_path / (name + ".bin"))
        ggjt.write_synth_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], m["wtype"], seed=0)
        assert hashlib.sha256(open(path, "rb").read()).hexdigest() == m["file_sha256"], name
        port = Q5PortSlice(path, 512)
        for i in range(len(m["schedule"])):
            y = port.forward(gold["%s/x%d" % (name, i)])
            want = gold["%s/y%d" % (name, i)]
            assert (y.view(np.uint32) == want.view(np.uint32)).all(), (name, i)
        port.close()


def _fma32(a, b, c):
    """fmaf through float64: a*b of two floats is exact in float64, one rounding of the sum to float64 then float32."""
    return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def _f16(u):
    return float(np.array([u], np.uint16).view(np.float16)[0])


@pytest.mark.parametrize("wt", Q5, ids=["q5_0", "q5_1"])
def test_single_dot_over_an_odd_block_count(wt):
    """One row of 67 blocks: the reference's `assert(nb % 2 == 0)` is compiled out, so the lane chains simply run over
    every block.  orc_dot_q5_x against a scalar restatement of the AVX2 branch (lanes of 4, fma per block, hsum)."""
    import q5_port
    L = q5_port.lib()
    rng = np.random.default_rng(9)
    nb = 67
    k = nb * 32
    x = rng.standard_normal((1, k)).astype(np.float32)
    a = rng.standard_normal(k).astype(np.float32)
    w = (ggjt.quantize_q5_0 if wt == ggjt.T_Q5_0 else ggjt.quantize_q5_1)(x)[0]
    aq = np.empty(k, np.int8)
    q = ggjt._unpack_q5(w[None, :, 2:6] if wt == ggjt.T_Q5_0 else w[None, :, 4:8],
                        w[None, :, 6:] if wt == ggjt.T_Q5_0 else w[None, :, 8:])[0]
    acc = [np.float32(0)] * 8
    summs = np.float32(0)
    if wt == ggjt.T_Q5_0:
        ad = np.empty(nb, np.uint16)
        L.orc_quant_q8_0(a.ctypes.data, k, aq.ctypes.data, ad.ctypes.data)
        got = L.orc_dot_q5_0_q8_0(w.ctypes.data, aq.ctypes.data, ad.ctypes.data, k)
    else:
        ad, as_ = np.empty(nb, np.float32), np.empty(nb, np.float32)
        L.orc_quant_q8_1(a.ctypes.data, k, aq.ctypes.data, ad.ctypes.data, as_.ctypes.data)
        got = L.orc_dot_q5_1_q8_1(w.ctypes.data, aq.ctypes.data, ad.ctypes.data, as_.ctypes.data, k)
    for b in range(nb):
        dw = _f16(int(w[b, 0]) | (int(w[b, 1]) << 8))
        if wt == ggjt.T_Q5_0:
            d = np.float32(np.float32(dw) * np.float32(_f16(int(ad[b]))))
            vals = q[b].astype(np.int64) - 16
        else:
            d = np.float32(np.float32(dw) * ad[b])
            mw = _f16(int(w[b, 2]) | (int(w[b, 3]) << 8))
            summs = np.float32(summs + np.float32(np.float32(mw) * as_[b]))
            vals = q[b].astype(np.int64)
        for lane in range(8):
            s = int((vals[4 * lane:4 * lane + 4] * aq[b * 32 + 4 * lane:b * 32 + 4 * lane + 4].astype(np.int64)).sum())
            acc[lane] = _fma32(d, np.float32(s), acc[lane])
    r0, r1, r2, r3 = acc[4] + acc[0], acc[5] + acc[1], acc[6] + acc[2], acc[7] + acc[3]
    want = np.float32(np.float32(np.float32(r0 + r2) + np.float32(r1 + r3)) + summs)
    assert np.float32(got).view(np.uint32) == want.view(np.uint32), (got, want)
