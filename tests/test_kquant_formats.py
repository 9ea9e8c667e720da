"""CPU: k-quant (Q4_K / Q6_K) files -- the GGJT reader and writer, the per-tensor types of the reference's `quantize`, and
the C restatement (tests/kq_port.c) against goldens dumped from the reference and, where oracle/_ref is built, against the
reference itself."""
import hashlib
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from distributedllm_b200 import ggjt

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
have_ref = os.path.isfile(os.path.join(REF_DIR, "libllmref.so")) and os.path.isfile(os.path.join(REF_DIR, "quantize"))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("wtype", [ggjt.T_Q4_K, ggjt.T_Q6_K], ids=["q4_K", "q6_K"])
def test_kquant_tensor_round_trip(tmp_path, wtype):
    """A Q4_K / Q6_K tensor is written, indexed and read back byte for byte; the numpy and C dequantisers agree."""
    from kq_port import lib
    rows, k = 16, 512
    bsz = ggjt.TYPE_BLOCK[wtype][1]
    blocks = ggjt._kquant_pool(3, k, wtype, rows * k // 256)
    raw = blocks.tobytes()
    assert ggjt.tensor_nbytes((k, rows), wtype) == len(raw)
    path = str(tmp_path / "t.bin")
    hp = ggjt.HParams(8, 256, 256, 4, 0, 64, ggjt.FTYPE_Q4_K_M, ggjt.NO_FIRST_LAYER)
    ggjt.write_file(path, hp, ggjt.default_vocab(8), [("m.weight", wtype, (k, rows), raw), ("v", ggjt.T_F32, (4,), bytes(16))])
    f = ggjt.read_file(path)
    t = f.tensors["m.weight"]
    assert (t.ttype, t.ne, t.nbytes) == (wtype, (k, rows), len(raw)) and t.offset % 32 == 0
    assert f.read_raw("m.weight") == raw
    b3 = np.frombuffer(raw, np.uint8).reshape(rows, k // 256, bsz)
    w = ggjt.dequantize_q4_K(b3) if wtype == ggjt.T_Q4_K else ggjt.dequantize_q6_K(b3)
    assert w.shape == (rows, k) and np.isfinite(w).all()
    assert 0.5 / np.sqrt(k) < w.std() < 2.0 / np.sqrt(k)          # the writer's blocks are well scaled
    if wtype == ggjt.T_Q4_K:
        c = np.empty(k, np.float32)
        for r in range(rows):
            row = np.ascontiguousarray(b3[r])
            lib().orc_dequant_q4_K(row.ctypes.data, k, c.ctypes.data)
            assert (_bits(c) == _bits(w[r])).all(), r


def test_writer_types_equal_reference_quantize():
    """ggjt.kquant_tensor_type against the type map the reference `quantize` wrote (tests/golden/ref_kquant_types.json),
    for 8- and 32-layer models; a slice keeps the types of the full model (use_more_bits sees the full layer count)."""
    g = json.load(open(os.path.join(GOLD, "ref_kquant_types.json")))
    assert len(g["types"]) == 12
    for key, types in g["types"].items():
        label, mix, what = key.split("/")
        n_layer = g["n_layer"][label]
        for name, tname in types.items():
            if tname == "f32":
                assert name.endswith("norm.weight") or name == "norm.weight", name
                continue
            assert ggjt.TYPE_NAME[ggjt.kquant_tensor_type(name, mix, n_layer)] == tname, (key, name)
        if what.startswith("slice") and mix == "q4_K_M":
            kept = {n for n, t in types.items() if t == "q6_K"}
            assert kept == {"layers.%d.%s" % (i, m) for i in (2, 3, 4) if ggjt.use_more_bits(i, n_layer)
                            for m in ("attention.wv.weight", "feed_forward.w2.weight")}, key
    # the writer applies the same map (layers 2-4 of tinyk: layer 3's wv / w2 are Q6_K in Q4_K_M)
    assert [ggjt.use_more_bits(i, 8) for i in range(8)] == [True, False, False, True, False, False, True, True]


def test_writer_files_carry_the_tool_types(tmp_path):
    path = str(tmp_path / "s.bin")
    sh = ggjt.SHAPES["tinyk"]
    for mix in ggjt.KQUANT_MIXES:
        ggjt.write_kquant_slice(path, sh, 2, 4, mix, seed=0)
        f = ggjt.read_file(path)
        assert f.hparams.ftype == ggjt.KQUANT_MIXES[mix] and f.hparams.first_layer == 2
        for name, t in f.tensors.items():
            want = ggjt.T_F32 if name.endswith("norm.weight") else ggjt.kquant_tensor_type(name, mix, sh.n_layer)
            assert t.ttype == want, (mix, name)
    a = open(path, "rb").read()
    ggjt.write_kquant_slice(path, sh, 2, 4, "q6_K", seed=0)
    assert open(path, "rb").read() == a                       # deterministic


def test_port_matches_reference_goldens(tmp_path):
    """The C restatement against hidden states dumped from the reference (all three mixes, both tiny shapes)."""
    from kq_port import KQPortSlice
    meta = json.load(open(os.path.join(GOLD, "slices_kquant.json")))
    gold = np.load(os.path.join(GOLD, "slices_kquant.npz"))
    for name, m in meta.items():
        path = str(tmp_path / (name + ".bin"))
        ggjt.write_kquant_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], m["mix"], seed=0)
        assert hashlib.sha256(open(path, "rb").read()).hexdigest() == m["file_sha256"], name
        port = KQPortSlice(path, 512)
        for i in range(len(m["schedule"])):
            y = port.forward(gold["%s/x%d" % (name, i)])
            assert (_bits(y) == _bits(gold["%s/y%d" % (name, i)])).all(), (name, i)
        port.close()


def test_port_extra_layers_match_reference_goldens(tmp_path):
    from kq_port import KQPortExtra
    g = np.load(os.path.join(GOLD, "extra_kquant.npz"))
    sh = ggjt.SHAPES["tinyk128"]
    path = str(tmp_path / "e.bin")
    ggjt.write_kquant_extra(path, sh, "q4_K_M", seed=0)
    ex = KQPortExtra(path)
    assert (_bits(ex.embed(g["tokens"].tolist())) == _bits(g["emb"])).all()
    assert (_bits(ex.logits(g["hidden"])) == _bits(g["logits_all"])).all()


@pytest.mark.skipif(not have_ref, reason="oracle/_ref not built")
@pytest.mark.parametrize("mix", sorted(ggjt.KQUANT_MIXES))
def test_port_matches_reference_live(tmp_path, mix):
    """Live: the reference quantises a seeded F32 tinyk128 model itself (`quantize <mix>`, `slice_model` layers 2-4), and
    the C restatement reproduces its hidden states bit for bit."""
    from kq_port import KQPortSlice
    from oracle import oracle
    sh = ggjt.SHAPES["tinyk128"]
    full, q, sl = str(tmp_path / "f32.bin"), str(tmp_path / "q.bin"), str(tmp_path / "s.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=5)
    subprocess.run([os.path.join(REF_DIR, "quantize"), full, q, mix], check=True, capture_output=True)
    subprocess.run([os.path.join(REF_DIR, "slice_model"), "slice", q, "2", "4", sl], check=True, capture_output=True)
    ref, port = oracle.RefSlice(sl, 3, 128), KQPortSlice(sl, 128)
    rng = np.random.default_rng(2)
    try:
        for n in (12, 1, 1, 5):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            assert (_bits(ref.forward(x)) == _bits(port.forward(x))).all(), n
    finally:
        ref.close()
        port.close()


def _write_one_tensor_file(path, ttype, nbytes):
    hp = ggjt.HParams(8, 256, 256, 4, 1, 64, ggjt.FTYPE_Q4_K_M, 0)
    with open(path, "wb") as f:
        ggjt._write_header(f, hp, ggjt.default_vocab(8))
        name = b"layers.0.feed_forward.w2.weight"
        f.write(struct.pack("<III", 2, len(name), ttype))
        f.write(struct.pack("<2I", 256, 256))
        f.write(name)
        f.write(b"\0" * ((-f.tell()) & 31))
        f.write(bytes(nbytes))


@pytest.mark.parametrize("ttype,name,bsz", [(13, "q5_K", 176), (11, "q3_K", 110), (10, "q2_K", 84)])
def test_unsupported_k_types_are_refused_by_name(tmp_path, ttype, name, bsz):
    path = str(tmp_path / "k.bin")
    _write_one_tensor_file(path, ttype, 256 * bsz)
    with pytest.raises(ValueError) as ei:
        ggjt.read_file(path, sliced=True)
    msg = str(ei.value)
    assert name in msg and "layers.0.feed_forward.w2.weight" in msg, msg


def _mixed_slice(tmp_path, name, ttype):
    """A Q4_K_S slice of tinyk with one matrix replaced by `ttype` blocks."""
    sh = ggjt.SHAPES["tinyk"]
    src, dst = str(tmp_path / "a.bin"), str(tmp_path / "b.bin")
    ggjt.write_kquant_slice(src, sh, 0, 0, "q4_K_S", seed=0)
    f = ggjt.read_file(src)

    def tensors():
        for n, t in f.tensors.items():
            if n == name:
                rows, k = t.ne[1], t.ne[0]
                w = np.random.default_rng(0).standard_normal((rows, k), dtype=np.float32) / 16
                yield n, ttype, t.ne, ggjt.encode_tensor(w, ttype)
            else:
                yield n, t.ttype, t.ne, f.read_raw(n)
    ggjt.write_file(dst, f.hparams, f.vocab, tensors())
    return dst


@pytest.mark.parametrize("name", ["layers.0.attention.wo.weight", "layers.0.feed_forward.w2.weight"])
def test_kquant_legacy_mix_is_refused_by_ggjt(tmp_path, name):
    """A Q4_K slice with one Q4_0 matrix: ggjt.check_slice_types names the tensor and its type (the library's own
    refusal is in the GPU tests); the C restatement refuses it through the same check."""
    from kq_port import KQPortSlice
    path = _mixed_slice(tmp_path, name, ggjt.T_Q4_0)
    with pytest.raises(ValueError) as ei:
        ggjt.check_slice_types(ggjt.read_file(path, sliced=True))
    assert name in str(ei.value) and "q4_0" in str(ei.value)
    with pytest.raises(ValueError):
        KQPortSlice(path, 64)


def test_check_slice_types_accepts_the_mixes(tmp_path):
    path = str(tmp_path / "s.bin")
    for mix in ggjt.KQUANT_MIXES:
        ggjt.write_kquant_slice(path, ggjt.SHAPES["tinyk"], 2, 4, mix, seed=0)
        types = ggjt.check_slice_types(ggjt.read_file(path, sliced=True))
        assert len(types) == 21 and set(types) <= {ggjt.T_Q4_K, ggjt.T_Q6_K}
        assert (ggjt.T_Q6_K in types) == (mix != "q4_K_S")


def test_kquant_shapes():
    for name, (e, ff, dh) in {"tinyk": (256, 768, 64), "tinyk128": (512, 1536, 128)}.items():
        sh = ggjt.SHAPES[name]
        assert (sh.n_embd, sh.n_ff, sh.n_embd // sh.n_head, sh.n_layer) == (e, ff, dh, 8)
        assert e % 256 == 0 and ff % 256 == 0
