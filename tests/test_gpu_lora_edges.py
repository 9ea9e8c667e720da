"""b200_slice_load_lora at its edges, compared by the packed device bytes of every matrix (Slice.debug_weights): every
case of tests/lora_ref.py's cases() and edges() (each equal to llama.cpp's merge byte for byte on the host), the ragged
64-row tiles of tiny128 / tiny3b, and one layer each of LLaMA-13B, 30B and 65B with loraB nonzero on a sample of rows."""
from __future__ import annotations

import os
import time

import numpy as np
import pytest

import lora_ref
from distributedllm_b200 import capi, ggjt
from test_gpu_lora import FAMS, bits

pytestmark = pytest.mark.gpu

CASES = lora_ref.cases() + lora_ref.edges()
QUANT_IDS = {"qkv": 0, "wo": 1, "w13": 2, "w2": 3}
F16_IDS = {"wq": 0, "wk": 1, "wv": 2, "wo": 3, "w1": 4, "w2": 5, "w3": 6}


def matrix_ids(wtype: int):
    return F16_IDS if wtype == ggjt.T_F16 else QUANT_IDS


def assert_same_packed(a: capi.Slice, b: capi.Slice, wtype: int, n_layers: int = 1, what: str = "") -> None:
    for layer in range(n_layers):
        for name, w in matrix_ids(wtype).items():
            pa, pb = a.debug_weights(layer, w), b.debug_weights(layer, w)
            assert pa.size > 0 and pa.size == pb.size, (what, layer, name, pa.size, pb.size)
            if not np.array_equal(pa, pb):
                bad = np.flatnonzero(pa != pb)
                raise AssertionError("%s layer %d %s: %d of %d packed bytes differ, first at %d"
                                     % (what, layer, name, bad.size, pa.size, bad[0]))


def assert_same_prompt_and_step(a: capi.Slice, b: capi.Slice, E: int, seed: int = 0) -> None:
    rng = np.random.default_rng(seed)
    for n in (5, 1):
        x = rng.standard_normal((n, E), dtype=np.float32)
        assert np.array_equal(bits(a.session_forward(0, x)), bits(b.session_forward(0, x)))


@pytest.mark.parametrize("case", CASES, ids=[lora_ref.case_id(c) for c in CASES])
def test_case_packed_bytes_equal_host_merge(tmp_path, case):
    """Each layer's slice loaded with the case's adapter (and base) holds the packed bytes of the host-merged slice."""
    d = str(tmp_path)
    m, ad, base = lora_ref.write_case(d, case)
    merged = os.path.join(d, "merged.bin")
    lora_ref.merge_file(m, merged, ad, base)
    wtype = lora_ref.FAMILIES[case[0]]
    for layer in range(lora_ref.SHAPE.n_layer):
        sp, mp, bp = (os.path.join(d, "%s%d.bin" % (k, layer)) for k in "smb")
        ggjt.slice_model(m, sp, layer, layer)
        ggjt.slice_model(merged, mp, layer, layer)
        if base:
            ggjt.slice_model(base, bp, layer, layer)
        a = capi.Slice(sp, 0, 64, n_sessions=1, lora=ad, lora_base=bp if base else None)
        b = capi.Slice(mp, 0, 64, n_sessions=1)
        try:
            assert_same_packed(a, b, wtype, what=lora_ref.case_id(case))
            assert_same_prompt_and_step(a, b, lora_ref.SHAPE.n_embd)
        finally:
            a.close(), b.close()


# ------------------------------------------------------------------------------------ LLaMA-13B / 30B / 65B layers
def sampled_rows(rows: int, stride: int = 8) -> np.ndarray:
    """The first and last 64-row tile, and one row per `stride` rows elsewhere (a different row of each 8-row group)."""
    keep = np.zeros(rows, bool)
    keep[:64] = True
    keep[(rows - 1) // 64 * 64:] = True
    g = np.arange(0, rows, stride)
    keep[np.minimum(g + (g // stride) % 8, rows - 1)] = True
    return np.flatnonzero(keep)


def sampled_adapter(slice_path: str, out: str, r: int, alpha: int, mats, seed: int = 0, stride: int = 8):
    """A rank-r adapter on `mats` of the slice's layer with loraB zero outside sampled_rows; returns {matrix name:
    (A, rows, B of those rows)}."""
    f = ggjt.read_file(slice_path)
    rng = np.random.default_rng([seed, r])
    ts, by = [], {}
    for name, t in f.tensors.items():
        if not name.endswith(tuple(mats)):
            continue
        k, rows = t.ne
        A = (rng.standard_normal((k, r), dtype=np.float32) * np.float32(0.05)).astype(np.float32)
        S = sampled_rows(rows, stride)
        B = np.zeros((rows, r), np.float32)
        B[S] = rng.standard_normal((S.size, r), dtype=np.float32) * np.float32(0.05)
        ts += [(name + ".loraA", A), (name + ".loraB", B)]
        by[name] = (A, S, B[S])
    ggjt.write_lora(out, r, alpha, ts)
    return by


def merge_sampled(src: str, dst: str, by, alpha: int, r_hdr: int, base: str = None, chunk: int = 1024) -> None:
    """lora_ref.merge_file for an adapter whose loraB is zero outside the sampled rows: BA is computed on those rows
    only (every other row's BA is +0, test_lora_ref.test_zero_b_rows_give_plus_zero) and the matrix is requantised in
    row chunks."""
    f = ggjt.read_file(src)
    bf = ggjt.read_file(base) if base else None
    with open(src, "rb") as fi:
        data = bytearray(fi.read())
    for name, (A, S, BS) in by.items():
        t = f.tensors[name]
        k, rows = t.ne
        dS = lora_ref.ba(A, BS, alpha, r_hdr)
        w_raw = f.read_raw(name)
        src_t, src_raw = (bf.tensors[name].ttype, bf.read_raw(name)) if bf else (t.ttype, w_raw)
        bpr = len(src_raw) // rows
        opr = t.nbytes // rows
        out = bytearray(t.nbytes)
        for r0 in range(0, rows, chunk):
            r1 = min(rows, r0 + chunk)
            x = lora_ref.dequantize(src_raw[r0 * bpr:r1 * bpr], src_t, r1 - r0, k)
            d = np.zeros_like(x)
            sel = (S >= r0) & (S < r1)
            d[S[sel] - r0] = dS[sel]
            x = (x + d).astype(np.float32)
            if bf is not None and src_t == ggjt.T_F16:
                x = x.astype(np.float16).astype(np.float32)
            out[r0 * opr:r1 * opr] = x.astype(np.float16).tobytes() if t.ttype == ggjt.T_F16 else lora_ref.quantize(x, t.ttype)
        data[t.offset:t.offset + t.nbytes] = out
    with open(dst, "wb") as fo:
        fo.write(bytes(data))


@pytest.mark.parametrize("shape", ["tiny128", "tiny3b"])
@pytest.mark.parametrize("fam", list(FAMS))
def test_ragged_tiles_rank65(tmp_path, shape, fam):
    """Shapes whose row counts end in a partial 64-row CTA tile (tiny128 n_ff 1376, tiny3b n_embd 800), at a rank with
    two FMA chunks and a leftover and a scale of 131 / 65; loraB is nonzero on every row of the first and last tile."""
    sh = ggjt.SHAPES[shape]
    p = str(tmp_path / "s.bin")
    ggjt.write_synth_slice(p, sh, 0, 0, FAMS[fam], seed=5)
    ad = str(tmp_path / "a.bin")
    by = sampled_adapter(p, ad, 65, 131, lora_ref.MATS[:1] + lora_ref.MATS[2:3] + lora_ref.MATS[4:6])
    m = str(tmp_path / "m.bin")
    merge_sampled(p, m, by, 131, 65)
    a = capi.Slice(p, 0, 64, n_sessions=1, lora=ad)
    b = capi.Slice(m, 0, 64, n_sessions=1)
    try:
        assert_same_packed(a, b, FAMS[fam], what=shape)
        assert_same_prompt_and_step(a, b, sh.n_embd)
    finally:
        a.close(), b.close()


# (shape, weight type, base type, r, alpha, matrices, sample stride): rank 64 runs two FMA chunks per element on the
# host, so its sample keeps one row in 64 outside the first and last tile
LARGE = [("13b", ggjt.T_Q5_0, None, 16, 40, lora_ref.MATS, 8),
         ("30b", ggjt.T_Q8_0, ggjt.T_F16, 8, 13, ("attention.wq.weight", "attention.wv.weight", "feed_forward.w2.weight"), 8),
         ("65b", ggjt.T_Q4_0, None, 64, 160, lora_ref.MATS, 64),
         ("65b", ggjt.T_F16, None, 16, 40, ("feed_forward.w1.weight", "feed_forward.w2.weight"), 8)]


@pytest.mark.parametrize("shape,wtype,btype,r,alpha,mats,stride", LARGE,
                         ids=["13b_q5_0_r16_all", "30b_q8_0_f16base_r8", "65b_q4_0_r64_all", "65b_f16_r16_w1w2"])
def test_large_layer_packed_bytes(tmp_path, shape, wtype, btype, r, alpha, mats, stride):
    """One layer at a real shape: 65B's w1 | w3 job has 22016-row sources (grid.y 344) and its w2 K = 22016 (grid.x 688);
    30B's w2 K = 17920.  Prints the host twin's time and the adapted load's time."""
    sh = ggjt.SHAPES[shape]
    p, bp = str(tmp_path / "s.bin"), str(tmp_path / "base.bin")
    if wtype == ggjt.T_F16:
        ggjt.write_fast_f16_slice(p, sh, 0, 0, seed=2)
    else:
        ggjt.write_fast_q4_slice(p, sh, 0, 0, seed=2, wtype=wtype)
    if btype is not None:
        ggjt.write_fast_f16_slice(bp, sh, 0, 0, seed=3)
    ad = str(tmp_path / "a.bin")
    by = sampled_adapter(p, ad, r, alpha, mats, stride=stride)
    m = str(tmp_path / "m.bin")
    t0 = time.perf_counter()
    merge_sampled(p, m, by, alpha, r, bp if btype is not None else None)
    t_host = time.perf_counter() - t0
    t0 = time.perf_counter()
    a = capi.Slice(p, 0, 64, n_sessions=1, lora=ad, lora_base=bp if btype is not None else None)
    t_lora = time.perf_counter() - t0
    t0 = time.perf_counter()
    b = capi.Slice(m, 0, 64, n_sessions=1)
    t_plain = time.perf_counter() - t0
    try:
        assert_same_packed(a, b, wtype, what=shape)
        assert_same_prompt_and_step(a, b, sh.n_embd)
    finally:
        a.close(), b.close()
    print("\n[lora large] %s type %d r %d: host twin %.1f s, adapted load %.2f s, plain load %.2f s"
          % (shape, wtype, r, t_host, t_lora, t_plain))
