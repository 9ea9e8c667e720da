"""Host twin of llama.cpp's LoRA merge (llama_apply_lora_from_file_internal, llama.cpp:3054-3100), in numpy.

For W [rows][K] with loraA [K][r] and loraB [rows][r]:
  1. BA[j][i] = ggml_vec_dot_f32(r, loraA[i], loraB[j]) in the AVX2 + FMA build's order: partial sums
     P[m] = fma(x[32c + m], y[32c + m], P[m]) over the chunks c of r & ~31, folded by GGML_F32x8_REDUCE, then the
     r % 32 leftovers added one by one (multiply, add).  The FMA is exact here: the float64 product of two floats is
     exact, TwoSum gives the sum's error, and rounding the double to odd before the cast to float32 rounds once.
  2. BA *= alpha / r when that is not 1.
  3. W += BA (dequantise, add, requantise with from_float), or W = quantise(base + BA) with an F16 sum for an F16 base.
"""
from __future__ import annotations

import os
import struct
from typing import Dict, Optional

import numpy as np

from distributedllm_b200 import ggjt

F32 = np.float32
MATS = ("attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight",
        "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight")


def _fma(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """float32 fma(a, b, c), correctly rounded."""
    p = a.astype(np.float64) * b.astype(np.float64)         # exact
    c64 = c.astype(np.float64)
    hi = p + c64
    bb = hi - p
    lo = (p - (hi - bb)) + (c64 - bb)                       # TwoSum: hi + lo == p + c exactly
    odd = (lo != 0) & ((hi.view(np.int64) & 1) == 0)       # round to odd, then one rounding to float32
    hi = np.where(odd, np.nextafter(hi, np.where(lo > 0, np.inf, -np.inf)), hi)
    return hi.astype(F32)


def ba(A: np.ndarray, B: np.ndarray, alpha: int, r_hdr: int) -> np.ndarray:
    """[rows][K] float32: BA, scaled as llama.cpp scales it."""
    A = np.ascontiguousarray(A, F32)
    B = np.ascontiguousarray(B, F32)
    r = A.shape[1]
    np_ = r & ~31
    X = A[None, :, :]                                       # x = loraA row i (column i of W)
    Y = B[:, None, :]                                       # y = loraB row j
    rows, K = B.shape[0], A.shape[0]
    s = np.zeros((rows, K), F32)
    if np_:
        P = [None] * 32
        for m in range(32):
            acc = np.zeros((rows, K), F32)
            for c in range(0, np_, 32):
                acc = _fma(np.broadcast_to(X[..., c + m], (rows, K)), np.broadcast_to(Y[..., c + m], (rows, K)), acc)
            P[m] = acc
        V = [(P[m] + P[16 + m]) + (P[8 + m] + P[24 + m]) for m in range(8)]
        s = ((V[0] + V[4]) + (V[1] + V[5])) + ((V[2] + V[6]) + (V[3] + V[7]))
    for k in range(np_, r):
        s = (s + (X[..., k] * Y[..., k]).astype(F32)).astype(F32)
    scale = F32(alpha) / F32(r_hdr)
    if scale != F32(1):
        s = (s * scale).astype(F32)
    return s


def _first_pick(xb: np.ndarray, key: np.ndarray, largest: bool) -> np.ndarray:
    idx = key.argmax(axis=-1) if largest else key.argmin(axis=-1)   # first occurrence, as a strict forward scan
    return np.take_along_axis(xb, idx[..., None], axis=-1)[..., 0]


def _fp16(x: np.ndarray) -> np.ndarray:
    return x.astype(np.float16).view(np.uint8).reshape(x.shape + (2,))


def quantize(x: np.ndarray, wtype: int) -> np.ndarray:
    """type_traits[wtype].from_float on [rows][K] float32: the _reference quantisers for Q4_0 / Q4_1 / Q5_0 / Q5_1,
    the AVX2 quantize_row_q8_0 (id = 127 / amax, round half to even) for Q8_0, fp16 for F16.  Returns the raw bytes."""
    x = np.ascontiguousarray(x, F32)
    if wtype == ggjt.T_F16:
        return x.astype(np.float16).tobytes()
    rows, k = x.shape
    xb = x.reshape(rows, k // 32, 32)
    with np.errstate(divide="ignore", invalid="ignore"):
        if wtype == ggjt.T_Q8_0:
            amax = np.abs(xb).max(axis=2)
            d = (amax / F32(127)).astype(F32)
            idv = np.where(amax != 0, F32(127) / np.where(amax != 0, amax, F32(1)), F32(0)).astype(F32)
            q = np.rint((xb * idv[..., None]).astype(F32)).astype(np.int8)
            out = np.empty((rows, k // 32, 34), np.uint8)
            out[..., 0:2] = _fp16(d)
            out[..., 2:] = q.view(np.uint8)
            return out.tobytes()
        if wtype in (ggjt.T_Q4_0, ggjt.T_Q5_0):
            half = F32(8) if wtype == ggjt.T_Q4_0 else F32(16)
            amax = np.abs(xb).max(axis=2)
            mx = np.where(amax == 0, F32(0), _first_pick(xb, np.abs(xb), True)).astype(F32)
            d = (mx / -half).astype(F32)
            idv = np.where(d != 0, F32(1) / np.where(d != 0, d, F32(1)), F32(0)).astype(F32)
            v = ((xb * idv[..., None]).astype(F32) + (half + F32(0.5))).astype(F32)
            q = np.minimum(15 if wtype == ggjt.T_Q4_0 else 31, np.trunc(v).astype(np.int32))
            m = None
        else:
            five = wtype == ggjt.T_Q5_1
            m = _first_pick(xb, xb, False).astype(F32)
            mx = _first_pick(xb, xb, True).astype(F32)
            d = ((mx - m) / F32(31 if five else 15)).astype(F32)
            idv = np.where(d != 0, F32(1) / np.where(d != 0, d, F32(1)), F32(0)).astype(F32)
            v = (((xb - m[..., None]).astype(F32) * idv[..., None]).astype(F32) + F32(0.5)).astype(F32)
            q = np.trunc(v).astype(np.int32)
            q = (q & 0xFF) if five else np.minimum(15, q)
    five = wtype in (ggjt.T_Q5_0, ggjt.T_Q5_1)
    parts = [_fp16(d)]
    if m is not None:
        parts.append(_fp16(m))
    if five:
        bits = ((q >> 4) & 1).astype(np.uint32) << np.arange(32, dtype=np.uint32)
        qh = np.bitwise_or.reduce(bits, axis=2).astype("<u4")
        parts.append(qh.view(np.uint8).reshape(rows, k // 32, 4))
    parts.append(((q[..., :16] & 0xF) | ((q[..., 16:] & 0xF) << 4)).astype(np.uint8))
    return np.concatenate(parts, axis=2).tobytes()


def dequantize(raw: bytes, wtype: int, rows: int, k: int) -> np.ndarray:
    if wtype == ggjt.T_F16:
        return np.frombuffer(raw, np.float16).astype(F32).reshape(rows, k)
    if wtype == ggjt.T_F32:
        return np.frombuffer(raw, F32).reshape(rows, k).copy()
    bb = ggjt.TYPE_BLOCK[wtype][1]
    blocks = np.frombuffer(raw, np.uint8).reshape(rows, k // 32, bb)
    return {ggjt.T_Q4_0: ggjt.dequantize_q4_0, ggjt.T_Q4_1: ggjt.dequantize_q4_1, ggjt.T_Q5_0: ggjt.dequantize_q5_0,
            ggjt.T_Q5_1: ggjt.dequantize_q5_1, ggjt.T_Q8_0: ggjt.dequantize_q8_0}[wtype](blocks)


def merge_tensor(w_raw: bytes, wtype: int, rows: int, k: int, A, B, alpha: int, r_hdr: int,
                 base_raw: Optional[bytes] = None, btype: Optional[int] = None) -> bytes:
    """The merged bytes of one matrix (steps 1-3)."""
    d = ba(A, B, alpha, r_hdr)
    if base_raw is None:
        if wtype == ggjt.T_F16:
            return (dequantize(w_raw, wtype, rows, k) + d).astype(F32).astype(np.float16).tobytes()
        return quantize((dequantize(w_raw, wtype, rows, k) + d).astype(F32), wtype)
    x = (dequantize(base_raw, btype, rows, k) + d).astype(F32)
    if btype == ggjt.T_F16:                                 # ggml_add of an F16 base is an F16 tensor
        x = x.astype(np.float16).astype(F32)
    return quantize(x, wtype)


def merge_file(src: str, dst: str, lora: str, base: Optional[str] = None) -> Dict[str, bytes]:
    """Write `src` (a slice or full model) with the adapter merged into every matrix it has both tensors for; returns
    the merged tensors' bytes by name."""
    r_hdr, alpha, ts = ggjt.read_lora(lora)
    f = ggjt.read_file(src)
    bf = ggjt.read_file(base) if base else None
    merged = {}
    for name, t in f.tensors.items():
        if name + ".loraA" in ts and name + ".loraB" in ts:
            k, rows = t.ne
            braw = bf.read_raw(name) if bf else None
            merged[name] = merge_tensor(f.read_raw(name), t.ttype, rows, k, ts[name + ".loraA"], ts[name + ".loraB"],
                                        alpha, r_hdr, braw, bf.tensors[name].ttype if bf else None)
    with open(src, "rb") as fi:
        data = bytearray(fi.read())
    for name, raw in merged.items():
        t = f.tensors[name]
        data[t.offset:t.offset + t.nbytes] = raw
    with open(dst, "wb") as fo:
        fo.write(bytes(data))
    return merged


# --------------------------------------------------------------------------- cases shared with the goldens
SHAPE = ggjt.ModelShape(64, 64, 32, 2, 2)          # n_ff 192
FAMILIES = {"q4_0": ggjt.T_Q4_0, "q4_1": ggjt.T_Q4_1, "q5_0": ggjt.T_Q5_0, "q5_1": ggjt.T_Q5_1,
            "q8_0": ggjt.T_Q8_0, "f16": ggjt.T_F16}
RANKS = (1, 8, 16, 31, 32, 40, 64)


def cases():
    """(family, r, alpha, base) of the byte-for-byte comparison: every rank with alpha == r and alpha != r and no base,
    and an F16 and an F32 base at a short and an FMA-path rank."""
    out = []
    for fam in FAMILIES:
        for r in RANKS:
            for alpha in (r, r + 3):
                out.append((fam, r, alpha, None))
        for base in ("f16", "f32"):
            for r in (8, 40):
                out.append((fam, r, r + 3, base))
    return out


EDGE_RANKS = (2, 33, 63, 64, 65, 96, 128, 307, 308, 1024)   # 307 / 308: the last rank under / first over 48 KB of smem
MIXED_RANKS = {"attention.wq.weight": 8, "attention.wk.weight": 40, "attention.wv.weight": 16, "attention.wo.weight": 64,
               "feed_forward.w1.weight": 40, "feed_forward.w2.weight": 16, "feed_forward.w3.weight": 8}
MIXED_LAYER1 = {"attention.wq.weight": 64, "attention.wv.weight": 8}


def edges():
    """Cases beyond cases(): every rank path at a scale that is not a power of two, alpha of 1, 0 and negative, one
    adapter whose tensors have ranks other than its header's r (kind "mixed"), and requantisation edges built into an
    F32 base (kind "designed", see designed_blocks)."""
    out = []
    for fam in FAMILIES:
        for r in EDGE_RANKS:
            out.append((fam, r, 2 * r + 1, None))
        for r in (8, 64):
            for alpha in (1, r + 3, 3 * r, 0, -r, -(r + 3)):
                if (fam, r, alpha, None) not in out and (fam, r, alpha, None) not in cases():
                    out.append((fam, r, alpha, None))
        out.append((fam, 16, 19, None, "mixed"))
        out.append((fam, 2, -4, "f32", "designed"))
    return out


def case_id(c) -> str:
    fam, r, alpha, base = c[:4]
    kind = c[4] + "_" if len(c) > 4 else ""
    return "%s_%sr%d_a%d_%s" % (fam, kind, r, alpha, base or "nobase")


# ------------------------------------------------------------------ designed blocks
# Layer 0's wq of a "designed" case: an F32 base and a rank-2 adapter of powers of two (scale -2), so BA is exact and
# x = base + BA is exactly the target block.  Each target sits on one requantisation edge of its family.  Rows whose
# loraB is zero get BA = -0 (+0 scaled by -2), so a -0 in the base stays -0 there.
DESIGN_ROWS, DESIGN_K = 64, 64
_ZERO_ROWS = (1, 2)                                     # loraB == 0: BA == -0


def _fma_trunc_split(div: float):
    """(mx, x): for a Q4_1 / Q5_1 block with m = 0 and max mx, a value x whose (x - m) * id + 0.5 truncates differently
    when the multiply and add are one fma."""
    for mx in np.arange(16.5, 40, 0.37, dtype=np.float64):
        mx = F32(mx * (div / 15))
        d = F32(mx / F32(div))
        idv = F32(F32(1) / d)
        x0 = F32(F32(0.5) / idv)
        for k in range(-40, 41):
            x = F32(x0 + F32(k) * np.spacing(x0))
            two = np.trunc(F32(F32(x * idv) + F32(0.5)))
            one = np.trunc(_fma(np.array([x]), np.array([idv]), np.array([F32(0.5)]))[0])
            if two != one:
                return mx, x
    raise AssertionError("no fma split found")


def designed_blocks(fam: str) -> Dict[str, np.ndarray]:
    """Target blocks of family fam by edge name.  Names starting with "z_" need BA == -0 (a loraB-zero row)."""
    wtype = FAMILIES[fam]
    ar = np.arange(32, dtype=F32)
    rng = np.random.default_rng(7)
    small = lambda lo, hi: (np.round(rng.uniform(lo, hi, 32) * 4096) / 4096).astype(F32)   # noqa: E731
    out = {"zero_from_base": np.zeros(32, F32)}         # base = -BA != 0
    if wtype == ggjt.T_Q8_0:
        h = ar - F32(15.5)
        h[0] = 127                                      # amax 127: id 1, x * id half-way between integers
        out["half"] = h
        h2 = (ar - F32(15.5)) / F32(2)
        h2[31] = F32(-63.5)                             # amax 63.5: id 2
        out["half_id2"] = h2.astype(F32)
    elif wtype in (ggjt.T_Q4_0, ggjt.T_Q5_0):
        half = 8 if wtype == ggjt.T_Q4_0 else 16
        t = small(-0.5, 0.5)
        t[3], t[17] = 0.75, -0.75                       # +a first: max = +a
        out["pm_tie"] = t
        t = small(-0.5, 0.5)
        t[2], t[30] = -0.75, 0.75                       # -a first: max = -a
        out["mp_tie"] = t
        t = (ar % (2 * half) - F32(half - 0.5)).astype(F32)
        t[0] = -half                                    # max -half: d 1, id 1, x * id + half + 0.5 on integers
        out["on_int"] = t
    elif wtype in (ggjt.T_Q4_1, ggjt.T_Q5_1):
        div = 15 if wtype == ggjt.T_Q4_1 else 31
        out["min_eq_max"] = np.full(32, F32(0.3), F32)
        t = (ar % div + F32(0.5)).astype(F32)
        t[0], t[1] = 0, div                             # m 0, max div: d 1, id 1, (x - m) * id + 0.5 on integers
        out["on_int"] = t
        mx, x = _fma_trunc_split(div)
        t = small(1.0, 2.0)
        t[0], t[1], t[2] = 0, mx, x
        out["fma_split"] = t
        t = small(0.25, 0.5)
        t[1], t[9] = 0, -0.0                            # minimum +0 first, -0 later
        out["z_zero_tie"] = t
        t = np.zeros(32, F32)
        t[5::3] = -0.0                                  # all zero, lane 0 +0 and lane 31 -0: m and max are the first
        t[31] = -0.0
        out["z_all_zero_signs"] = t
    else:                                               # F16
        u = F32(2.0 ** -10)                             # ulp of fp16 at 1
        out["ties"] = (np.where(ar < 16, 1, -1) * (1 + (ar % 16) * u + u / 2)).astype(F32)
        s = F32(2.0 ** -24)                             # smallest fp16 subnormal
        t = ((ar - 16) * s / 2).astype(F32)             # subnormals, half-way subnormals, +-2^-25 (ties with zero)
        out["subnormal"] = t
        t = np.zeros(32, F32)
        t[1::2] = -0.0
        out["z_signed_zero"] = t
    return out


def _design_ab():
    """loraA [K][2], loraB [rows][2] of the designed matrix: powers of two, loraB zero on _ZERO_ROWS."""
    A = np.zeros((DESIGN_K, 2), F32)
    A[:, 0] = 2.0 ** -3
    A[:, 1] = np.where(np.arange(DESIGN_K) % 2, 2.0 ** -6, -2.0 ** -6)
    B = np.zeros((DESIGN_ROWS, 2), F32)
    B[:, 0] = np.array([1, -1, 0.5, -0.5], F32)[np.arange(DESIGN_ROWS) % 4] * F32(2.0 ** -8)
    B[1::2, 1] = B[1::2, 0]
    B[list(_ZERO_ROWS)] = 0
    return A, B


def designed_matrix(fam: str):
    """(base [64][64] F32, loraA, loraB, targets, placement {edge: (row, block)}) of a designed case."""
    A, B = _design_ab()
    d = ba(A, B, -4, 2)
    rng = np.random.default_rng(8)
    base = (rng.standard_normal((DESIGN_ROWS, DESIGN_K), dtype=F32) * F32(0.125)).astype(F32)
    target = (base + d).astype(F32)
    place = {}
    rows = iter(r for r in range(DESIGN_ROWS) if r not in _ZERO_ROWS)
    zrows = iter(_ZERO_ROWS)
    for name, blk in designed_blocks(fam).items():
        j = next(zrows) if name.startswith("z_") else next(rows)
        dj = d[j, 0:32]
        target[j, 0:32] = blk
        base[j, 0:32] = np.where(dj == 0, blk, (blk.astype(np.float64) - dj).astype(F32))
        place[name] = (j, 0)
    for name, (j, b) in place.items():                  # every designed x is base + BA with no rounding
        cols = slice(32 * b, 32 * b + 32)
        assert np.array_equal(base[j, cols].astype(np.float64) + d[j, cols], target[j, cols].astype(np.float64)), name
    assert np.array_equal((base + d).astype(F32).view(np.uint32), target.view(np.uint32))
    return base, A, B, target, place


def _matrix(rng, rows: int, k: int) -> np.ndarray:
    w = (rng.standard_normal((rows, k), dtype=F32) * F32(1 / np.sqrt(k))).astype(F32)
    w[0] = 0                                            # all-zero blocks
    tie4 = np.arange(k, dtype=F32) % 16 - F32(7.5)      # Q4_0: max -8 gives id 1, so x*id + 8.5 lands on integers
    tie4[::32] = -8
    w[1] = tie4
    tie8 = np.arange(k, dtype=F32) % 64 - F32(31.5)     # Q8_0: amax 127 gives id 1, x*id half-way between integers
    tie8[::32] = 127
    w[2] = tie8
    return w


def write_case(d: str, c, seed: int = 0):
    """Full model, adapter (and base model) of case c under directory d: (model, adapter, base or None)."""
    fam, r, alpha, base = c[:4]
    kind = c[4] if len(c) > 4 else None
    wtype = FAMILIES[fam]
    sh = SHAPE
    rng = np.random.default_rng([seed, r, alpha % (1 << 32), wtype] + ([len(kind)] if kind else []))
    e, ff = sh.n_embd, sh.n_ff
    dims = {"attention.wq.weight": (e, e), "attention.wk.weight": (e, e), "attention.wv.weight": (e, e),
            "attention.wo.weight": (e, e), "feed_forward.w1.weight": (ff, e), "feed_forward.w2.weight": (e, ff),
            "feed_forward.w3.weight": (ff, e)}
    mats = {}
    for layer in range(sh.n_layer):
        for nm in MATS:
            mats["layers.%d.%s" % (layer, nm)] = _matrix(rng, *dims[nm])
    designed = {}
    if kind == "designed":
        wq = "layers.0.attention.wq.weight"
        assert dims["attention.wq.weight"] == (DESIGN_ROWS, DESIGN_K)
        mats[wq], dA, dB = designed_matrix(fam)[:3]
        designed[wq] = (dA, dB)
    vocab = ggjt.default_vocab(sh.n_vocab)

    def model(wt):
        ex = {n: (t, ne, raw) for n, t, ne, raw in ggjt.synth_extra_tensors(sh, ggjt.T_Q4_0 if wt == ggjt.T_F32 else wt, seed)}
        for n in ("tok_embeddings.weight", "norm.weight", "output.weight"):
            yield (n,) + ex[n]
        for layer in range(sh.n_layer):
            for nm in ggjt.LAYER_TENSORS:
                name = "layers.%d.%s" % (layer, nm)
                if nm.endswith("norm.weight"):
                    yield name, ggjt.T_F32, (e,), np.ones(e, F32).tobytes()
                else:
                    w = mats[name]
                    yield name, wt, (w.shape[1], w.shape[0]), ggjt.encode_tensor(w, wt)

    ftype = {ggjt.T_F32: ggjt.FTYPE_F32}.get(wtype, ggjt._FTYPE_OF[wtype])
    hp = ggjt.HParams(sh.n_vocab, e, sh.n_mult, sh.n_head, sh.n_layer, e // sh.n_head, ftype, None)
    mpath = os.path.join(d, "model.bin")
    ggjt.write_file(mpath, hp, vocab, model(wtype))
    bpath = None
    if base:
        bt = ggjt.T_F16 if base == "f16" else ggjt.T_F32
        bpath = os.path.join(d, "base.bin")
        ggjt.write_file(bpath, ggjt.HParams(sh.n_vocab, e, sh.n_mult, sh.n_head, sh.n_layer, e // sh.n_head,
                                            ggjt._FTYPE_OF.get(bt, ggjt.FTYPE_F32), None), vocab, model(bt))
    tens = []
    for name, w in mats.items():
        layer = int(name.split(".")[1])
        if layer == 1 and not name.endswith(("wq.weight", "wv.weight")):
            continue                                    # layer 1: alpaca-lora's targets only
        rows, k = w.shape
        rt = r
        if kind == "mixed":                             # tensor ranks other than the header's r
            rt = (MIXED_RANKS if layer == 0 else MIXED_LAYER1)[name.split(".", 2)[2]]
        A = (rng.standard_normal((k, rt), dtype=F32) * F32(0.05)).astype(F32)
        B = (rng.standard_normal((rows, rt), dtype=F32) * F32(0.05)).astype(F32)
        B[:3] = 0                                       # the zero and tie rows keep their values (BA == +-0)
        if name in designed:
            A, B = designed[name]
        tens += [(name + ".loraA", A), (name + ".loraB", B)]
    apath = os.path.join(d, "adapter.bin")
    ggjt.write_lora(apath, r, alpha, tens)
    return mpath, apath, bpath
