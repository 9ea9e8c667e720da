"""Numeric edge cases for the exact path (TEST INFRASTRUCTURE): slice recipes, input classes and a witness.

Gaussian activations and quantised-Gaussian weights never reach several branches of the exact kernels: all-zero
activation blocks, exact round-half-even ties in `x * id`, equal magnitudes in a Q8_K super-block, fp16 scales that
round to 0 or are subnormal, outlier channels, saturated softmax rows.  The recipes rewrite the tensors of a synthetic
slice (or extra-layers) file so that such values occur; the input classes feed rows that reach them; `witness` counts,
on the C restatement's own primitives, how often the first matmul's activation quantiser meets each edge, so the tests
can assert that they reach it and do not just claim to.

Every class is finite: with NaN inputs the reference's max reductions depend on their order, so "bit-identical" has no
meaning there.
"""
from __future__ import annotations

import ctypes as C
import os
import tempfile

import numpy as np

from distributedllm_b200 import ggjt

LEGACY = (ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0)
HAS_MIN = (ggjt.T_Q4_1, ggjt.T_Q5_1)
RECIPES = ("unit_norm", "zeros", "scales", "k_large")
CLASSES = ("gauss", "outlier", "zeros", "alternating", "constant", "lattice", "tiny30", "tiny40", "huge")
SUBNORMAL_D = np.uint16(0x0010)           # 2^-20 as fp16 (subnormal)
# k_large: wk times this puts the largest cached K values of most classes in [3e4, 65504).  Constant rows sum each wk
# row; a Q4_K row's sum is biased, reaches ~1.2e5 and is cached as fp16 inf: every score of those rows is then NaN.
K_SCALE = 9000.0


# --------------------------------------------------------------------------- tensor rewriting
def _blocks(raw: bytes, ttype: int, ne) -> np.ndarray:
    """[rows, nb, block bytes] u8 view of a quantised matrix, or [rows, k] fp16 / f32 values."""
    k, rows = ne[0], (ne[1] if len(ne) > 1 else 1)
    if ttype == ggjt.T_F16:
        return np.frombuffer(raw, np.float16).reshape(rows, k).copy()
    if ttype == ggjt.T_F32:
        return np.frombuffer(raw, np.float32).reshape(rows, k).copy()
    blk, sz = ggjt.TYPE_BLOCK[ttype]
    return np.frombuffer(raw, np.uint8).reshape(rows, k // blk, sz).copy()


def _set_f16(b: np.ndarray, off: int, mask: np.ndarray, val) -> None:
    """Field of fp16 bits at byte `off` of the blocks selected by `mask` := val (uint16 bits, scalar or array)."""
    v = np.broadcast_to(np.asarray(val, np.uint16).reshape(-1), b[mask].shape[:-1]).copy()
    b[mask, off:off + 2] = v.view(np.uint8).reshape(-1, 2)


def _get_f16(b: np.ndarray, off: int) -> np.ndarray:
    return b[..., off:off + 2].copy().view(np.float16)[..., 0]


def pack_q4_k_scales(sc: np.ndarray, m: np.ndarray) -> np.ndarray:
    """[..., 8] 6-bit scales and minima -> the 12 packed bytes (inverse of ggjt._q4_k_scale_min)."""
    sc, m = sc.astype(np.int32), m.astype(np.int32)
    q = np.empty(sc.shape[:-1] + (12,), np.int32)
    q[..., 0:4] = (sc[..., :4] & 63) | ((sc[..., 4:] >> 4) << 6)
    q[..., 4:8] = (m[..., :4] & 63) | ((m[..., 4:] >> 4) << 6)
    q[..., 8:12] = (sc[..., 4:] & 0xF) | ((m[..., 4:] & 0xF) << 4)
    return q.astype(np.uint8)


def _pow2_f16(d: np.ndarray) -> np.ndarray:
    """fp16 bits of sign(d) * 2^round(log2|d|) (0 stays 0)."""
    a = np.abs(d.astype(np.float32))
    p = np.where(a > 0, np.exp2(np.round(np.log2(np.where(a > 0, a, 1)))), 0) * np.sign(d.astype(np.float32))
    return p.astype(np.float16).view(np.uint16)


def scale_edges(name: str, ttype: int, w: np.ndarray, big_ok: bool) -> np.ndarray:
    """Block scales of 0, 2^-20 (subnormal) and powers of two; Q4_1 / Q5_1 minima made negative; Q4_K sub-block scales /
    minima of 0 and 63 and d / dmin of 0 or subnormal; Q6_K scales -128 and 127; F16 subnormals and, where `big_ok`, a few
    weights near +-65504."""
    if ttype == ggjt.T_F16:
        v = w.astype(np.float32)
        flat = v.reshape(-1)
        flat[3::13] = np.float32(2.0 ** -20) * np.sign(flat[3::13] + np.float32(1e-30))
        flat[7::29] = np.float32(5.96e-8)                     # the smallest fp16 subnormal
        if big_ok:
            flat[11::4099] = np.float32(65504.0)
            flat[17::6007] = np.float32(-65000.0)
        return flat.reshape(w.shape).astype(np.float16)
    if ttype == ggjt.T_F32:
        return w
    idx = np.arange(w.shape[0] * w.shape[1]).reshape(w.shape[:2])
    if ttype in LEGACY:
        _set_f16(w, 0, idx % 7 == 0, 0)
        _set_f16(w, 0, idx % 7 == 1, SUBNORMAL_D)
        sel = idx % 7 == 2
        _set_f16(w, 0, sel, _pow2_f16(_get_f16(w, 0)[sel]))
        if ttype in HAS_MIN:
            sel = idx % 7 == 3
            m = _get_f16(w, 2)[sel].astype(np.float32)
            _set_f16(w, 2, sel, (-np.abs(m) * np.float32(3)).astype(np.float16).view(np.uint16))
            _set_f16(w, 2, idx % 7 == 4, 0)
    elif ttype == ggjt.T_Q4_K:
        r = idx % 6
        sc, m = ggjt._q4_k_scale_min(w[..., 4:16])
        sc[r == 0], m[r == 0] = 63, 0
        sc[r == 1], m[r == 1] = 0, 63
        sc[r == 2, ::2], m[r == 2, ::2] = 63, 63
        w[..., 4:16] = pack_q4_k_scales(sc, m)
        _set_f16(w, 0, r == 3, 0)
        _set_f16(w, 2, r == 4, 0)
        _set_f16(w, 0, r == 5, SUBNORMAL_D)
        _set_f16(w, 2, r == 5, np.uint16(0x0001))
    elif ttype == ggjt.T_Q6_K:
        r = idx % 4
        sc = w[..., 192:208].view(np.int8)
        sc[r == 0] = -128
        sc[r == 1] = 127
        sc[r == 2, ::2] = -128
        sc[r == 2, 1::2] = 127
        _set_f16(w, 208, r == 3, _pow2_f16(_get_f16(w, 208)[r == 3]))
    return w


def _zero_rows(w: np.ndarray, rows) -> np.ndarray:
    w[rows] = 0
    return w


def _constant_rows(ttype: int, w: np.ndarray, rows) -> np.ndarray:
    """Every weight of these rows equal (one value per block)."""
    if ttype in (ggjt.T_F16, ggjt.T_F32):
        w[rows] = 0.01
    elif ttype in (ggjt.T_Q4_0, ggjt.T_Q8_0):
        w[rows, :, 2:] = 0x5B if ttype == ggjt.T_Q8_0 else 0xCC
    elif ttype == ggjt.T_Q4_1:
        w[rows, :, 4:] = 0xCC
    elif ttype == ggjt.T_Q5_0:
        w[rows, :, 2:6], w[rows, :, 6:] = 0xFF, 0x33            # 5-bit value 19 everywhere
    elif ttype == ggjt.T_Q5_1:
        w[rows, :, 4:8], w[rows, :, 8:] = 0x00, 0x77
    elif ttype == ggjt.T_Q4_K:
        w[rows, :, 4:16] = pack_q4_k_scales(np.full(8, 40), np.zeros(8, np.int32))
        w[rows, :, 16:] = 0xAA
    elif ttype == ggjt.T_Q6_K:
        w[rows, :, 0:128], w[rows, :, 128:192], w[rows, :, 192:208] = 0x55, 0x00, 0x20
    return w


def _scale_matrix(ttype: int, w: np.ndarray, f: float) -> np.ndarray:
    """Every weight times f (block scales and minima times f, rounded to fp16)."""
    if ttype in (ggjt.T_F16, ggjt.T_F32):
        return (w.astype(np.float32) * np.float32(f)).astype(w.dtype)
    offs = {ggjt.T_Q4_K: (0, 2), ggjt.T_Q6_K: (208,)}.get(ttype, (0, 2) if ttype in HAS_MIN else (0,))
    allb = np.ones(w.shape[:2], bool)
    for o in offs:
        _set_f16(w, o, allb, (_get_f16(w, o).astype(np.float32) * np.float32(f)).astype(np.float16).view(np.uint16))
    return w


def rewrite(src: str, dst: str, recipe: str) -> str:
    """Write `dst`: the slice or extra-layers file `src` with the tensors rewritten by `recipe` (see RECIPES)."""
    f = ggjt.read_file(src, sliced=True)
    d_head = f.hparams.n_embd // f.hparams.n_head

    def gen():
        for name, t in f.tensors.items():
            raw = f.read_raw(name)
            w = _blocks(raw, t.ttype, t.ne)
            if name.endswith("norm.weight"):
                if recipe in ("unit_norm", "zeros", "k_large", "extra"):
                    w[:] = 1.0
            elif recipe == "zeros":
                if name.endswith("attention.wv.weight"):
                    _zero_rows(w, slice(0, d_head))
                elif name.endswith(("feed_forward.w1.weight", "feed_forward.w3.weight")):
                    _zero_rows(w, slice(32, 64))
                    if t.ttype in (ggjt.T_Q4_K, ggjt.T_Q6_K):
                        _zero_rows(w, slice(256, 512))
                    if name.endswith("w1.weight"):
                        _zero_rows(w, slice(96, 128))        # SiLU(0) * w3 x: a block of signed zeros
                elif name.endswith("attention.wq.weight"):
                    _constant_rows(t.ttype, w, slice(0, 8))
            elif recipe == "scales":
                w = scale_edges(name, t.ttype, w, name.endswith(("attention.wo.weight", "feed_forward.w2.weight")))
            elif recipe == "k_large" and name.endswith("attention.wk.weight"):
                w = _scale_matrix(t.ttype, w, K_SCALE)
            elif recipe == "extra":
                w = scale_edges(name, t.ttype, w, name.startswith("tok_embeddings"))
            elif recipe in ("no_v", "pass") and name.startswith("layers.%d." % f.hparams.first_layer):
                # the first layer's attention output is 0 (wv = 0), so its ffn norm sees the layer input exactly; with
                # w2 = 0 as well ("pass") the layer returns its input and the next layer's attention norm sees it
                if name.endswith("attention.wv.weight") or (recipe == "pass" and name.endswith("feed_forward.w2.weight")):
                    _zero_rows(w, slice(None))
            yield name, t.ttype, t.ne, np.ascontiguousarray(w).tobytes()

    ggjt.write_file(dst, f.hparams, f.vocab, list(gen()))
    return dst


def make_slice(dirpath: str, shape: str, wtype, recipe: str, layers=(0, 1), seed: int = 5) -> str:
    """A synthetic slice (legacy type `wtype`, or a k-quant mix name) rewritten by `recipe`."""
    sh = ggjt.SHAPES[shape]
    tag = wtype if isinstance(wtype, str) else ggjt.TYPE_NAME[wtype]
    src = os.path.join(dirpath, "%s_%s_%d_%d_s%d.bin" % (shape, tag, layers[0], layers[1], seed))
    if not os.path.exists(src):
        if isinstance(wtype, str):
            ggjt.write_kquant_slice(src, sh, layers[0], layers[1], wtype, seed=seed)
        else:
            ggjt.write_synth_slice(src, sh, layers[0], layers[1], wtype, seed=seed)
    return rewrite(src, src[:-4] + "_" + recipe + ".bin", recipe)


EXTRA_SHAPE = "tinyk128"                  # n_embd 512: every tok_embeddings type, Q4_K included


def make_extra(dirpath: str, wtype: int) -> str:
    """An extra-layers file of EXTRA_SHAPE with tok_embeddings in `wtype` (Q4_K: output.weight Q6_K, otherwise the same
    type as tok_embeddings; F32: F16 output), unit norm weights and edge block scales in both matrices."""
    sh = ggjt.SHAPES[EXTRA_SHAPE]
    src = os.path.join(dirpath, "extra_%s.bin" % ggjt.TYPE_NAME[wtype])
    if wtype == ggjt.T_Q4_K:
        ggjt.write_kquant_extra(src, sh, "q4_K_M", seed=5)
    else:
        ex = list(ggjt.synth_extra_tensors(sh, wtype, 5))
        if wtype == ggjt.T_F32:                           # an F32 output.weight is not a supported lm_head
            ex = [e if e[0] != "output.weight" else
                  ("output.weight", ggjt.T_F16, e[2], np.frombuffer(e[3], np.float32).astype(np.float16).tobytes()) for e in ex]
        hp = ggjt.HParams(sh.n_vocab, sh.n_embd, sh.n_mult, sh.n_head, 0, sh.n_embd // sh.n_head,
                          ggjt._FTYPE_OF[wtype], ggjt.NO_FIRST_LAYER)
        ggjt.write_file(src, hp, ggjt.default_vocab(sh.n_vocab), ex)
    return rewrite(src, src[:-4] + "_edges.bin", "extra")


def embed_tokens(n_vocab: int) -> list:
    """32 ids (the reference's eval arena holds no more per call) whose rows hold every block-scale pattern."""
    return list(range(24)) + [n_vocab - 1 - 37 * i for i in range(8)]


_DEQUANT = {ggjt.T_Q4_0: ggjt.dequantize_q4_0, ggjt.T_Q4_1: ggjt.dequantize_q4_1, ggjt.T_Q5_0: ggjt.dequantize_q5_0,
            ggjt.T_Q5_1: ggjt.dequantize_q5_1, ggjt.T_Q8_0: ggjt.dequantize_q8_0, ggjt.T_Q4_K: ggjt.dequantize_q4_K,
            ggjt.T_Q6_K: ggjt.dequantize_q6_K}


def dequant_rows(f: ggjt.GGJTFile, name: str, rows) -> np.ndarray:
    """Rows of a matrix of file f as float32, by ggjt's dequantisers (one rounding per product, as ggml's)."""
    t = f.tensors[name]
    w = _blocks(f.read_raw(name), t.ttype, t.ne)[np.asarray(rows)]
    if t.ttype in (ggjt.T_F16, ggjt.T_F32):
        return w.astype(np.float32)
    return _DEQUANT[t.ttype](w)


PORT_OUTPUT_TYPES = (ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0, ggjt.T_F16, ggjt.T_Q6_K)


def port_logits(path: str, x: np.ndarray) -> np.ndarray:
    """Logits of every row of x on the C restatement: RMSNorm * norm.weight, then the Q6_K lm_head of kq_port, or for
    Q4_0, Q4_1, Q8_0 and F16 slice_oracle.c's activation quantisers and dots (F16: fp16 activations), for Q5_0 and Q5_1
    q5_port's."""
    f = ggjt.read_file(path, sliced=True)
    wt = f.tensors["output.weight"].ttype
    if wt == ggjt.T_Q6_K:
        from kq_port import KQPortExtra
        return KQPortExtra(path).logits(x)
    import q5_port
    assert wt in PORT_OUTPUT_TYPES, ggjt.TYPE_NAME.get(wt, wt)
    k, nv = f.hparams.n_embd, f.hparams.n_vocab
    w = np.frombuffer(f.read_raw("output.weight"), np.uint8).copy()
    nw = np.frombuffer(f.read_raw("norm.weight"), np.float32).copy()
    x = np.ascontiguousarray(x, np.float32).reshape(-1, k)
    y = np.empty((len(x), nv), np.float32)
    q5_port.lib().q5_logits(wt, ptr(w), nv, k, ptr(nw), ptr(x), len(x), ptr(y))
    return y


# --------------------------------------------------------------------------- input classes
def _lattice_row(rng: np.random.Generator, k: int, qk_max: int) -> np.ndarray:
    """Odd integers with one +-254 per 32-block (one +-256 per 256-block instead where qk_max == 256), fixed up so that
    the mean square is exactly 4096: RMSNorm then scales by exactly 1/64, and with unit norm weights x * id lands on
    k + 1/2 for every odd entry (Q8_0 / Q8_1: id = 127 / (254/64) = 32; Q8_K: iscale = -128 / (256/64) = -32)."""
    x = np.clip(np.round(rng.standard_normal(k) * 64 / 2) * 2 + 1, -253, 253).astype(np.int64)
    fixed = np.zeros(k, bool)
    for b in range(k // 32):
        j = b * 32 + int(rng.integers(0, 32))
        x[j], fixed[j] = (256 if (qk_max == 256 and b % 8 == 0) else 254) * (1 if rng.random() < 0.5 else -1), True
    target = 4096 * k
    # odd squares are 1 mod 8: a few even entries make the residue right, odd-for-odd swaps close the rest
    resid = (target - int((x * x).sum())) % 8
    evens = {0: [], 1: [2, 2, 2], 2: [2, 4], 3: [2], 4: [2, 2, 2, 2], 5: [2, 2, 4], 6: [2, 2], 7: [4]}[resid]
    free = [j for j in rng.permutation(k) if not fixed[j]]
    for e in evens:
        j = free.pop()
        x[j], fixed[j] = e * (1 if x[j] > 0 else -1), True
    diff = target - int((x * x).sum())
    assert diff % 8 == 0
    it = 0
    while diff:
        it += 1
        assert it < 100000
        m = diff // 8
        if abs(m) > 120:
            j = free[int(rng.integers(0, len(free)))]
            a = abs(int(x[j]))
            want = a * a + diff
            b = int(np.sqrt(max(want, 1)))
            b = min(253, max(1, b - (1 - b % 2)))
        else:
            a = 2 * m - 1 if m > 0 else 2 * (-m) + 1
            cand = [j for j in free if abs(int(x[j])) == a]
            if cand:
                j, b = cand[0], a + 2 if m > 0 else a - 2
            else:
                j = free[int(rng.integers(0, len(free)))]
                b = a
        a = abs(int(x[j]))
        x[j] = b * (1 if x[j] > 0 else -1)
        diff -= b * b - a * a
    return x.astype(np.float32)


def inputs(cls: str, n: int, k: int, rng: np.random.Generator) -> np.ndarray:
    """n rows of input class `cls` (see CLASSES), n_embd k."""
    g = rng.standard_normal((n, k), dtype=np.float32)
    if cls == "gauss":
        return g
    if cls == "outlier":
        x = g.copy()
        x[:, [5, 37 % k, k // 2 + 3]] *= np.float32(1500)
        x[:, k - 9] *= np.float32(3e4)
        return x
    if cls == "zeros":
        x = g.copy()
        x[0::3] = 0                                       # whole rows
        x[1::3, 32:64] = 0                                # a 32-block
        x[1::3, 256:512] = 0 if k >= 512 else x[1::3, 256:512]
        x[2::3, 0:256] = 0                                # a 256-block
        x[2::3, 64:96] = -0.0
        return x
    if cls == "alternating":
        c = np.abs(g[:, :1]) + np.float32(0.25)
        s = np.where(np.arange(k) % 2 == 0, -1, 1).astype(np.float32)
        s = np.where((np.arange(n) % 2 == 0)[:, None], s, -s)            # negative element first in half the rows
        return (c * s).astype(np.float32)
    if cls == "constant":
        return np.repeat(g[:, :1] * np.float32(3), k, axis=1)
    if cls == "lattice":
        return np.stack([_lattice_row(rng, k, 256 if i % 2 else 32) for i in range(n)])
    if cls == "tiny30":
        return (g * np.float32(1e-30)).astype(np.float32)
    if cls == "tiny40":
        return (np.sign(g) * np.float32(1e-40) * (1 + (np.arange(k) % 3))).astype(np.float32)
    if cls == "huge":
        x = g.copy()
        x[:, 3::97] = np.float32(1e15)
        x[:, 50::211] = np.float32(-1e19)
        x[::2, k - 1] = np.float32(1e19)
        return x
    raise ValueError(cls)


# --------------------------------------------------------------------------- witness
def witness(port_lib, kq_lib, x: np.ndarray, norm_w: np.ndarray) -> dict:
    """Edges the first matmul's activation quantiser meets on rows x (layer norm weight norm_w), on the C restatement's
    primitives: RMSNorm, then Q8_0 / Q8_1 per 32-block and Q8_K per 256-block."""
    x = np.ascontiguousarray(x, np.float32)
    n, k = x.shape
    norm_w = np.ascontiguousarray(norm_w, np.float32)
    c = dict(ties=0, zero_blocks=0, d16_zero=0, id_inf=0, q8k_ties=0, q8k_ties_neg_first=0, q8k_ties_pos_first=0,
             q8k_zero=0)
    for r in range(n):
        v = np.empty(k, np.float32)
        port_lib.orc_rmsnorm(x[r].ctypes.data, norm_w.ctypes.data, k, v.ctypes.data)
        q = np.empty(k, np.int8)
        d = np.empty(k // 32, np.uint16)
        port_lib.orc_quant_q8_0(v.ctypes.data, k, q.ctypes.data, d.ctypes.data)
        vb = v.reshape(-1, 32)
        amax = np.abs(vb).max(1)
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            idv = np.where(amax != 0, np.float32(127) / amax, np.float32(0)).astype(np.float32)
            t = (vb * idv[:, None]).astype(np.float32)
            fin = np.isfinite(t)
            c["ties"] += int((fin & (t - np.floor(t) == np.float32(0.5))).sum())
        c["zero_blocks"] += int((amax == 0).sum())
        c["d16_zero"] += int(((amax != 0) & (d == 0)).sum())
        c["id_inf"] += int(((amax != 0) & np.isinf(idv)).sum())
        if k % 256 == 0:
            q8 = np.empty(k, np.int8)
            dk, bs = np.empty(k // 256, np.float32), np.empty(k // 16, np.int32)
            kq_lib.orc_quantize_q8_K(v.ctypes.data, k, q8.ctypes.data, dk.ctypes.data, bs.ctypes.data)
            for b in v.reshape(-1, 256):
                a = np.abs(b)
                mx = a.max()
                if mx == 0:
                    c["q8k_zero"] += 1
                    continue
                at = np.flatnonzero(a == mx)
                with np.errstate(over="ignore", invalid="ignore"):
                    t = (np.float32(-128) / b[at[0]] * b).astype(np.float32)          # nearest_int(iscale * x)
                    c["q8k_ties"] += int((np.isfinite(t) & (t - np.floor(t) == np.float32(0.5))).sum())
                if len(at) > 1 and (b[at] > 0).any() and (b[at] < 0).any():
                    c["q8k_ties_neg_first" if b[at[0]] < 0 else "q8k_ties_pos_first"] += 1
    return c


def slice_norm(path: str) -> np.ndarray:
    f = ggjt.read_file(path, sliced=True)
    return np.frombuffer(f.read_raw("layers.%d.attention_norm.weight" % f.hparams.first_layer), np.float32).copy()


def tmpdir() -> str:
    return tempfile.mkdtemp(prefix="b200_edges_")


def ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)
