"""Float64 restatement of one fast-mode matmul (csrc/fastgemm2.cuh), in numpy.

Both operands of the tensor-core matmul can be reproduced bit for bit on the host:
  * activations, as k_prep_q8_f16 makes them: [RMSNorm * w ->] Q8_0 quantise (fp16 scale, round half to even) ->
    fp16(q * d);
  * weights, as the dequant warps make them: fp16((n - 8) * d) for Q4_0, fp16(q * d) for Q8_0 -- the exact fp32
    product rounded once (the HMUL2).
So the only freedom the kernel has is the fp32 summation order of the products, and its error is bounded by
tau * sum_k |w16 * x16| for a small tau.  `reference` computes the float64 sum and that magnitude; `store_error` and
`gate_error` return, per output, the smallest tau for which the kernel value is inside the bound.
"""
from __future__ import annotations

import ctypes
import ctypes.util

import numpy as np

from distributedllm_b200 import ggjt

F32, F16 = np.float32, np.float16


# ---------------------------------------------------------------------------------------------- operands
def prep(x: np.ndarray, norm_w: np.ndarray = None) -> np.ndarray:
    """k_prep_q8_f16: [N][K] fp32 rows -> [N][K] fp16 activations."""
    x = np.ascontiguousarray(x, dtype=F32)
    n, k = x.shape
    v = x
    if norm_w is not None:
        tot = (x * x).astype(np.float64).sum(axis=1)                    # double sum of the fp32 squares
        ms = (tot / k).astype(F32)
        scale = (F32(1) / np.sqrt((ms + F32(1e-6)).astype(F32))).astype(F32)
        v = ((x * scale[:, None]).astype(F32) * np.asarray(norm_w, F32)[None, :]).astype(F32)
    vb = v.reshape(n, k // 32, 32)
    amax = np.abs(vb).max(axis=2)
    d = (amax / F32(127)).astype(F32).astype(F16).astype(F32)
    with np.errstate(divide="ignore"):
        idv = np.where(amax != 0, F32(127) / np.where(amax != 0, amax, F32(1)), F32(0)).astype(F32)
    q = np.rint((vb * idv[..., None]).astype(F32))                     # round half to even, like rint_small
    q = q + F32(0)                                                      # rint_small returns an int: a zero quant is +0
    return (q * d[..., None]).astype(F32).astype(F16).reshape(n, k)


def weights16(blocks: np.ndarray, wtype: int) -> np.ndarray:
    """[rows][nb][block bytes] file blocks -> [rows][nb*32] fp16, as the dequant warps expand them."""
    if wtype == ggjt.T_Q4_0:
        w = ggjt.dequantize_q4_0(blocks)
    elif wtype == ggjt.T_Q8_0:
        w = ggjt.dequantize_q8_0(blocks)
    else:
        raise ValueError("fast mode has no %s path" % ggjt.TYPE_NAME[wtype])
    return w.astype(F16)                                                # exact fp32 product -> one rounding


def file_rows(path: str, name: str, rows: np.ndarray) -> tuple:
    """(fp16 weights of the listed rows of tensor `name`, wtype) straight from a slice file."""
    f = ggjt.read_file(path, sliced=True)
    t = f.tensors[name]
    blk, bsz = ggjt.TYPE_BLOCK[t.ttype]
    k, n_rows = t.ne
    mm = np.memmap(path, dtype=np.uint8, mode="r", offset=t.offset, shape=(n_rows, k // blk, bsz))
    return weights16(np.asarray(mm[rows]), t.ttype), t.ttype


def file_f32(path: str, name: str) -> np.ndarray:
    f = ggjt.read_file(path, sliced=True)
    return np.frombuffer(f.read_raw(name), F32).copy()


_SILU = None


def silu_table() -> np.ndarray:
    """fp16 -> fp16 SiLU, built like build_tables does: f / (1 + expf(-f)) with libm's expf, rounded to fp16."""
    global _SILU
    if _SILU is None:
        libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
        f = np.arange(65536, dtype=np.uint16).view(F16).astype(F32)
        e = np.array([libm.expf(float(-v)) for v in f], F32)
        with np.errstate(over="ignore", invalid="ignore"):
            _SILU = (f / (F32(1) + e).astype(F32)).astype(F32).astype(F16)
    return _SILU


# ---------------------------------------------------------------------------------------------- reference
def reference(w16: np.ndarray, x16: np.ndarray) -> tuple:
    """(sum_k w16 * x16, sum_k |w16 * x16|) in float64: [N][rows] each."""
    w, x = w16.astype(np.float64), x16.astype(np.float64)
    return x @ w.T, np.abs(x) @ np.abs(w).T


def ulp32(y: np.ndarray) -> np.ndarray:
    return np.spacing(np.abs(np.asarray(y, F32))).astype(np.float64)


def store_error(y: np.ndarray, ref: np.ndarray, mag: np.ndarray, resid: np.ndarray = None) -> np.ndarray:
    """Per output: the smallest tau with |y - (ref [+ resid])| <= tau * mag [+ one fp32 ulp of |y| for the residual add]."""
    y = np.asarray(y, F32).astype(np.float64)
    want = ref if resid is None else ref + np.asarray(resid, F32).astype(np.float64)
    err = np.abs(y - want)
    if resid is not None:
        err = np.maximum(err - ulp32(y), 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0, 0.0, err / mag)


SILU_ARGMIN = -1.2784645427610738                 # x / (1 + e^-x) is smallest where 1 + x + e^x = 0


def _gate_inside(y, g, sg, u, su, tau):
    """Is y inside the set fp32(silu16(h) * u') for fp16 h = f2h(g') with |g' - g| <= tau*sg, |u' - u| <= tau*su?
    f2h is monotone, so h lies between the roundings of the two ends of the g interval.  SiLU falls down to its minimum
    at SILU_ARGMIN and rises after it, and the fp16 table keeps that order, so over the interval its extremes are at the
    two ends and, when the interval contains SILU_ARGMIN, the table's smallest entry.  The product's extremes are at
    the corners."""
    tab = silu_table()
    silu_min16 = float(np.nanmin(tab.astype(np.float64)))
    g_lo, g_hi = g - tau * sg, g + tau * sg
    s_a = tab[g_lo.astype(F16).view(np.uint16)].astype(np.float64)
    s_b = tab[g_hi.astype(F16).view(np.uint16)].astype(np.float64)
    s_m = np.where((g_lo < SILU_ARGMIN) & (g_hi > SILU_ARGMIN), np.minimum(s_a, silu_min16), s_a)
    s_lo, s_hi = np.minimum(np.minimum(s_a, s_b), s_m), np.maximum(s_a, s_b)
    u_a, u_b = u - tau * su, u + tau * su
    corners = np.stack([s_lo * u_a, s_lo * u_b, s_hi * u_a, s_hi * u_b])
    slack = ulp32(y)
    return (y >= corners.min(axis=0) - slack) & (y <= corners.max(axis=0) + slack)


def gate_error(y: np.ndarray, g: np.ndarray, sg: np.ndarray, u: np.ndarray, su: np.ndarray) -> np.ndarray:
    """Per output of the FG_GATE epilogue y = fp32(silu16(f2h(g))) * u: the smallest tau (found by bisection, to 0.3 %)
    for which y is inside the bound of `_gate_inside`, with g / u the float64 w1 / w3 dots and sg / su their magnitudes.
    0 when y is reached with the float64 dots themselves; inf when not even tau = 2^-4 reaches it."""
    y = np.asarray(y, F32).astype(np.float64)
    lo = np.full(y.shape, -60.0)
    hi = np.full(y.shape, -4.0)
    exact = _gate_inside(y, g, sg, u, su, 0.0)
    far = ~_gate_inside(y, g, sg, u, su, 2.0 ** -4)
    for _ in range(14):
        mid = 0.5 * (lo + hi)
        ok = _gate_inside(y, g, sg, u, su, 2.0 ** mid)
        hi = np.where(ok, mid, hi)
        lo = np.where(ok, lo, mid)
    return np.where(exact, 0.0, np.where(far, np.inf, 2.0 ** hi))


# ---------------------------------------------------------------------------------------------- sampling
def row_sample(rows: int, tile: int) -> np.ndarray:
    """Every row of the first and the last `tile`-row tile, and in every other tile the rows at one position (which
    cycles with the tile index) of each 8-row group: covers every tile, every 8-row group and every position in it."""
    r = np.arange(rows)
    t = r // tile
    keep = (t == 0) | (t == t[-1]) | (r % 8 == t % 8)
    return r[keep]
