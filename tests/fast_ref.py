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


TOKEN_SAMPLE_ABOVE = 512


def token_sample(n: int) -> np.ndarray:
    """The tokens a call of n rows is checked on: all of them up to TOKEN_SAMPLE_ABOVE rows, else row_sample(n, 256) --
    every row of the first and the last 256-token tile (so of the first and last 128-token tile too) and 32 rows of
    every other 256-token tile (so at least 16 of every 128-token tile), which keeps the float64 sums a few seconds."""
    return np.arange(n) if n <= TOKEN_SAMPLE_ABOVE else row_sample(n, 256)


# ---------------------------------------------------------------------------------------------- one layer
class LayerWeights:
    """A row sample of one layer's matrices as fp16 (every row of the first and last 128-row tile of qkv, wo and w2, of
    the first and last 64-row tile of w1 / w3, and one row per 8-row group in the others) and its norm weights."""

    def __init__(self, path: str, layer: int, n_embd: int, n_ff: int):
        E, FF = n_embd, n_ff
        self.layer, self.E, self.FF = layer, E, FF
        self.r_qkv, self.r_e, self.r_ff = row_sample(3 * E, 128), row_sample(E, 128), row_sample(FF, 64)
        pre = "layers.%d." % layer
        self.w_qkv = stacked_rows(path, [pre + "attention.wq.weight", pre + "attention.wk.weight",
                                         pre + "attention.wv.weight"], E, self.r_qkv)
        self.w_o = stacked_rows(path, [pre + "attention.wo.weight"], E, self.r_e)
        self.w_1 = stacked_rows(path, [pre + "feed_forward.w1.weight"], FF, self.r_ff)
        self.w_3 = stacked_rows(path, [pre + "feed_forward.w3.weight"], FF, self.r_ff)
        self.w_2 = stacked_rows(path, [pre + "feed_forward.w2.weight"], E, self.r_e)
        self.attn_norm = file_f32(path, pre + "attention_norm.weight")
        self.ffn_norm = file_f32(path, pre + "ffn_norm.weight")


def stacked_rows(path: str, names, per: int, sample: np.ndarray) -> np.ndarray:
    """fp16 weights of `sample` rows of the matrices `names` stacked by rows (`per` rows each), as the packer stacks them."""
    parts = []
    for i, nm in enumerate(names):
        sel = sample[(sample >= i * per) & (sample < (i + 1) * per)] - i * per
        if len(sel):
            parts.append(file_rows(path, nm, sel)[0])
    return np.concatenate(parts)


def read_layer(gpu, n: int, E: int, FF: int) -> dict:
    """The debug reads of the last layer a fast call of n rows ran: the qkv, att, ffin and gate buffers and xh (w2's
    fp16 input, as uint16)."""
    return {"qkv": gpu.debug_read(0, n * 3 * E).reshape(n, 3 * E),
            "att": gpu.debug_read(1, n * E).reshape(n, E),
            "ffin": gpu.debug_read(2, n * E).reshape(n, E),
            "gate": gpu.debug_read(3, n * FF).reshape(n, FF),
            "xh": gpu.debug_read(9, n * FF // 2, np.uint32).view(np.uint16).reshape(n, FF)}


def check_layer(w: LayerWeights, x: np.ndarray, reads: dict, y: np.ndarray, tau, floor: float, label: str,
                tokens: np.ndarray = None, lost_tokens: int = 1) -> tuple:
    """The four matmuls of one fast-mode layer against the float64 bound, on the rows `tokens` (default: all) of a call.
    x is the layer's input rows, reads what read_layer returned, y the layer's output rows; tau(K) is the bound of a
    matmul with K-wide rows, floor the share of outputs one lost 32-wide K block must move outside it.
      * xh == prep(gate) bit for bit on every row: the activation restatement the bound relies on;
      * per matmul, the largest normalised error |y - y_ref| / sum_k |w16 * x16| over the sampled rows <= tau(K);
      * zeroing activation block (K / 32) / 3 in the reference puts >= floor of the outputs outside the bound (numpy
        only: the bound is tight enough to see one lost block).  lost_tokens = 1 zeroes it in the middle sampled token;
        more zero it in that many sampled tokens spread from the first to the last and pool their outputs, which
        estimates the same share from lost_tokens times as many outputs.
    Returns ({matmul: largest normalised error}, {matmul: share moved by the lost block})."""
    n = x.shape[0]
    tokens = np.arange(n) if tokens is None else np.asarray(tokens)
    assert tokens[0] == 0 and tokens[-1] == n - 1
    qkv, att, ffin, gate, xh = (reads[k] for k in ("qkv", "att", "ffin", "gate", "xh"))
    x_2 = prep(gate)
    bad = int((xh != x_2.view(np.uint16)).sum())
    assert bad == 0, "%s: xh differs from prep(gate) at %d of %d halves" % (label, bad, xh.size)
    tk = tokens
    x_2 = x_2[tk]
    xs, atts, ffins, gates, ys, qkvs = x[tk], att[tk], ffin[tk], gate[tk], y[tk], qkv[tk]
    x_qkv, x_o, x_13 = prep(xs, w.attn_norm), prep(atts), prep(ffins, w.ffn_norm)
    r_qkv, r_e, r_ff = w.r_qkv, w.r_e, w.r_ff
    errs, moved = {}, {}
    t = np.array([len(tk) // 2]) if lost_tokens == 1 else np.unique(np.linspace(0, len(tk) - 1, lost_tokens).astype(int))
    # qkv: plain store
    ref, mag = reference(w.w_qkv, x_qkv)
    errs["qkv"] = store_error(qkvs[:, r_qkv], ref, mag)
    moved["qkv"] = (x_qkv, lambda xm: store_error(qkvs[t][:, r_qkv], *reference(w.w_qkv, xm)))
    # wo: + residual (the layer input)
    ref, mag = reference(w.w_o, x_o)
    errs["wo"] = store_error(ffins[:, r_e], ref, mag, xs[:, r_e])
    moved["wo"] = (x_o, lambda xm: store_error(ffins[t][:, r_e], *reference(w.w_o, xm), xs[t][:, r_e]))
    # w1 | w3: SiLU gate
    g, sg = reference(w.w_1, x_13)
    u, su = reference(w.w_3, x_13)
    errs["w13"] = gate_error(gates[:, r_ff], g, sg, u, su)
    moved["w13"] = (x_13, lambda xm: gate_error(gates[t][:, r_ff], *reference(w.w_1, xm), *reference(w.w_3, xm)))
    # w2: + residual (ffin)
    ref, mag = reference(w.w_2, x_2)
    errs["w2"] = store_error(ys[:, r_e], ref, mag, ffins[:, r_e])
    moved["w2"] = (x_2, lambda xm: store_error(ys[t][:, r_e], *reference(w.w_2, xm), ffins[t][:, r_e]))
    worst = {mat: float(e.max()) for mat, e in errs.items()}
    print("\n[fast-matmul] %s  max normalised error  %s" % (label, "  ".join("%s %.3g" % (m, worst[m]) for m in errs)))
    bound = {mat: tau(w.FF if mat == "w2" else w.E) for mat in errs}
    for mat, e in errs.items():
        assert e.max() <= bound[mat], "%s %s: normalised error %.3g > TAU %.3g at %d outputs" % (
            label, mat, e.max(), bound[mat], int((e > bound[mat]).sum()))
    lost = {}
    for mat, (xa, err_of) in moved.items():
        xm = xa[t].copy()
        blk = (xm.shape[1] // 32) // 3
        xm[:, blk * 32:(blk + 1) * 32] = 0
        outside = err_of(xm) > bound[mat]
        lost[mat] = float(np.mean(outside))
        each = "" if len(t) == 1 else " (%d tokens pooled; per token %.4f .. %.4f)" % (
            len(t), outside.mean(axis=1).min(), outside.mean(axis=1).max())
        print("[fast-matmul] %s  %s: a lost K block moves %.4f of the outputs outside the bound%s" % (
            label, mat, lost[mat], each))
        assert lost[mat] >= floor, "%s %s: a lost K block moves only %.3f of the outputs outside the bound" % (
            label, mat, lost[mat])
    return worst, lost
