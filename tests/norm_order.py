"""RMSNorm rows whose scale depends on the order of the float64 sum of squares (TEST INFRASTRUCTURE).

The reference (ggml_compute_forward_rms_norm_f32) adds (double)(x_i * x_i) in index order, then takes
mean = (float)(sum / K) and scale = 1.0f / sqrtf(mean + 1e-6f).  A parallel kernel adds the same terms as a tree.  A
witness row makes the two orders give different scales, deterministically:

* a few large entries whose squares bring the sequential sum to exactly K * tie, where tie = f + ulp(f) / 2 is a float32
  rounding tie, so the sequential mean rounds to the even one of f and f + ulp(f);
* tiny entries everywhere else, each square below half an ulp of the running sum ("down": the sequential sum absorbs
  every one after the large entries and stays on the tie, the exact sum lies above it) or between half an ulp and one ulp
  ("up": each rounds the sequential sum up by a whole ulp, the exact sum ends below the tie).

Any order that adds tiny terms together before they meet the large ones lands on the exact sum's side, and its mean
and scale are one float off.  `witness_rows` also makes sure the family's activation quantiser turns the two scales into
different activations: Q8_1 and Q8_K keep a float32 block scale, which almost always moves; Q8_0 rounds its block scale
to fp16 and the F16 matmul rounds every activation to fp16, so there the largest entry is chosen from its allowed range
so that its block's fp16 rounding flips between the two scales.

`certified_mean` restates the kernels' check (rms_scale in kernels.cuh): the tree sum S, a bound B on the distance to
any other order's sum, and the reference's float steps at S - B and S + B with directed rounding.
"""
from __future__ import annotations

import math

import numpy as np

EPS = np.float32(1e-6)
WIDTHS = (256, 512, 800, 3200, 4096, 5120, 6656, 8192)     # n_embd of tiny, tiny128, tiny3b, 3b, 7b, 13b, 30b, 65b
FAMILIES = ("q8_0", "q8_1", "q8_k", "f16")
DIRECTIONS = ("down", "up")
PLACES = ("first", "mid", "last")
N_BIG = 8                                                    # slots for the large entries (unused ones hold 0)


def squares(x: np.ndarray) -> np.ndarray:
    """The terms (double)(x_i * x_i), the product rounded in float32."""
    x = np.asarray(x, np.float32)
    return (x * x).astype(np.float64)


def sequential_sum(t: np.ndarray) -> np.ndarray:
    """Sum of the last axis in index order (add.accumulate is a sequential loop; np.sum is pairwise)."""
    return np.cumsum(np.asarray(t, np.float64), axis=-1)[..., -1]


def fsum(t) -> float:
    """The exact sum, correctly rounded."""
    return math.fsum(np.asarray(t, np.float64).tolist())


def ref_mean(s, k: int):
    return np.float32(np.float64(s) / k)


def ref_scale(s, k: int):
    """ggml's float steps from the sum of squares s of a row of k."""
    return np.float32(1) / np.sqrt(np.float32(ref_mean(s, k) + EPS))


def family_of(wtype) -> str:
    """The activation quantiser in front of a matmul with weights of type wtype (ggjt type id or k-quant mix name)."""
    from distributedllm_b200 import ggjt
    if isinstance(wtype, str) or wtype in (ggjt.T_Q4_K, ggjt.T_Q6_K):
        return "q8_k"
    if wtype in (ggjt.T_Q4_1, ggjt.T_Q5_1):
        return "q8_1"
    if wtype in (ggjt.T_F16, ggjt.T_F32):
        return "f16"
    return "q8_0"


def activations(family: str, x: np.ndarray, scale, norm_w: np.ndarray) -> tuple:
    """What the family's matmul sees of x * scale * norm_w: the activation quantiser of the C restatements, or the fp16
    rounding of the F16 matmul."""
    v = np.ascontiguousarray((np.asarray(x, np.float32) * np.float32(scale)).astype(np.float32) * norm_w, np.float32)
    k = len(v)
    if family == "f16":
        return (v.astype(np.float16).view(np.uint16),)
    if family == "q8_k":
        from kq_port import lib as kq_lib
        q, d, bs = np.empty(k, np.int8), np.empty(k // 256, np.float32), np.empty(k // 16, np.int32)
        kq_lib().orc_quantize_q8_K(v.ctypes.data, k, q.ctypes.data, d.ctypes.data, bs.ctypes.data)
        return q, d.view(np.uint32), bs
    from oracle import oracle
    L = oracle.port_lib()
    q = np.empty(k, np.int8)
    if family == "q8_1":
        d, s = np.empty(k // 32, np.float32), np.empty(k // 32, np.float32)
        L.orc_quant_q8_1(v.ctypes.data, k, q.ctypes.data, d.ctypes.data, s.ctypes.data)
        return q, d.view(np.uint32), s.view(np.uint32)
    d = np.empty(k // 32, np.uint16)
    L.orc_quant_q8_0(v.ctypes.data, k, q.ctypes.data, d.ctypes.data)
    return q, d


def activations_differ(family: str, x, s1, s2, norm_w) -> bool:
    return any((a != b).any() for a, b in zip(activations(family, x, s1, norm_w), activations(family, x, s2, norm_w)))


def _float_squares_down(r: float) -> np.float32:
    """The largest float32 b with fl32(b * b) <= r."""
    b = np.float32(math.sqrt(r))
    while float(b * b) > r:
        b = np.nextafter(b, np.float32(0))
    while float(np.nextafter(b, np.float32(np.inf)) * np.nextafter(b, np.float32(np.inf))) <= r:
        b = np.nextafter(b, np.float32(np.inf))
    return b


def _four_squares(n: int):
    """n as a sum of at most four squares (Lagrange), small n."""
    r = int(math.isqrt(n))
    for a in range(r, -1, -1):
        m = n - a * a
        for b in range(int(math.isqrt(m)), -1, -1):
            m2 = m - b * b
            for c in range(int(math.isqrt(m2)), -1, -1):
                d2 = m2 - c * c
                d = int(math.isqrt(d2))
                if d * d == d2:
                    return [a, b, c, d]
    raise AssertionError(n)


def _position(k: int, where: str) -> int:
    if where == "first":
        return 0
    if where == "mid":                 # across a 32-element block boundary and a 128-element (one warp's) span
        return max(128, (k // 2) // 128 * 128) - 3
    if where == "last":                # inside the last 32-block, with tiny entries after it
        return k - 32 + 1
    raise ValueError(where)


def _tiny(e: int, direction: str) -> np.float32:
    """A tiny entry whose square is exact and lies in (0, 1/2) ulp ("down") or (1/2, 1) ulp ("up") of sums in
    [2^e, 2^(e+1))."""
    ulp_exp = e - 52
    if direction == "down":
        # (11/8)^2 / 4 = 0.47 or (31/32)^2 / 2 = 0.47 ulp
        return np.float32(1.375 * 2.0 ** (ulp_exp // 2 - 1)) if ulp_exp % 2 == 0 else np.float32(0.96875 * 2.0 ** ((ulp_exp - 1) // 2))
    # (7/4)^2 / 4 = 0.77 or (5/4)^2 / 2 = 0.78 ulp
    return np.float32(1.75 * 2.0 ** (ulp_exp // 2 - 1)) if ulp_exp % 2 == 0 else np.float32(1.25 * 2.0 ** ((ulp_exp - 1) // 2))


def _build(k: int, f: np.float32, direction: str, where: str, a0: np.float32):
    """The row for mean candidate f and largest entry a0, or None where a0 does not fit."""
    tie = float(f) + float(np.spacing(f)) / 2
    target = k * tie                                          # exact: tie has 25 significant bits, k < 2^14
    e = math.frexp(target)[1] - 1
    ulp = 2.0 ** (e - 52)
    u = _tiny(e, direction)
    tau = float(u) * float(u)
    p0 = _position(k, where)
    n_suf = k - p0 - N_BIG
    g = target if direction == "down" else target - n_suf * ulp    # the running sum after the large entries
    a = p0 * tau + float(a0 * a0)                            # the prefix sum is exact (few bits per term)
    if not (2.0 ** e <= a <= g):
        return None
    big = [a0]
    r = g - a                                                 # exact: both on the ulp grid of [2^e, 2^(e+1))
    if r != 0 and r < 2.0 ** (e - 29):
        return None
    while r >= 2.0 ** (e - 28):
        b = _float_squares_down(r)
        big.append(b)
        r -= float(b * b)
    q_exp = (e - 52) + ((e - 52) % 2)                         # an even exponent at or above the ulp
    n = r / 2.0 ** q_exp
    if n != int(n):
        return None
    n, cs = int(n), []
    while n > 10000:                                          # integers up to 4095: their squares are exact floats
        cs.append(min(math.isqrt(n), 4095))
        n -= cs[-1] ** 2
    cs += [c for c in _four_squares(n) if c]
    if len(big) + len(cs) > N_BIG:
        return None
    big += [np.float32(c * 2.0 ** (q_exp // 2)) for c in cs]
    x = np.full(k, u, np.float32) * np.where(np.arange(k) % 2 == 0, 1, -1).astype(np.float32)
    x[p0:p0 + N_BIG] = 0
    x[p0:p0 + len(big)] = big
    return x


def _candidates(k, f, where, family, norm_w):
    """Largest entries a0 to try, in a fixed order: for the fp16 families, those that put the fp16 rounding of the a0
    block's scale (Q8_0) or of a0's activation (F16) next to a midpoint; otherwise a few near the top of the range."""
    tie = float(f) + float(np.spacing(f)) / 2
    lo, top = math.sqrt(k * tie * (1 - 2.0 ** -4)), math.sqrt(k * tie * (1 - 2.0 ** -6))
    if family not in ("q8_0", "f16"):
        return [np.float32(top * (1 - j * 2.0 ** -12)) for j in range(8)]
    to_h = float(ref_scale(k * tie, k)) * abs(float(norm_w[_position(k, where)])) / (127.0 if family == "q8_0" else 1.0)
    out = []
    h = np.float16(top * to_h)
    while True:
        h2 = np.nextafter(h, np.float16(0))
        c = np.float32((float(h) + float(h2)) / 2 / to_h)
        if c < lo:
            return out
        out += [np.float32(c + d * np.spacing(c)) for d in range(-3, 4)]
        h = h2


def witness_row(k: int, family: str, norm_w: np.ndarray, direction: str = "down", where: str = "first", skip: int = 0):
    """One witness row of width k (see the module doc).  `skip` picks a later one (another mean candidate f)."""
    norm_w = np.asarray(norm_w, np.float32)
    parity = 0 if direction == "down" else 1                 # down: the tie rounds to f (even); up: to f + ulp
    # k * tie in [1.5, 2) * 2^e with e even: the ulp of the sum is an even power of two, a square
    e = 2 * math.ceil(math.log2(k) / 2)
    base = np.array([1.75 * 2.0 ** e / k], np.float32).view(np.uint32)[0]
    base += (int(base) & 1) ^ parity
    for j in range(1, 400):
        f = np.array([base + 2 * j], np.uint32).view(np.float32)[0]
        tie = float(f) + float(np.spacing(f)) / 2
        s_seq, s_other = ref_scale(k * tie, k), ref_scale(k * tie + (1 if direction == "down" else -1) * k * 2.0 ** -30, k)
        if s_seq == s_other:
            continue
        for a0 in _candidates(k, f, where, family, norm_w):
            x = _build(k, f, direction, where, a0)
            if x is None or not is_witness(x, family, norm_w):
                continue
            if skip == 0:
                return x
            skip -= 1
            break
    raise AssertionError("no witness row for k=%d %s %s %s" % (k, family, direction, where))


def witness_rows(k: int, family: str, norm_w: np.ndarray, direction: str = "down", where: str = "first", n: int = 1):
    return np.stack([witness_row(k, family, norm_w, direction, where, i) for i in range(n)])


def scales(x: np.ndarray) -> tuple:
    """(scale of the sequential sum, scale of the exact sum) of a row."""
    t = squares(x)
    return ref_scale(sequential_sum(t), len(t)), ref_scale(fsum(t), len(t))


def is_witness(x: np.ndarray, family: str, norm_w: np.ndarray) -> bool:
    s_seq, s_exact = scales(x)
    return bool(s_seq != s_exact) and activations_differ(family, x, s_seq, s_exact, norm_w)


# --------------------------------------------------------------------------- the kernels' certification, restated
def _two_sum_err(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = a * 134217729.0                                       # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod_err(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def certified_mean(s, k: int):
    """float32 mean the kernels accept without re-summing, from a sum s of the row's squares in any order, or NaN where
    they re-sum: B = RU(s * k * 0x1.01p-52), the float steps at RD(s - B) and RU(s + B)."""
    s = np.asarray(s, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        p, e = _two_prod_err(s, np.float64(k * 1.00390625 * 2.0 ** -52))
        b = np.where(e > 0, np.nextafter(p, np.inf), p)
        lo, el = _two_sum_err(s, -b)
        lo = np.where(el < 0, np.nextafter(lo, -np.inf), lo)
        hi, eh = _two_sum_err(s, b)
        hi = np.where(eh > 0, np.nextafter(hi, np.inf), hi)
        mlo, mhi = (lo / k).astype(np.float32), (hi / k).astype(np.float32)
    return np.where(mlo == mhi, mlo, np.float32(np.nan))
