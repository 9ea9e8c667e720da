"""CPU: llama.cpp's classifier-free guidance (llama_sample_classifier_free_guidance) and its host twin client.cfg_logits.

* With libm's expf / logf the twin equals the compiled reference (oracle/_ref/cfg_shim, built by oracle/cfg.mk) bit for
  bit, NaN positions included, on random rows, rows whose spread makes lb underflow (sf 1 gives NaN there), rows where lb
  and lg underflow at one index (the whole row NaN), ties for the max and values where one FMA and a multiply-add round
  differently.
* With correctly rounded expf / logf (the device's) a row can differ from libm's only where libm's result on an argument
  the row evaluates is not the correctly rounded one.
* The guidance arguments the C ABI refuses before it touches a handle, on a process without a device."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from distributedllm_b200.client import _exp_f32, _fma_f32, _log_f32, cfg_greedy, cfg_logits

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SHIM = os.path.join(ROOT, "oracle", "_ref", "cfg_shim")
N_VOCAB = ggjt.SHAPES["tiny"].n_vocab
SETTINGS = [(1.5, 1.0), (3.0, 0.5), (1.0001, 0.0), (7.25, -0.75)]

_libm = C.CDLL("libm.so.6")
_libm.expf.restype = _libm.logf.restype = C.c_float
_libm.expf.argtypes = _libm.logf.argtypes = [C.c_float]


def libm_expf(v):
    v = np.asarray(v, np.float32)
    return np.array([_libm.expf(float(x)) for x in v.ravel()], np.float32).reshape(v.shape)


def libm_logf(v):
    v = np.asarray(v, np.float32)
    return np.array([_libm.logf(float(x)) for x in v.ravel()], np.float32).reshape(v.shape)


def cases():
    """-> (base, guidance) float32 [n][N_VOCAB], one pair per edge listed in the module docstring."""
    rng = np.random.default_rng(7)
    n = N_VOCAB
    b, g = [], []
    for s in (1.0, 3.0, 8.0):                                           # random rows
        b.append(rng.standard_normal(n) * s)
        g.append(rng.standard_normal(n) * s)
    x = rng.standard_normal(n) * 2                                       # spread > 104: lb underflows at a few ids
    x[rng.choice(n, 9, replace=False)] -= 150
    b.append(x)
    g.append(rng.standard_normal(n))
    x, y = rng.standard_normal(n), rng.standard_normal(n)                # both underflow at id 5: lg2 all NaN
    x[5] -= 200
    y[5] -= 300
    b.append(x)
    g.append(y)
    x = rng.standard_normal(n)                                           # ties for the max in every row
    x[[3, 40, 300]] = 6.0
    y = rng.standard_normal(n)
    y[[0, 77]] = 5.0
    b.append(x)
    g.append(y)
    b.append(np.round(rng.standard_normal(n) * 4, 1))                    # coarse values: many equal outputs
    g.append(np.round(rng.standard_normal(n) * 4, 1))
    return np.array(b, np.float32), np.array(g, np.float32)


def run_shim(base, guid, scale, sf):
    with tempfile.TemporaryDirectory() as d:
        model, rows, out = (os.path.join(d, f) for f in ("m.bin", "rows.bin", "out.bin"))
        ggjt.write_synth_full(model, ggjt.SHAPES["tiny"], ggjt.T_Q4_0, seed=0)
        np.concatenate([base, guid]).astype(np.float32).tofile(rows)
        subprocess.run([SHIM, model, rows, out, repr(scale), repr(sf)], check=True, capture_output=True, timeout=300)
        return np.fromfile(out, np.float32).reshape(base.shape)


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.where(np.isnan(a), 0, a).view(np.uint32),
                                                                       np.where(np.isnan(b), 0, b).view(np.uint32))


@pytest.mark.skipif(not os.path.isfile(SHIM), reason="oracle/_ref/cfg_shim not built")
@pytest.mark.parametrize("scale,sf", SETTINGS)
def test_twin_with_libm_equals_the_reference(scale, sf):
    base, guid = cases()
    want = run_shim(base, guid, scale, sf)
    got = cfg_logits(base, guid, scale, sf, expf=libm_expf, logf=libm_logf)
    for k in range(len(base)):
        assert same_bits(got[k], want[k]), "row %d" % k
        assert cfg_greedy(got[k]) == cfg_greedy(want[k])


def test_edges_are_reached():
    """The cases hold what they claim: NaN at underflowed ids for sf 1, an all-NaN row, and FMAs that a multiply-add
    would round differently."""
    base, guid = cases()
    out = cfg_logits(base, guid, 1.5, 1.0)
    assert 0 < np.isnan(out[3]).sum() < N_VOCAB
    assert np.isnan(out[4]).all() and cfg_greedy(out[4]) == 0
    assert not np.isnan(out[0]).any()
    # mix_i = fmaf(scale, lb - lg, lg) against scale * (lb - lg) + lg rounded twice
    with np.errstate(all="ignore"):
        lb = np.log(np.exp(base[0].astype(np.float64) - base[0].max()) / np.exp(base[0].astype(np.float64) - base[0].max()).sum())
        lg = np.log(np.exp(guid[0].astype(np.float64) - guid[0].max()) / np.exp(guid[0].astype(np.float64) - guid[0].max()).sum())
    lb, lg = lb.astype(np.float32), lg.astype(np.float32)
    d = lb - lg
    assert (_fma_f32(np.float32(1.5), d, lg) != np.float32(1.5) * d + lg).any()


def test_greedy_is_max_element():
    nan = np.float32("nan")
    assert cfg_greedy(np.array([nan, 1, 2], np.float32)) == 0
    assert cfg_greedy(np.array([1, nan, 2, 2], np.float32)) == 2
    assert cfg_greedy(np.array([-np.inf, nan, -np.inf], np.float32)) == 0
    assert cfg_greedy(np.array([-0.0, 0.0], np.float32)) == 0


def _recording(fn, exact, seen):
    def f(v):
        r = fn(v)
        seen.append(int((r.view(np.uint32) != exact(v).view(np.uint32)).sum() - (np.isnan(r) & np.isnan(exact(v))).sum()))
        return r
    return f


def test_correctly_rounded_twin_differs_only_where_libm_is_not():
    base, guid = cases()
    for scale, sf in SETTINGS[:2]:
        for k in range(len(base)):
            seen = []
            libm = cfg_logits(base[k:k + 1], guid[k:k + 1], scale, sf, expf=_recording(libm_expf, _exp_f32, seen),
                              logf=_recording(libm_logf, _log_f32, seen))
            exact = cfg_logits(base[k:k + 1], guid[k:k + 1], scale, sf)
            if not same_bits(libm, exact):
                assert sum(seen) > 0, "row %d differs though libm was correctly rounded on every argument" % k


def _abi(code: str) -> str:
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    prog = ("import sys, ctypes as C; sys.path.insert(0, %r)\n"
            "from distributedllm_b200 import capi\n"
            "L = capi.lib()\n"
            "def show(rc): print('code', rc, L.b200_last_error().decode())\n" % ROOT) + code
    out = subprocess.run([sys.executable, "-c", prog], env=env, capture_output=True, text=True, timeout=120)
    return out.stdout + out.stderr


def test_abi_refusals_without_a_device():
    out = _abi(
        "h = (C.c_void_p * 1)(1); s = (C.c_int * 1)(0); c = (C.c_int * 1)(1); t = (C.c_int32 * 1)(0)\n"
        "ids = (C.c_int32 * 4)()\n"
        "gs = (C.c_int * 1)(1)\n"
        "def g(scale, sf): return capi.Guidance(C.cast(gs, C.c_void_p), C.cast(c, C.c_void_p), C.cast(t, C.c_void_p), scale, sf)\n"
        "show(L.b200_generate_cfg(h, 1, C.c_void_p(1), s, c, 1, t, 2, None, None, ids, None))\n"
        "show(L.b200_generate_cfg(None, 1, C.c_void_p(1), s, c, 1, t, 2, C.byref(g(2.0, 1.0)), None, ids, None))\n"
        "for sc, sf in ((1.0, 1.0), (0.5, 1.0), (float('nan'), 1.0), (float('inf'), 1.0), (2.0, float('nan')), (2.0, float('-inf'))):\n"
        "    show(L.b200_generate_cfg(h, 1, C.c_void_p(1), s, c, 1, t, 2, C.byref(g(sc, sf)), None, ids, None))\n"
        "f = (C.c_float * 4)(); o = (C.c_float * 4)()\n"
        "show(L.b200_extra_cfg(C.c_void_p(1), f, f, 1, C.c_float(1.0), C.c_float(1.0), o, None))\n"
        "show(L.b200_extra_cfg(C.c_void_p(1), f, f, 1, C.c_float(2.0), C.c_float(float('inf')), o, None))\n"
        "show(L.b200_extra_cfg(C.c_void_p(1), f, f, 0, C.c_float(2.0), C.c_float(1.0), o, None))\n")
    lines = [l for l in out.splitlines() if l.startswith("code")]
    assert lines == [
        "code 1 b200_generate_cfg: null guidance",
        "code 1 b200_generate_cfg: null argument or empty list",
        "code 1 guidance scale must be finite and > 1 (got 1): at 1 guidance is off, so do not ask for it",
        "code 1 guidance scale must be finite and > 1 (got 0.5): at 1 guidance is off, so do not ask for it",
        "code 1 guidance scale must be finite and > 1 (got nan): at 1 guidance is off, so do not ask for it",
        "code 1 guidance scale must be finite and > 1 (got inf): at 1 guidance is off, so do not ask for it",
        "code 1 guidance smooth_factor must be finite (got nan)",
        "code 1 guidance smooth_factor must be finite (got -inf)",
        "code 1 guidance scale must be finite and > 1 (got 1): at 1 guidance is off, so do not ask for it",
        "code 1 guidance smooth_factor must be finite (got inf)",
        "code 1 b200_extra_cfg: null argument or no rows",
    ], out


def test_python_guidance_arguments():
    from distributedllm_b200 import capi
    with pytest.raises(TypeError):
        capi._guidance(1, ([1], [[2]], 2.0))
    with pytest.raises(ValueError):
        capi._guidance(2, ([1], [[2]], 2.0, 1.0))
    g, keep = capi._guidance(2, ([3, 4], [[5], [6, 7]], 2.0, 0.5))
    assert (keep[1] == [1, 2]).all() and (keep[2] == [5, 6, 7]).all() and g.scale == 2.0 and g.smooth_factor == 0.5


@pytest.mark.skipif(not os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "main")), reason="oracle/_ref/main not built")
def test_fixture_is_what_main_prints():
    import json
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import gen_golden_cfg as gen
    with open(os.path.join(HERE, "golden", "cfg_main.json")) as f:
        fx = json.load(f)
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "full.bin")
        assert gen.write_model(model) == fx["model_sha256"]
        for case in fx["cases"]:
            p, n, text = gen.run_main(model, case["scale"], case["smooth_factor"])
            assert (p, n, text) == (fx["prompt_ids"], fx["negative_ids"], case["text"])
