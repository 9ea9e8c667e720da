"""GPU on RMSNorm rows whose scale depends on the order of the float64 sum of squares (tests/norm_order.py), bit for bit
against the C restatement and, where oracle/_ref is built, the reference itself.  Every norm site is reached:

* single-token steps, graphed and not (k_gemv's ring prologue), and without the ring (B200_RING=0, the plain prologue);
* prompt chunks, batched steps, mixed passes and decode rows (k_norm_quant, k_gemv_f16_mc, k_quant_q8k);
* the grid-barrier norm+quant epilogue (B200_NQ=1: the ffn norm in wo, the next layer's attention norm in w2);
* the F16 kernels (ring, multi-column with 4 and 8 columns, the ring-less single column, K % 256 != 0);
* the lm_head of every output type.

The slices are rewritten so that the norm under test sees the witness row itself (edge_cases "no_v": the first layer's
ffn norm; "pass": the second layer's attention norm; unmodified: the first layer's attention norm)."""
import os
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt
from oracle import oracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import edge_cases as ec  # noqa: E402
import norm_order as no  # noqa: E402
from test_gpu_numeric_edges import _bad, _Checkers  # noqa: E402
from test_oracle_edges import _fid  # noqa: E402

pytestmark = pytest.mark.gpu

FAMILIES = [("tiny", ggjt.T_Q4_0), ("tiny128", ggjt.T_Q4_1), ("tiny3b", ggjt.T_Q5_0), ("tiny", ggjt.T_Q5_1),
            ("tiny128", ggjt.T_Q8_0), ("tiny", ggjt.T_F16), ("tiny3b", ggjt.T_F16), ("tinyk", "q4_K_S"),
            ("tinyk128", "q4_K_M"), ("tinyk", "q6_K")]
# recipe -> the norm weight (tensor of the slice file) that sees the witness row
RECIPES = {"none": "layers.%d.attention_norm.weight", "no_v": "layers.%d.ffn_norm.weight",
           "pass": "layers.%d.attention_norm.weight"}


def _slice(tmp, shape, wtype, recipe, layers=None):
    sh = ggjt.SHAPES[shape]
    layers = layers or ((2, 3) if isinstance(wtype, str) else (0, 1))
    src = os.path.join(tmp, "%s_%s.bin" % (shape, wtype))
    if not os.path.exists(src):
        if isinstance(wtype, str):
            ggjt.write_kquant_slice(src, sh, layers[0], layers[1], wtype, seed=4)
        else:
            ggjt.write_synth_slice(src, sh, layers[0], layers[1], wtype, seed=4)
    path = src if recipe == "none" else ec.rewrite(src, src[:-4] + "_" + recipe + ".bin", recipe)
    f = ggjt.read_file(path, sliced=True)
    layer = f.hparams.first_layer + (1 if recipe == "pass" else 0)
    w = np.frombuffer(f.read_raw(RECIPES[recipe] % layer), np.float32).copy()
    # the layer's matmul behind that norm decides the quantiser: wq (attention) or w1 (ffn)
    mat = "layers.%d.%s" % (layer, "feed_forward.w1.weight" if recipe == "no_v" else "attention.wq.weight")
    return path, w, no.family_of(f.tensors[mat].ttype)


def _witness(k, fam, w, n=6):
    rows = [no.witness_row(k, fam, w, d, where, i) for i in range((n + 5) // 6) for d in no.DIRECTIONS for where in no.PLACES]
    return np.stack(rows[:n])


def _run(path, wtype, x, schedule, tag):
    """A fresh context: the rows of x fed in calls of `schedule` sizes, each against the checkers."""
    from distributedllm_b200 import capi
    gpu, chk = capi.Slice(path, 0, 64), _Checkers(path, wtype, 64)
    bad = []
    try:
        r0 = 0
        for i, n in enumerate(schedule):
            rows = x[r0:r0 + n]
            r0 += n
            y = gpu.forward(rows)
            for j, want in enumerate(chk.forward(rows)):
                if _bad(y, want):
                    bad.append((tag, i, n, j, _bad(y, want)))
    finally:
        gpu.close()
        chk.close()
    return bad


SCHEDULE = (9, 1, 1, 1, 1, 1, 1, 2, 3)          # a prompt chunk, single-token steps, short chunks


@pytest.mark.parametrize("recipe", list(RECIPES))
@pytest.mark.parametrize("family", FAMILIES, ids=_fid)
def test_witness_rows_prompt_and_steps(tmp_path, family, recipe):
    shape, wtype = family
    path, w, fam = _slice(str(tmp_path), shape, wtype, recipe)
    x = _witness(ggjt.SHAPES[shape].n_embd, fam, w, sum(SCHEDULE))
    bad = _run(path, wtype, x, SCHEDULE, (family, recipe))
    assert not bad, bad


SWITCHES = [{"B200_GRAPH": "0"}, {"B200_RING": "0"}, {"B200_NQ": "1"}, {"B200_F16_MC": "0"}, {"B200_F16_MC": "8"},
            {"B200_F16_RING": "0"}]
SWITCH_FAMILIES = [("tiny", ggjt.T_Q4_0), ("tiny128", ggjt.T_Q4_1), ("tiny", ggjt.T_Q5_1), ("tiny128", ggjt.T_F16),
                   ("tiny3b", ggjt.T_F16), ("tinyk128", "q4_K_M")]


CASES = [(f, e) for f in SWITCH_FAMILIES for e in SWITCHES if f[1] == ggjt.T_F16 or not any("F16" in k for k in e)]


@pytest.mark.parametrize("family,env", CASES, ids=lambda c: _fid(c) if isinstance(c, tuple) else "-".join("%s=%s" % kv for kv in c.items()))
def test_witness_rows_under_switches(tmp_path, monkeypatch, family, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    shape, wtype = family
    bad = []
    for recipe in RECIPES:
        path, w, fam = _slice(str(tmp_path), shape, wtype, recipe)
        x = _witness(ggjt.SHAPES[shape].n_embd, fam, w, 12)
        bad += _run(path, wtype, x, (4, 1, 1, 6), (family, env, recipe))
    assert not bad, bad


@pytest.mark.parametrize("family", [("tiny", ggjt.T_Q4_1), ("tiny", ggjt.T_F16), ("tinyk128", "q4_K_M")], ids=_fid)
def test_witness_row_among_ordinary_rows_batched_and_mixed(tmp_path, family):
    """One witness row beside ordinary rows of other sessions, in batched steps, mixed passes and decode rows."""
    from distributedllm_b200 import capi
    shape, wtype = family
    k = ggjt.SHAPES[shape].n_embd
    path, w, fam = _slice(str(tmp_path), shape, wtype, "none")
    wit = _witness(k, fam, w, 12)
    rng = np.random.default_rng(3)
    gpu = capi.Slice(path, 0, 64, n_sessions=3)
    chk = [_Checkers(path, wtype, 64) for _ in range(3)]
    it = iter(wit)
    try:
        for place in range(3):
            rows = [rng.standard_normal((1, k), dtype=np.float32) for _ in range(3)]
            rows[place] = next(it)[None]
            y = gpu.batch_forward([0, 1, 2], np.concatenate(rows))
            for j in range(3):
                assert all(_bad(y[j:j + 1], c) == 0 for c in chk[j].forward(rows[j])), ("batch", place, j)
        counts = [3, 1, 2]
        xs = [rng.standard_normal((c, k), dtype=np.float32) for c in counts]
        xs[0][1], xs[1][0], xs[2][1] = next(it), next(it), next(it)
        y = gpu.mixed_forward([0, 1, 2], counts, np.concatenate(xs))
        r0 = 0
        for j, c in enumerate(counts):
            assert all(_bad(y[r0:r0 + c], want) == 0 for want in chk[j].forward(xs[j])), ("mixed", j)
            r0 += c
        x = np.concatenate([next(it)[None], rng.standard_normal((2, k), dtype=np.float32), next(it)[None]])
        y = gpu.forward_steps(1, x)
        for i in range(len(x)):
            for want in chk[1].forward(x[i:i + 1]):
                assert _bad(y[i:i + 1], want) == 0, ("steps", i)
    finally:
        gpu.close()
        for c in chk:
            c.close()


@pytest.mark.parametrize("shape", ["7b", "13b", "30b", "65b"])
@pytest.mark.parametrize("wtype", [ggjt.T_Q4_0, "q4_K_M"], ids=["q4_0", "q4_K_M"])
def test_witness_rows_one_large_layer(tmp_path, shape, wtype):
    """One layer at real widths (real tile counts, ring wrap), a 1-token call and a 9-token call."""
    sh = ggjt.SHAPES[shape]
    path = str(tmp_path / "l.bin")
    if wtype == "q4_K_M":
        ggjt.write_kquant_slice(path, sh, 0, 0, "q4_K_M", seed=3)
    else:
        ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=3)
    w = ec.slice_norm(path)
    x = _witness(sh.n_embd, no.family_of(wtype), w, 10)
    bad = _run(path, wtype, x, (1, 9), (shape, wtype))
    assert not bad, bad


OUTPUTS = [ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0, ggjt.T_F16, ggjt.T_Q4_K]


@pytest.mark.parametrize("wtype", OUTPUTS, ids=lambda t: "q6_K" if t == ggjt.T_Q4_K else ggjt.TYPE_NAME[t])
def test_witness_rows_lm_head(tmp_path, wtype):
    """Extra.logits of 1, 8 and 9 rows and Extra.next_token (Q4_K files carry a Q6_K output.weight)."""
    from distributedllm_b200 import capi
    path = ec.make_extra(str(tmp_path), wtype)
    f = ggjt.read_file(path, sliced=True)
    out_t = f.tensors["output.weight"].ttype
    w = np.frombuffer(f.read_raw("norm.weight"), np.float32).copy()
    x = _witness(f.hparams.n_embd, no.family_of(out_t), w, 9)
    want = [ec.port_logits(path, x)]
    if oracle.have_ref():
        want.append(oracle.ref_logits(path, x, f.hparams.n_vocab, True))
    extra = capi.Extra(path, 0)
    try:
        for rows in (x[:1], x[:8], x):
            got = extra.logits(rows)
            for wl in want:
                assert _bad(got, wl[:len(rows)]) == 0, (len(rows), _bad(got, wl[:len(rows)]))
        for i in range(len(x)):
            assert extra.next_token(x[i:i + 1]) == int(np.argmax(want[0][i])), i
    finally:
        extra.close()
