"""CPU: the host twin of the device's logprobs (client.token_logprobs) against scipy, and the capi logprobs bindings'
argument checks and record unpacking against a fake library."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.special import log_softmax

from distributedllm_b200 import capi
from distributedllm_b200.client import token_logprobs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _want(x, t, n):
    x = np.asarray(x, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = log_softmax(x)
        ref[np.exp(x - x.max()) == 0] = -np.inf          # the client's log(e_t / S): an e_t that underflows gives -inf
    order = np.lexsort((np.arange(len(x)), -x))[:n]
    return ref[t], order, ref[order]


def _close(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same_inf = np.isinf(a) & (a == b)
    with np.errstate(invalid="ignore"):
        return bool(np.all(same_inf | (np.abs(a - b) <= 1e-12 * np.maximum(1.0, np.abs(b)))))


def _rows():
    rng = np.random.default_rng(5)
    rows = [(rng.standard_normal(n) * s).astype(np.float32) for n, s in ((512, 1), (1031, 4), (32000, 3), (7, 0.1))]
    tie = rng.integers(-3, 3, 2000).astype(np.float32)             # a few values, thousands of ties
    rows.append(tie)
    r = rng.standard_normal(300).astype(np.float32)
    r[::3] = -np.inf                                               # -inf entries
    rows.append(r)
    r = np.zeros(100, np.float32)
    r[5] = -1e4                                                    # exp underflows: -inf
    rows.append(r)
    r = np.full(40, -np.inf, np.float32)
    r[[3, 30]] = 2.0                                               # two finite ids among -inf
    rows.append(r)
    return rows


@pytest.mark.parametrize("n_top", [0, 1, 5, 20])
def test_token_logprobs_equal_scipy_and_lexsort(n_top):
    for i, x in enumerate(_rows()):
        n = min(n_top, len(x))
        for t in {0, len(x) - 1, 5 % len(x), int(np.argmax(x))}:
            lp, alts = token_logprobs(x, t, n)
            want, order, want_top = _want(x, t, n)
            assert _close(lp, want), (i, t)
            assert [a for a, _ in alts] == order.tolist(), (i, t)
            assert _close([b for _, b in alts], want_top), (i, t)
            assert [b for a, b in alts if a == t] in ([], [lp])      # the drawn id's lp is the same number in both


def test_greedy_id_ranks_first_and_ties_go_to_the_lower_id():
    x = np.array([1.0, 5.0, 5.0, -2.0, 5.0], np.float32)
    lp, alts = token_logprobs(x, 1, 5)
    assert [a for a, _ in alts] == [1, 2, 4, 0, 3]
    assert alts[0][1] == alts[1][1] == alts[2][1] == lp


def test_underflow_gives_minus_inf():
    x = np.zeros(64, np.float32)
    x[9] = -1e4
    lp, alts = token_logprobs(x, 9, 0)
    assert lp == -np.inf and alts == []


@pytest.mark.parametrize("bad", ["nan", "+inf", "all -inf"])
def test_rows_without_distribution_give_nan_and_minus_one(bad):
    x = np.random.default_rng(1).standard_normal(50).astype(np.float32)
    if bad == "nan":
        x[7] = np.nan
    elif bad == "+inf":
        x[7] = np.inf
    else:
        x[:] = -np.inf
    lp, alts = token_logprobs(x, 3, 4)
    assert np.isnan(lp)
    assert [a for a, _ in alts] == [-1] * 4 and all(np.isnan(b) for _, b in alts)


def test_token_logprobs_argument_checks():
    x = np.zeros(10, np.float32)
    for exc, args in ((ValueError, (x, 10, 0)), (ValueError, (x, -1, 0)), (TypeError, (x, 1.0, 0)),
                      (ValueError, (x, 0, 11)), (ValueError, (x, 0, -1)), (TypeError, (x, 0, True)),
                      (ValueError, (np.zeros(30, np.float32), 0, 21)), (ValueError, (np.zeros(0, np.float32), 0, 0))):
        with pytest.raises(exc):
            token_logprobs(*args)


# ---- capi against a fake library ----------------------------------------------------------------------------------

class _Fake:
    """Implements the logprobs entry points: fills every output it is given and records the calls."""

    def __init__(self):
        self.calls = []

    def b200_generate_lp(self, handles, n_slices, extra, sessions, counts, n_seq, toks, n_steps, sp, ids, lp):
        s = C.cast(lp, C.POINTER(capi.Logprobs)).contents if isinstance(lp, int) else lp._obj
        self.calls.append(("generate_lp", n_seq, n_steps, s.n_top, sp is not None))
        n = n_steps * n_seq
        np.ctypeslib.as_array(C.cast(s.lp, C.POINTER(C.c_double)), (n,))[:] = -1.5
        if s.n_top:
            np.ctypeslib.as_array(C.cast(s.top_ids, C.POINTER(C.c_int32)), (n * s.n_top,))[:] = 7
            np.ctypeslib.as_array(C.cast(s.top_lp, C.POINTER(C.c_double)), (n * s.n_top,))[:] = -0.5
        return 0

    def b200_generate_greedy(self, *args):
        self.calls.append(("generate_greedy",))
        return 0

    def b200_stream_open(self, handles, n, extra, max_rows, lookahead, out):
        out._obj.value = 1
        return 0

    def b200_stream_add_lp(self, h, session, prompt, n_prompt, max_tokens, sp, stops, n_stop, n_top):
        self.calls.append(("add_lp", session, n_top))
        return 0

    def b200_stream_add(self, h, session, prompt, n_prompt, max_tokens, sp, stops, n_stop):
        self.calls.append(("add", session))
        return 0

    def b200_stream_read_lp(self, h, sessions, ids, lp, top_ids, top_lp, cap, n_out):
        """Two records: session 4 with 3 alternatives, session 9 added without logprobs."""
        self.calls.append(("read_lp", cap))
        S = np.ctypeslib.as_array(C.cast(sessions.value, C.POINTER(C.c_int32)), (cap,))
        I = np.ctypeslib.as_array(C.cast(ids.value, C.POINTER(C.c_int32)), (cap,))
        L = np.ctypeslib.as_array(C.cast(lp.value, C.POINTER(C.c_double)), (cap,))
        TI = np.ctypeslib.as_array(C.cast(top_ids.value, C.POINTER(C.c_int32)), (cap, 20))
        TL = np.ctypeslib.as_array(C.cast(top_lp.value, C.POINTER(C.c_double)), (cap, 20))
        S[:2], I[:2], L[:2] = [4, 9], [11, 12], [-0.25, np.nan]
        TI[:2], TL[:2] = -1, np.nan
        TI[0, :3], TL[0, :3] = [11, 3, 8], [-0.25, -2.0, -3.0]
        n_out._obj.value = 2
        return 0

    def b200_stream_close(self, h):
        return 0


class _Handle:
    handle = None
    n_vocab = 100


@pytest.fixture
def fake(monkeypatch):
    f = _Fake()
    monkeypatch.setattr(capi, "lib", lambda: f)
    return f


def test_generate_logprobs_checks_and_shapes(fake):
    for exc, n in ((ValueError, -1), (ValueError, 21), (TypeError, 2.0), (TypeError, True)):
        with pytest.raises(exc):
            capi.generate_greedy([_Handle()], _Handle(), [0, 1], [[1], [2, 3]], 4, logprobs=n)
    small = _Handle()
    small.n_vocab = 8
    with pytest.raises(ValueError):
        capi.generate_greedy([_Handle()], small, [0], [[1]], 4, logprobs=9)     # more than n_vocab alternatives
    assert fake.calls == []
    ids, lp, ti, tl = capi.generate_greedy([_Handle()], _Handle(), [0, 1], [[1], [2, 3]], 4, logprobs=3)
    assert ids.shape == (4, 2) and lp.shape == (4, 2) and ti.shape == (4, 2, 3) and tl.shape == (4, 2, 3)
    assert (lp == -1.5).all() and (ti == 7).all() and (tl == -0.5).all()
    ids, lp, ti, tl = capi.generate_greedy([_Handle()], _Handle(), [0], [[1]], 2, logprobs=0)
    assert ti.shape == (2, 1, 0) and (lp == -1.5).all()
    out = capi.generate_greedy([_Handle()], _Handle(), [0], [[1]], 2)
    assert out.shape == (2, 1)
    assert fake.calls == [("generate_lp", 2, 4, 3, False), ("generate_lp", 1, 2, 0, False), ("generate_greedy",)]


def test_stream_logprobs_checks_and_record_unpacking(fake):
    st = capi.Stream([_Handle()], _Handle())
    for exc, n in ((ValueError, -1), (ValueError, 21), (TypeError, 1.5)):
        with pytest.raises(exc):
            st.add(0, [1], 4, logprobs=n)
    assert fake.calls == []
    st.add(4, [1], 4, logprobs=3)
    st.add(9, [1], 4)
    assert fake.calls == [("add_lp", 4, 3), ("add", 9)]
    recs = st.read_logprobs(8)
    assert fake.calls[-1] == ("read_lp", 8)
    assert recs[0] == (4, 11, -0.25, [(11, -0.25), (3, -2.0), (8, -3.0)])
    assert recs[1][:2] == (9, 12) and np.isnan(recs[1][2]) and recs[1][3] == []
    with pytest.raises((ValueError, TypeError)):
        st.read_logprobs(0)
    st.close()


def test_header_declares_the_logprobs_entry_points():
    text = open(os.path.join(ROOT, "include", "b200_slice.h")).read()
    for name in ("b200_generate_lp", "b200_generate_speculative_lp", "b200_stream_add_lp", "b200_stream_read_lp",
                 "b200_extra_logprobs"):
        assert name + "(" in text, name
    assert "b200_logprobs_t" in text
