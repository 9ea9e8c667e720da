"""CPU: the generation stream's entry points without a GPU, and capi.Stream's argument checks, which refuse bad Python
arguments before anything reaches the library."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_stream_open_without_a_device_is_enodev():
    code = ("import sys, ctypes as C; sys.path.insert(0, %r)\n"
            "from distributedllm_b200 import capi\n"
            "L = capi.lib()\n"
            "h = (C.c_void_p * 1)(1)\n"
            "out = C.c_void_p()\n"
            "print('code', L.b200_stream_open(h, 1, C.c_void_p(1), 0, 0, C.byref(out)), out.value)\n" % ROOT)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert "code 3 None" in out.stdout, out.stdout + out.stderr      # B200_ENODEV, no stream


class _FakeLib:
    """Records the stream calls that reach it."""

    def __init__(self):
        self.calls = []

    def b200_stream_open(self, handles, n, extra, max_rows, lookahead, out):
        self.calls.append(("open", max_rows, lookahead))
        out._obj.value = 1
        return 0

    def b200_stream_add(self, h, session, prompt, n_prompt, max_tokens, sp, stops, n_stop):
        self.calls.append(("add", session, n_prompt, max_tokens, n_stop))
        return 0

    def b200_stream_read(self, h, sessions, ids, cap, n_out):
        self.calls.append(("read", cap))
        n_out._obj.value = 0
        return 0

    def b200_stream_cancel(self, h, session):
        self.calls.append(("cancel", session))
        return 0

    def b200_stream_close(self, h):
        self.calls.append(("close",))
        return 0


class _Handle:
    handle = None
    n_vocab = 100


@pytest.fixture
def fake(monkeypatch):
    from distributedllm_b200 import capi
    f = _FakeLib()
    monkeypatch.setattr(capi, "lib", lambda: f)
    return f


def test_stream_rejects_bad_arguments_before_the_library(fake):
    from distributedllm_b200 import capi
    with pytest.raises(ValueError):
        capi.Stream([], _Handle())
    with pytest.raises(TypeError):
        capi.Stream([_Handle()], _Handle(), max_rows=1.5)
    with pytest.raises(TypeError):
        capi.Stream([_Handle()], _Handle(), lookahead="4")
    assert fake.calls == []
    st = capi.Stream([_Handle()], _Handle(), max_rows=16, lookahead=2)
    assert fake.calls == [("open", 16, 2)]
    bad = [
        (ValueError, dict(session=-1)),
        (TypeError, dict(session=1.0)),
        (TypeError, dict(session=True)),
        (ValueError, dict(prompt=[])),
        (TypeError, dict(prompt="the")),
        (TypeError, dict(prompt=5)),
        (ValueError, dict(prompt=[1, 100])),
        (ValueError, dict(prompt=[-1])),
        (TypeError, dict(prompt=[1.5])),
        (ValueError, dict(max_tokens=0)),
        (TypeError, dict(max_tokens=None)),
        (ValueError, dict(stop_ids=[100])),
        (TypeError, dict(stop_ids=2)),
        (ValueError, dict(temperature=-0.5)),
        (ValueError, dict(temperature=float("nan"))),
        (ValueError, dict(temperature=float("inf"))),
        (ValueError, dict(temperature=0.7, repeat_penalty=0.0)),
        (ValueError, dict(temperature=0.7, repeat_penalty=float("nan"))),
        (ValueError, dict(temperature=0.7, seed=-1)),
        (ValueError, dict(temperature=0.7, seed=2 ** 64)),
        (ValueError, dict(temperature=0.7, first_draw=-1)),
        (ValueError, dict(temperature=0.7, history=[3, 100])),
        (TypeError, dict(temperature=0.7, history=7)),
        (ValueError, dict(history=[3])),                       # history without a temperature (greedy)
        (ValueError, dict(first_draw=2)),
    ]
    for exc, kw in bad:
        args = dict(session=0, prompt=[1, 2], max_tokens=4)
        args.update(kw)
        with pytest.raises(exc):
            st.add(**args)
    assert fake.calls == [("open", 16, 2)]
    st.add(0, np.array([1, 2, 99]), 4, temperature=0.7, seed=2 ** 64 - 1, history=[5], stop_ids=[2])
    st.add(1, [7], 1)
    assert fake.calls[1:] == [("add", 0, 3, 4, 1), ("add", 1, 1, 1, 0)]
    for kw in (dict(cap=0), dict(cap=2.0)):
        with pytest.raises((ValueError, TypeError)):
            st.read(**kw)
    with pytest.raises(ValueError):
        st.cancel(-3)
    assert st.read(8) == [] and list(st) == []
    st.cancel(1)
    st.close()
    st.close()                                                 # a second close is a no-op
    assert fake.calls[3:] == [("read", 8), ("read", 1), ("cancel", 1), ("close",)]
    with pytest.raises(ValueError):
        st.add(0, [1], 1)                                      # closed: nothing reaches the library
    with pytest.raises(ValueError):
        st.read()
    assert len(fake.calls) == 7
    with capi.Stream([_Handle()], _Handle()) as st2:
        assert isinstance(st2, capi.Stream)
    assert fake.calls[-1] == ("close",)


def test_header_declares_the_stream_entry_points():
    text = open(os.path.join(ROOT, "include", "b200_slice.h")).read()
    for name in ("b200_stream_open", "b200_stream_add", "b200_stream_read", "b200_stream_cancel", "b200_stream_close"):
        assert name + "(" in text, name
    assert "one thread" in text
