"""CPU: the session-state entry points (b200_session_copy / _state_size / _save / _restore, b200_stream_fork) without a
GPU, and capi's argument checks, which refuse bad Python arguments before anything reaches the library."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_entry_points_without_a_device_refuse():
    code = ("import sys, ctypes as C; sys.path.insert(0, %r)\n"
            "from distributedllm_b200 import capi\n"
            "L = capi.lib()\n"
            "d = (C.c_int * 2)(1, 2)\n"
            "n = C.c_size_t(7)\n"
            "buf = (C.c_uint8 * 64)()\n"
            "print('copy', L.b200_session_copy(None, 0, d, 2, 0))\n"
            "print('size', L.b200_session_state_size(None, 0, C.byref(n)), n.value)\n"
            "print('save', L.b200_session_save(None, 0, buf, 64, C.byref(n)), n.value)\n"
            "print('restore', L.b200_session_restore(None, 0, buf, 64))\n"
            "print('fork', L.b200_stream_fork(None, 0, 1, 0))\n"
            "out = C.c_void_p()\n"
            "print('load', L.b200_slice_load_ex(b'/nonexistent.bin', 0, 64, 2, C.byref(out)), out.value)\n" % ROOT)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    lines = out.stdout.splitlines()
    assert lines[:5] == ["copy 1", "size 1 7", "save 1 7", "restore 1", "fork 1"], out.stdout + out.stderr   # B200_EINVAL
    assert lines[5] == "load 3 None", out.stdout + out.stderr                                                  # B200_ENODEV


class _FakeLib:
    """Records the session-state calls that reach it; a saved state is 64 + 4 * n_past bytes of a fixed pattern."""

    def __init__(self):
        self.calls = []

    def b200_slice_load_ex(self, path, device, n_ctx, n_sessions, out):
        out._obj.value = 1
        return 0

    def b200_slice_info(self, h, info):
        info._obj.n_embd = 32
        return 0

    def b200_session_copy(self, h, src, dsts, n_dst, n_keep):
        self.calls.append(("copy", src, C.cast(dsts, C.POINTER(C.c_int))[:n_dst], n_keep))
        return 0

    def b200_session_state_size(self, h, session, n):
        self.calls.append(("size", session))
        n._obj.value = 64 + 4 * 3
        return 0

    def b200_session_save(self, h, session, buf, cap, written):
        self.calls.append(("save", session, cap))
        C.memmove(buf, bytes(range(cap)), cap)
        return 0

    def b200_session_restore(self, h, session, buf, n):
        self.calls.append(("restore", session, C.string_at(buf, n)))
        return 0

    def b200_stream_open(self, handles, n, extra, max_rows, lookahead, out):
        out._obj.value = 1
        return 0

    def b200_stream_fork(self, h, src, dst, n_keep):
        self.calls.append(("fork", src, dst, n_keep))
        return 0

    def b200_stream_close(self, h):
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


def test_slice_state_rejects_bad_arguments_before_the_library(fake):
    from distributedllm_b200 import capi
    sl = capi.Slice("any.bin", 0, 64, n_sessions=4)
    bad_copy = [
        (ValueError, (-1, [1], 0)),
        (TypeError, (0.0, [1], 0)),
        (TypeError, (True, [1], 0)),
        (ValueError, (0, [], 0)),
        (TypeError, (0, 1, 0)),
        (TypeError, (0, "12", 0)),
        (ValueError, (0, [1, -2], 0)),
        (TypeError, (0, [1.0], 0)),
        (ValueError, (0, [1], -1)),
        (TypeError, (0, [1], None)),
        (ValueError, (0, [2 ** 31], 0)),
    ]
    for exc, args in bad_copy:
        with pytest.raises(exc):
            sl.session_copy(*args)
    for exc, arg in ((ValueError, -1), (TypeError, 1.5), (TypeError, None)):
        with pytest.raises(exc):
            sl.session_save(arg)
        with pytest.raises(exc):
            sl.session_restore(arg, b"B2KV")
    for blob in ("B2KV", [1, 2], np.zeros(64, np.uint8), None):
        with pytest.raises(TypeError):
            sl.session_restore(0, blob)
    assert fake.calls == []
    sl.session_copy(0, np.array([3, 1]), 5)
    sl.session_copy(2, (0,), 0)
    blob = sl.session_save(1)
    assert blob == bytes(range(76))
    sl.session_restore(3, blob)
    sl.session_restore(2, bytearray(b"xyz"))
    sl.session_restore(0, b"")
    assert fake.calls == [("copy", 0, [3, 1], 5), ("copy", 2, [0], 0), ("size", 1), ("save", 1, 76),
                          ("restore", 3, blob), ("restore", 2, b"xyz"), ("restore", 0, b"")]


def test_stream_fork_rejects_bad_arguments_before_the_library(fake):
    from distributedllm_b200 import capi
    st = capi.Stream([_Handle()], _Handle())
    for exc, args in ((ValueError, (-1, 1, 0)), (ValueError, (0, -1, 0)), (ValueError, (0, 1, -1)),
                      (TypeError, (0, 1, 2.0)), (TypeError, ("0", 1, 2)), (TypeError, (0, False, 2))):
        with pytest.raises(exc):
            st.fork(*args)
    assert fake.calls == []
    st.fork(0, 3, 17)
    assert fake.calls == [("fork", 0, 3, 17)]
    st.close()
    with pytest.raises(ValueError):
        st.fork(0, 3, 1)                                        # closed: nothing reaches the library
    assert len(fake.calls) == 1


def test_header_declares_the_session_state_entry_points():
    text = open(os.path.join(ROOT, "include", "b200_slice.h")).read()
    for name in ("b200_session_copy", "b200_session_state_size", "b200_session_save", "b200_session_restore",
                 "b200_stream_fork"):
        assert name + "(" in text, name
    assert "does not identify the" in text and "weights" in text
