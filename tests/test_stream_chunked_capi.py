"""CPU: capi.Stream's prefill_chunk plumbing without a GPU.  0 opens the stream with b200_stream_open exactly as before
(so libraries without b200_stream_open_ex still work); C > 0 goes to b200_stream_open_ex; bad values never reach the
library."""
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _FakeLib:
    """Records the open calls that reach it."""

    def __init__(self):
        self.calls = []

    def b200_stream_open(self, handles, n, extra, max_rows, lookahead, out):
        self.calls.append(("open", max_rows, lookahead))
        out._obj.value = 1
        return 0

    def b200_stream_open_ex(self, handles, n, extra, max_rows, lookahead, prefill_chunk, out):
        self.calls.append(("open_ex", max_rows, lookahead, prefill_chunk))
        out._obj.value = 1
        return 0

    def b200_stream_stats(self, h, steps, rows, most_rows):
        self.calls.append(("stats",))
        steps._obj.value, rows._obj.value, most_rows._obj.value = 3, 40, 17
        return 0

    def b200_stream_close(self, h):
        self.calls.append(("close",))
        return 0


class _OldLib(_FakeLib):
    """A library from before prefill_chunk: no b200_stream_open_ex."""
    b200_stream_open_ex = None


class _Handle:
    handle = None
    n_vocab = 100


@pytest.fixture
def fake(monkeypatch):
    from distributedllm_b200 import capi
    f = _FakeLib()
    monkeypatch.setattr(capi, "lib", lambda: f)
    return f


def test_prefill_chunk_selects_the_entry_point(fake):
    from distributedllm_b200 import capi
    with capi.Stream([_Handle()], _Handle(), max_rows=16, lookahead=2) as st:
        pass
    with capi.Stream([_Handle()], _Handle(), max_rows=16, lookahead=2, prefill_chunk=0):
        pass
    with capi.Stream([_Handle()], _Handle(), max_rows=24, lookahead=3, prefill_chunk=8) as st:
        assert st.stats() == {"steps": 3, "rows": 40, "most_rows": 17}
    with capi.Stream([_Handle()], _Handle(), prefill_chunk=1):
        pass
    assert fake.calls == [("open", 16, 2), ("close",), ("open", 16, 2), ("close",),
                          ("open_ex", 24, 3, 8), ("stats",), ("close",), ("open_ex", 0, 0, 1), ("close",)]


def test_prefill_chunk_zero_needs_no_open_ex(monkeypatch):
    from distributedllm_b200 import capi
    f = _OldLib()
    monkeypatch.setattr(capi, "lib", lambda: f)
    with capi.Stream([_Handle()], _Handle(), max_rows=8):
        pass
    assert f.calls == [("open", 8, 0), ("close",)]


@pytest.mark.parametrize("exc, value", [(ValueError, -1), (ValueError, -2 ** 31), (ValueError, 2 ** 31),
                                        (TypeError, 1.0), (TypeError, "8"), (TypeError, None), (TypeError, True)])
def test_prefill_chunk_is_checked_before_the_library(fake, exc, value):
    from distributedllm_b200 import capi
    with pytest.raises(exc):
        capi.Stream([_Handle()], _Handle(), max_rows=16, prefill_chunk=value)
    assert fake.calls == []


def test_header_declares_the_chunked_entry_points():
    text = open(os.path.join(ROOT, "include", "b200_slice.h")).read()
    for name in ("b200_stream_open_ex", "b200_stream_stats"):
        assert name + "(" in text, name
