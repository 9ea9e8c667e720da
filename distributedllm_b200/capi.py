"""ctypes binding of libb200slice.so (include/b200_slice.h).  No torch, no CPU fallback:
importing works anywhere, every call needs an H100."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200slice.so")

ERRORS = {1: "EINVAL", 2: "EFILE", 3: "ENODEV", 4: "ECUDA", 5: "ECONTEXT", 6: "ENCCL"}


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("b200 error %d (%s): %s" % (code, ERRORS.get(code, "?"), msg))
        self.code = code


class SliceInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_embd", "n_head", "n_ff", "n_layer", "first_layer", "n_ctx", "n_past",
                                          "weight_type", "device")] + [("weight_bytes", C.c_int64),
                                                                        ("kv_bytes_per_pos", C.c_int64)]


class Sampling(C.Structure):
    """b200_sampling_t."""
    _fields_ = [("temperature", C.c_double), ("repeat_penalty", C.c_double), ("seeds", C.c_void_p),
                ("first_draw", C.c_int64), ("history", C.c_void_p), ("history_counts", C.c_void_p),
                ("top_k", C.c_int32), ("top_p", C.c_double)]


class Logprobs(C.Structure):
    """b200_logprobs_t."""
    _fields_ = [("n_top", C.c_int32), ("lp", C.c_void_p), ("top_ids", C.c_void_p), ("top_lp", C.c_void_p)]


MAX_TOP = 20            # the most alternatives a logprobs call returns per id (OpenAI's top_logprobs cap)

_lib: Optional[C.CDLL] = None


class Guidance(C.Structure):
    _fields_ = [("sessions", C.c_void_p), ("prompt_counts", C.c_void_p), ("prompt_tokens", C.c_void_p),
                ("scale", C.c_float), ("smooth_factor", C.c_float)]


def lib() -> C.CDLL:
    """Load the native library; raises if it has not been built (there is no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise ImportError("libb200slice.so is not built: run `python -m distributedllm_b200.build`")
        L = C.CDLL(LIB_PATH)
        vp, ci, cf = C.c_void_p, C.c_int, C.c_float
        L.b200_last_error.restype = C.c_char_p
        L.b200_version.restype = C.c_char_p
        L.b200_slice_load.argtypes = [C.c_char_p, ci, ci, C.POINTER(vp)]
        L.b200_slice_load_ex.argtypes = [C.c_char_p, ci, ci, ci, C.POINTER(vp)]
        if hasattr(L, "b200_slice_load_lora"):
            L.b200_slice_load_lora.argtypes = [C.c_char_p, ci, ci, ci, C.c_char_p, C.c_char_p, C.POINTER(vp)]
        L.b200_session_count.argtypes = [vp]
        L.b200_session_n_past.argtypes = [vp, ci]
        L.b200_session_clear.argtypes = [vp, ci]
        L.b200_session_rewind.argtypes = [vp, ci, ci]
        L.b200_session_forward.argtypes = [vp, ci, vp, ci, vp]
        L.b200_session_forward_device.argtypes = [vp, ci, vp, ci, vp, ci]
        L.b200_batch_forward.argtypes = [vp, vp, ci, vp, vp]
        L.b200_batch_forward_device.argtypes = [vp, vp, ci, vp, vp, ci]
        L.b200_mixed_forward.argtypes = [vp, vp, vp, ci, vp, vp]
        L.b200_mixed_forward_device.argtypes = [vp, vp, vp, ci, vp, vp, ci]
        L.b200_slice_unload.argtypes = [vp]
        L.b200_slice_clear.argtypes = [vp]
        L.b200_slice_rewind.argtypes = [vp, ci]
        L.b200_slice_info.argtypes = [vp, C.POINTER(SliceInfo)]
        L.b200_slice_forward.argtypes = [vp, vp, ci, vp]
        L.b200_slice_forward_device.argtypes = [vp, vp, ci, vp, ci]
        L.b200_slice_sync.argtypes = [vp]
        L.b200_slice_last_ms.argtypes = [vp]
        L.b200_slice_last_ms.restype = cf
        L.b200_slice_launch_count.argtypes = [vp]
        L.b200_slice_launch_count.restype = C.c_int64
        L.b200_slice_set_fast_prefill.argtypes = [vp, ci, ci]
        L.b200_slice_mark.argtypes = [vp, ci]
        L.b200_slice_mark_elapsed_ms.argtypes = [vp]
        L.b200_slice_mark_elapsed_ms.restype = cf
        L.b200_slice_profile.argtypes = [vp, ci]
        L.b200_slice_profile_read.argtypes = [vp, vp, vp, ci]
        L.b200_debug_read.argtypes = [vp, ci, C.c_size_t, C.c_size_t, vp]
        L.b200_debug_weights.argtypes = [vp, ci, ci, C.c_size_t, C.c_size_t, vp, C.POINTER(C.c_size_t)]
        L.b200_debug_trace_enable.argtypes = [vp, ci]
        L.b200_debug_skip_attention.argtypes = [vp, ci]
        L.b200_debug_trace_read.argtypes = [vp, vp, vp, vp, ci]
        L.b200_slice_dev_in.argtypes = [vp]
        L.b200_slice_dev_in.restype = vp
        L.b200_slice_dev_out.argtypes = [vp]
        L.b200_slice_dev_out.restype = vp
        L.b200_pipeline_result.argtypes = [vp]
        L.b200_pipeline_result.restype = vp
        L.b200_device_init.argtypes = [ci]
        for name, args in (("b200_pipeline_unique_id", [vp]), ("b200_pipeline_init", [vp, ci, ci, vp]),
                           ("b200_pipeline_step", [vp, vp, ci, ci]),
                           ("b200_pipeline_mailbox_export", [vp, vp]), ("b200_pipeline_mailbox_connect", [vp, vp, ci]),
                           ("b200_pipeline_collect", [vp, ci, vp]), ("b200_pipeline_pingpong", [vp, ci, ci, vp]), ("b200_pipeline_transport", [vp]), ("b200_pipeline_set_transport", [vp, ci]), ("b200_pipeline_error", [vp]),
                           ("b200_pipeline_step_session", [vp, ci, vp, ci, ci]), ("b200_pipeline_step_batch", [vp, vp, ci, vp, ci]),
                           ("b200_pipeline_step_mixed", [vp, vp, vp, ci, vp, ci]), ("b200_pipeline_destroy", [vp]),
                           ("b200_extra_load", [C.c_char_p, ci, C.POINTER(vp)]), ("b200_extra_unload", [vp]),
                           ("b200_extra_dims", [vp, C.POINTER(ci), C.POINTER(ci)]),
                           ("b200_extra_embed", [vp, vp, ci, vp]), ("b200_extra_logits", [vp, vp, ci, ci, vp]),
                           ("b200_extra_next_token", [vp, vp, ci, C.POINTER(C.c_int32)]),
                           ("b200_extra_tokenize", [vp, C.c_char_p, vp, ci]),
                           ("b200_generate_greedy", [vp, ci, vp, vp, vp, ci, vp, ci, vp]),
                           ("b200_generate_sample", [vp, ci, vp, vp, vp, ci, vp, ci, vp, vp]),
                           ("b200_generate_speculative", [vp, ci, vp, ci, vp, ci, vp, ci, vp, ci, ci, ci, vp, vp, vp]),
                           ("b200_session_forward_steps", [vp, ci, vp, ci, vp]),
                           ("b200_session_forward_steps_device", [vp, ci, vp, ci, vp, ci]),
                           ("b200_extra_sample", [vp, vp, ci, vp, vp]),
                           ("b200_score", [vp, ci, vp, vp, vp, ci, vp, vp]), ("b200_extra_nll", [vp, vp, ci, vp, vp]),
                           ("b200_perplexity_windows", [vp, ci, vp, vp, ci, vp, ci, ci, ci, ci, vp]),
                           ("b200_extra_ppl_terms", [vp, vp, ci, vp, vp]),
                           ("b200_stream_open", [vp, ci, vp, ci, ci, C.POINTER(vp)]),
                           ("b200_stream_add", [vp, ci, vp, ci, ci, vp, vp, ci]),
                           ("b200_stream_read", [vp, vp, vp, ci, C.POINTER(ci)]),
                           ("b200_stream_cancel", [vp, ci]), ("b200_stream_close", [vp]),
                           ("b200_generate_lp", [vp, ci, vp, vp, vp, ci, vp, ci, vp, vp, vp]),
                           ("b200_generate_speculative_lp", [vp, ci, vp, ci, vp, ci, vp, ci, vp, ci, ci, ci, vp, vp, vp, vp]),
                           ("b200_extra_logprobs", [vp, vp, ci, vp, ci, vp, vp, vp]),
                           ("b200_generate_cfg", [vp, ci, vp, vp, vp, ci, vp, ci, vp, vp, vp, vp]),
                           ("b200_extra_cfg", [vp, vp, vp, ci, cf, cf, vp, vp]),
                           ("b200_stream_add_cfg", [vp, ci, vp, ci, ci, vp, vp, ci, ci, ci, vp, ci, cf, cf]),
                           ("b200_stream_add_lp", [vp, ci, vp, ci, ci, vp, vp, ci, ci]),
                           ("b200_stream_read_lp", [vp, vp, vp, vp, vp, vp, ci, C.POINTER(ci)]),
                           ("b200_stream_fork", [vp, ci, ci, ci]),
                           ("b200_stream_open_ex", [vp, ci, vp, ci, ci, ci, C.POINTER(vp)]),
                           ("b200_stream_stats", [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(ci)]),
                           ("b200_session_copy", [vp, ci, vp, ci, ci]),
                           ("b200_session_state_size", [vp, ci, C.POINTER(C.c_size_t)]),
                           ("b200_session_save", [vp, ci, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
                           ("b200_session_restore", [vp, ci, vp, C.c_size_t])):
            if hasattr(L, name):
                getattr(L, name).argtypes = args
        if hasattr(L, "b200_extra_token_text"):
            L.b200_extra_token_text.argtypes = [vp, C.c_int32, C.POINTER(ci)]
            L.b200_extra_token_text.restype = C.POINTER(C.c_char)
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise B200Error(rc, (lib().b200_last_error() or b"").decode("utf-8", "replace"))


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


class Slice:
    """One slice resident on one GPU (mirrors llm.load_slice / propagate_forward / clear_context)."""

    def __init__(self, path: str, device: int = 0, n_ctx: int = 0, n_sessions: int = 1, lora: Optional[str] = None,
                 lora_base: Optional[str] = None):
        """lora: a `ggla` adapter merged into the weights at load (b200_slice_load_lora); lora_base: the F16 / F32 slice
        file whose matrices the adapted ones are computed from (llama.cpp's --lora-base)."""
        if lora_base is not None and lora is None:
            raise ValueError("lora_base needs lora")
        self._h = C.c_void_p()
        if lora is None:
            check(lib().b200_slice_load_ex(os.fsencode(path), device, n_ctx, n_sessions, C.byref(self._h)))
        else:
            check(lib().b200_slice_load_lora(os.fsencode(path), device, n_ctx, n_sessions, os.fsencode(lora),
                                             None if lora_base is None else os.fsencode(lora_base), C.byref(self._h)))
        self.info = self._info()
        self.n_sessions = n_sessions

    # ---- sessions / batched steps (additive API, include/b200_slice.h) ----
    def session_forward(self, session: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        check(lib().b200_session_forward(self._h, session, _ptr(x), x.shape[0], _ptr(out)))
        return out

    def forward_steps(self, session: int, x: np.ndarray) -> np.ndarray:
        """Decode rows (b200_session_forward_steps): the rows of x as single-token steps of `session`, in one pass;
        bit-identical to one session_forward call per row."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        check(lib().b200_session_forward_steps(self._h, session, _ptr(x), x.shape[0], _ptr(out)))
        return out

    def batch_forward(self, sessions, x: np.ndarray) -> np.ndarray:
        """One token for each listed session: x is [len(sessions)][n_embd]."""
        ids = np.ascontiguousarray(sessions, dtype=np.int32)
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(len(ids), self.n_embd)
        out = np.empty_like(x)
        check(lib().b200_batch_forward(self._h, _ptr(ids), len(ids), _ptr(x), _ptr(out)))
        return out

    def batch_forward_device(self, sessions, d_in: int, d_out: int, sync: bool = False) -> None:
        ids = np.ascontiguousarray(sessions, dtype=np.int32)
        check(lib().b200_batch_forward_device(self._h, _ptr(ids), len(ids), C.c_void_p(d_in), C.c_void_p(d_out), int(sync)))

    def mixed_forward(self, sessions, counts, x: np.ndarray) -> np.ndarray:
        """counts[k] tokens of sessions[k] in one pass: x is [sum(counts)][n_embd], rows grouped by session in list order."""
        ids = np.ascontiguousarray(sessions, dtype=np.int32)
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        if len(cnt) != len(ids):
            raise ValueError("need one count per listed session")
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        if x.shape[0] != int(cnt.astype(np.int64).sum()):
            raise ValueError("need sum(counts) rows of n_embd floats")
        check(lib().b200_mixed_forward(self._h, _ptr(ids), _ptr(cnt), len(ids), _ptr(x), _ptr(out)))
        return out

    def mixed_forward_device(self, sessions, counts, d_in: int, d_out: int, sync: bool = False) -> None:
        ids = np.ascontiguousarray(sessions, dtype=np.int32)
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        if len(cnt) != len(ids):
            raise ValueError("need one count per listed session")
        check(lib().b200_mixed_forward_device(self._h, _ptr(ids), _ptr(cnt), len(ids), C.c_void_p(d_in), C.c_void_p(d_out), int(sync)))

    def pipeline_step_mixed(self, sessions, counts, d_in: Optional[int], ring: int = 1) -> None:
        """One mixed pass through the layer-slice pipeline (every rank passes the same lists)."""
        ids = np.ascontiguousarray(sessions, dtype=np.int32)
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        if len(cnt) != len(ids):
            raise ValueError("need one count per listed session")
        check(lib().b200_pipeline_step_mixed(self._h, _ptr(ids), _ptr(cnt), len(ids), C.c_void_p(d_in), ring))

    def session_n_past(self, session: int) -> int:
        return lib().b200_session_n_past(self._h, session)

    def session_clear(self, session: int = -1) -> None:
        check(lib().b200_session_clear(self._h, session))

    def session_rewind(self, session: int, n_past: int) -> None:
        check(lib().b200_session_rewind(self._h, session, n_past))

    def session_copy(self, src: int, dsts, n_keep: int) -> None:
        """Rows [0, n_keep) of session src's KV cache to every session in dsts (b200_session_copy), whose positions become
        n_keep: each then continues bit for bit as src would from n_keep."""
        src = _int("src", src, 0, 2 ** 31 - 1)
        if isinstance(dsts, (str, bytes)) or not hasattr(dsts, "__len__"):
            raise TypeError("dsts must be a sequence of sessions")
        d = np.array([_int("dsts[%d]" % i, k, 0, 2 ** 31 - 1) for i, k in enumerate(dsts)] or [0], np.int32)
        if len(dsts) < 1:
            raise ValueError("dsts needs at least one session")
        n_keep = _int("n_keep", n_keep, 0, 2 ** 31 - 1)
        check(lib().b200_session_copy(self._h, src, _ptr(d), len(dsts), n_keep))

    def session_save(self, session: int) -> bytes:
        """The session's state (b200_session_save): a 64-byte header, then its K and V rows [0, n_past) in fp16."""
        session = _int("session", session, 0, 2 ** 31 - 1)
        n = C.c_size_t()
        check(lib().b200_session_state_size(self._h, session, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        check(lib().b200_session_save(self._h, session, _ptr(buf), n.value, None))
        return buf.tobytes()

    def session_restore(self, session: int, blob) -> None:
        """Set the session's rows and position from a session_save blob of a slice of the same shape
        (b200_session_restore)."""
        session = _int("session", session, 0, 2 ** 31 - 1)
        if not isinstance(blob, (bytes, bytearray, memoryview)):
            raise TypeError("blob must be bytes, bytearray or memoryview, got %s" % type(blob).__name__)
        buf = np.frombuffer(blob, np.uint8) if len(blob) else np.zeros(1, np.uint8)
        check(lib().b200_session_restore(self._h, session, _ptr(buf), len(blob)))

    def _info(self) -> SliceInfo:
        i = SliceInfo()
        check(lib().b200_slice_info(self._h, C.byref(i)))
        return i

    @property
    def n_embd(self) -> int:
        return self.info.n_embd

    @property
    def n_past(self) -> int:
        return self._info().n_past

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def forward(self, x: np.ndarray) -> np.ndarray:
        """HOST buffers in and out: [n_tokens][n_embd] float32."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        check(lib().b200_slice_forward(self._h, _ptr(x), x.shape[0], _ptr(out)))
        return out

    def forward_device(self, d_in: int, n_tokens: int, d_out: int, sync: bool = False) -> None:
        check(lib().b200_slice_forward_device(self._h, C.c_void_p(d_in), n_tokens, C.c_void_p(d_out), int(sync)))

    def sync(self) -> None:
        check(lib().b200_slice_sync(self._h))

    def clear_context(self) -> None:
        check(lib().b200_slice_clear(self._h))

    def rewind(self, n_past: int) -> None:
        check(lib().b200_slice_rewind(self._h, n_past))

    @property
    def dev_in(self) -> int:
        return lib().b200_slice_dev_in(self._h)

    @property
    def dev_out(self) -> int:
        return lib().b200_slice_dev_out(self._h)

    @property
    def pipeline_result(self) -> int:
        """Device pointer of the step's final activation: dev_out, or on rank 0 of a ring pipeline the last slice's output."""
        return lib().b200_pipeline_result(self._h)

    def set_fast_prefill(self, on: bool, min_tokens: int = 0) -> None:
        check(lib().b200_slice_set_fast_prefill(self._h, int(on), min_tokens))

    def mark(self, which: int) -> None:
        check(lib().b200_slice_mark(self._h, which))

    def mark_elapsed_ms(self) -> float:
        return float(lib().b200_slice_mark_elapsed_ms(self._h))

    def profile(self, enable: bool) -> None:
        check(lib().b200_slice_profile(self._h, int(enable)))

    def profile_read(self):
        ms = np.zeros(7, np.float32)
        cnt = np.zeros(7, np.int32)
        check(lib().b200_slice_profile_read(self._h, _ptr(ms), _ptr(cnt), 7))
        return ms, cnt

    def debug_read(self, which: int, count: int, dtype=np.float32) -> np.ndarray:
        out = np.zeros(count, np.uint32)
        check(lib().b200_debug_read(self._h, which, 0, count, _ptr(out)))
        return out.view(dtype)

    def debug_weights(self, layer: int, which: int) -> np.ndarray:
        """Packed device bytes of one matrix (b200_debug_weights): qkv / wo / w13 / w2 (0..3), or wq .. w3 (0..6) of an
        F16 slice.  A test hook; nothing on a serving path calls it."""
        n = C.c_size_t(0)
        check(lib().b200_debug_weights(self._h, layer, which, 0, 0, None, C.byref(n)))
        out = np.zeros(n.value, np.uint8)
        if n.value:
            check(lib().b200_debug_weights(self._h, layer, which, 0, n.value, _ptr(out), None))
        return out

    def skip_attention(self, on: bool) -> None:
        check(lib().b200_debug_skip_attention(self._h, int(on)))

    def trace_enable(self, on: bool) -> None:
        check(lib().b200_debug_trace_enable(self._h, int(on)))

    def trace_read(self, max_launches: int = 512):
        """-> (stamps [n][ctas][8] uint64 ns, class ids [n], cta counts [n])"""
        buf = np.zeros((max_launches, 1024, 8), np.uint64)
        cls = np.zeros(max_launches, np.int32)
        ctas = np.zeros(max_launches, np.int32)
        n = lib().b200_debug_trace_read(self._h, _ptr(buf), _ptr(cls), _ptr(ctas), max_launches)
        return buf[:n], cls[:n], ctas[:n]

    def last_ms(self) -> float:
        return float(lib().b200_slice_last_ms(self._h))

    def launch_count(self) -> int:
        return int(lib().b200_slice_launch_count(self._h))

    def close(self) -> None:
        if self._h:
            check(lib().b200_slice_unload(self._h))
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Extra:
    """The client-side extra layers (tokenizer, tok_embeddings, norm, output) resident on one GPU."""

    def __init__(self, path: str, device: int = 0):
        self._h = C.c_void_p()
        check(lib().b200_extra_load(os.fsencode(path), device, C.byref(self._h)))
        self.device = device
        v, e = C.c_int(), C.c_int()
        check(lib().b200_extra_dims(self._h, C.byref(v), C.byref(e)))
        self.n_vocab, self.n_embd = v.value, e.value

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def tokenize(self, prompt: str) -> list:
        text = prompt.encode("utf-8")
        n = lib().b200_extra_tokenize(self._h, text, None, 0)
        if n < 0:
            check(-n)
        out = np.zeros(max(n, 1), np.int32)
        lib().b200_extra_tokenize(self._h, text, _ptr(out), n)
        return out[:n].tolist()

    def embed(self, tokens) -> np.ndarray:
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        out = np.empty((len(t), self.n_embd), np.float32)
        check(lib().b200_extra_embed(self._h, _ptr(t), len(t), _ptr(out)))
        return out

    def logits(self, x: np.ndarray) -> np.ndarray:
        """[n][n_embd] hidden states -> [n][n_vocab] logits (final RMSNorm + output.weight)."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty((x.shape[0], self.n_vocab), np.float32)
        check(lib().b200_extra_logits(self._h, _ptr(x), x.shape[0], 1, _ptr(out)))
        return out

    def next_token(self, x: np.ndarray) -> int:
        """Argmax of the last row's logits (first maximum wins)."""
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        tok = C.c_int32()
        check(lib().b200_extra_next_token(self._h, _ptr(x), x.shape[0], C.byref(tok)))
        return tok.value

    def token_text(self, token_id: int) -> str:
        """llm.decode_token: the token's text (invalid UTF-8 replaced)."""
        n = C.c_int()
        p = lib().b200_extra_token_text(self._h, int(token_id), C.byref(n))
        if not p:
            raise IndexError("token id %d out of range" % token_id)
        return C.string_at(p, n.value).decode("utf-8", "replace")

    def sample(self, logits: np.ndarray, temperature: float, repeat_penalty: float, seeds, first_draw: int = 0,
               history=None, top_k: int = 0, top_p: float = 0.0) -> np.ndarray:
        """The client's Sampler on the device (b200_extra_sample): row k of [n][n_vocab] logits takes draw first_draw of
        the Philox stream keyed seeds[k], with history[k] (ids already sampled) penalised, truncated to top_k / top_p
        (0: off).  -> [n] ids."""
        x = np.ascontiguousarray(logits, dtype=np.float32).reshape(-1, self.n_vocab)
        sp, keep = _sampling(len(x), temperature, repeat_penalty, seeds, first_draw, history, top_k, top_p)
        out = np.zeros(len(x), np.int32)
        check(lib().b200_extra_sample(self._h, _ptr(x), len(x), C.byref(sp), _ptr(out)))
        return out

    def nll(self, logits: np.ndarray, targets) -> np.ndarray:
        """The client's perplexity term on the device (b200_extra_nll): -log softmax(row k)[targets[k]] in float64 for
        each row of [n][n_vocab] logits.  -> [n] float64."""
        x = np.ascontiguousarray(logits, dtype=np.float32).reshape(-1, self.n_vocab)
        t = np.ascontiguousarray(targets, dtype=np.int32)
        if len(t) != len(x):
            raise ValueError("need one target per row (%d), got %d" % (len(x), len(t)))
        out = np.zeros(len(x), np.float64)
        check(lib().b200_extra_nll(self._h, _ptr(x), len(x), _ptr(t), _ptr(out)))
        return out

    def ppl_terms(self, logits: np.ndarray, targets) -> np.ndarray:
        """llama.cpp's perplexity term on the device (b200_extra_ppl_terms): -logf(softmax(row k)[targets[k]]) with the
        float exps summed in double in index order (client.ppl_terms is the host twin).  -> [n] float32."""
        x = np.ascontiguousarray(logits, dtype=np.float32).reshape(-1, self.n_vocab)
        t = np.ascontiguousarray(targets, dtype=np.int32)
        if len(t) != len(x):
            raise ValueError("need one target per row (%d), got %d" % (len(x), len(t)))
        out = np.zeros(len(x), np.float32)
        check(lib().b200_extra_ppl_terms(self._h, _ptr(x), len(x), _ptr(t), _ptr(out)))
        return out

    def logprobs(self, logits: np.ndarray, ids, n_top: int):
        """k_logprob_rows on the device (b200_extra_logprobs): for each row of [n][n_vocab] logits, log softmax(row)[ids[k]]
        in float64 and the n_top ids of largest logit (equal logits: lower id first) with theirs.
        -> (lp [n], top_ids [n][n_top], top_lp [n][n_top])."""
        x = np.ascontiguousarray(logits, dtype=np.float32).reshape(-1, self.n_vocab)
        t = np.ascontiguousarray(ids, dtype=np.int32)
        if len(t) != len(x):
            raise ValueError("need one id per row (%d), got %d" % (len(x), len(t)))
        n_top = _n_top(n_top, self.n_vocab)
        out = _LpOut((len(x),), n_top)
        check(lib().b200_extra_logprobs(self._h, _ptr(x), len(x), _ptr(t), n_top, _ptr(out.lp), _ptr(out.top_ids),
                                        _ptr(out.top_lp)))
        return out.lp, out.top_ids, out.top_lp

    def cfg(self, base: np.ndarray, guidance: np.ndarray, scale: float, smooth_factor: float):
        """llama.cpp's classifier-free guidance on the device (b200_extra_cfg) for each row pair of [n][n_vocab] logits
        (client.cfg_logits is the host twin).  -> (out float32 [n][n_vocab], greedy ids [n])."""
        b = np.ascontiguousarray(base, dtype=np.float32).reshape(-1, self.n_vocab)
        g = np.ascontiguousarray(guidance, dtype=np.float32).reshape(-1, self.n_vocab)
        if g.shape != b.shape:
            raise ValueError("need one guidance row per base row (%d), got %d" % (len(b), len(g)))
        out = np.zeros_like(b)
        greedy = np.zeros(len(b), np.int32)
        check(lib().b200_extra_cfg(self._h, _ptr(b), _ptr(g), len(b), float(scale), float(smooth_factor), _ptr(out),
                                   _ptr(greedy)))
        return out, greedy

    def close(self) -> None:
        if self._h:
            check(lib().b200_extra_unload(self._h))
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _n_top(n_top, n_vocab: int) -> int:
    return _int("logprobs", n_top, 0, min(MAX_TOP, n_vocab))


class _LpOut:
    """The output arrays of a logprobs call for ids of `shape`, and the b200_logprobs_t that points into them."""

    def __init__(self, shape, n_top: int):
        self.lp = np.full(shape, np.nan, np.float64)
        self.top_ids = np.full(tuple(shape) + (n_top,), -1, np.int32)
        self.top_lp = np.full(tuple(shape) + (n_top,), np.nan, np.float64)
        self.c = Logprobs(n_top, self.lp.ctypes.data, self.top_ids.ctypes.data if n_top else None,
                          self.top_lp.ctypes.data if n_top else None)


def _guidance(n: int, guidance):
    """guidance = (sessions, negative prompts, scale, smooth_factor) -> (b200_guidance_t, the arrays it points into)."""
    try:
        sessions, prompts, scale, smooth_factor = guidance
    except (TypeError, ValueError):
        raise TypeError("guidance must be (sessions, negative prompts, scale, smooth_factor)") from None
    gs = np.ascontiguousarray(sessions, dtype=np.int32)
    if len(gs) != n or len(prompts) != n:
        raise ValueError("need one guidance session and one negative prompt per listed session (%d)" % n)
    counts = np.array([len(p) for p in prompts], np.int32)
    toks = np.ascontiguousarray([int(t) for p in prompts for t in p] or [0], dtype=np.int32)
    return Guidance(gs.ctypes.data, counts.ctypes.data, toks.ctypes.data, float(scale), float(smooth_factor)), [gs, counts, toks]


def _generate_cfg(slices, extra, ids, counts, toks, n_steps, guidance, sp, logprobs):
    """b200_generate_cfg for generate_greedy (sp None) and generate_sample."""
    g, keep = _guidance(len(ids), guidance)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    out = np.zeros((max(n_steps, 0), len(ids)), np.int32)
    lp = _LpOut(out.shape, _n_top(logprobs, extra.n_vocab)) if logprobs is not None else None
    check(lib().b200_generate_cfg(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks), n_steps,
                                  C.byref(g), C.byref(sp) if sp is not None else None, _ptr(out),
                                  C.byref(lp.c) if lp is not None else None))
    return out if lp is None else (out, lp.lp, lp.top_ids, lp.top_lp)


def generate_greedy(slices, extra: Extra, sessions, prompts, n_steps: int, logprobs: Optional[int] = None, guidance=None):
    """Greedy decoding on the device (b200_generate_greedy): session sessions[k] is fed prompts[k] (a list of token ids),
    then n_steps - 1 of its own ids.  `slices` are in layer order, all on the extra layers' GPU.  -> [n_steps][n_seq] ids.
    logprobs = n_top (0..20): b200_generate_lp instead, -> (ids, lp [n_steps][n_seq], top_ids and top_lp
    [n_steps][n_seq][n_top]) in the raw distribution (include/b200_slice.h).
    guidance = (guidance sessions, negative prompts, scale, smooth_factor): classifier-free guidance (b200_generate_cfg),
    guidance session k fed negative prompt k, then session k's ids."""
    ids = np.ascontiguousarray(sessions, dtype=np.int32)
    if len(prompts) != len(ids):
        raise ValueError("need one prompt per listed session")
    counts = np.array([len(p) for p in prompts], np.int32)
    toks = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int64) for p in prompts]) if len(prompts) else [],
                                dtype=np.int32)
    if guidance is not None:
        return _generate_cfg(slices, extra, ids, counts, toks, n_steps, guidance, None, logprobs)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    out = np.zeros((max(n_steps, 0), len(ids)), np.int32)
    if logprobs is not None:
        lp = _LpOut(out.shape, _n_top(logprobs, extra.n_vocab))
        check(lib().b200_generate_lp(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks),
                                     n_steps, None, _ptr(out), C.byref(lp.c)))
        return out, lp.lp, lp.top_ids, lp.top_lp
    check(lib().b200_generate_greedy(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks),
                                     n_steps, _ptr(out)))
    return out


def _truncation(top_k, top_p):
    """top_k as an int in [0, 2^31), top_p as a float >= 0 (inf allowed: no cut), or ValueError / TypeError."""
    top_k = _int("top_k", top_k, 0, 2 ** 31 - 1)
    if isinstance(top_p, (bool, np.bool_)) or not isinstance(top_p, (int, float, np.integer, np.floating)):
        raise TypeError("top_p must be a number, got %r" % (top_p,))
    top_p = float(top_p)
    if not top_p >= 0:
        raise ValueError("top_p must be >= 0 and not NaN, got %r" % top_p)
    return top_k, top_p


def _sampling(n: int, temperature: float, repeat_penalty: float, seeds, first_draw: int, history, top_k=0, top_p=0.0):
    """-> (b200_sampling_t, the arrays it points into)."""
    top_k, top_p = _truncation(top_k, top_p)
    keys = np.ascontiguousarray([int(k) for k in seeds], dtype=np.uint64)
    if len(keys) != n:
        raise ValueError("need one seed per session (%d), got %d" % (n, len(keys)))
    sp = Sampling(float(temperature), float(repeat_penalty), keys.ctypes.data, int(first_draw), None, None, top_k, top_p)
    keep = [keys]
    if history is not None:
        if len(history) != n:
            raise ValueError("need one history per session (%d), got %d" % (n, len(history)))
        counts = np.array([len(h) for h in history], np.int32)
        ids = np.ascontiguousarray([int(t) for h in history for t in h] or [0], dtype=np.int32)
        sp.history, sp.history_counts = ids.ctypes.data, counts.ctypes.data
        keep += [counts, ids]
    return sp, keep


def generate_sample(slices, extra: Extra, sessions, prompts, n_steps: int, temperature: float, repeat_penalty: float,
                    seeds, first_draw: int = 0, history=None, top_k: int = 0, top_p: float = 0.0,
                    logprobs: Optional[int] = None, guidance=None):
    """Sampled generation on the device (b200_generate_sample): generate_greedy's loop with the client's Sampler in place
    of the argmax.  Session sessions[k] draws from numpy.random.Philox(key=seeds[k]) starting at draw first_draw, with
    history[k] (ids it sampled before) penalised and every row truncated to top_k / top_p (0: off).
    -> [n_steps][n_seq] ids; with logprobs = n_top, (ids, lp, top_ids, top_lp) as generate_greedy.  guidance as
    generate_greedy: the Sampler draws from the guided rows."""
    ids = np.ascontiguousarray(sessions, dtype=np.int32)
    if len(prompts) != len(ids):
        raise ValueError("need one prompt per listed session")
    sp, keep = _sampling(len(ids), temperature, repeat_penalty, seeds, first_draw, history, top_k, top_p)
    counts = np.array([len(p) for p in prompts], np.int32)
    toks = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int64) for p in prompts]) if len(prompts) else [],
                                dtype=np.int32)
    if guidance is not None:
        return _generate_cfg(slices, extra, ids, counts, toks, n_steps, guidance, sp, logprobs)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    out = np.zeros((max(n_steps, 0), len(ids)), np.int32)
    if logprobs is not None:
        lp = _LpOut(out.shape, _n_top(logprobs, extra.n_vocab))
        check(lib().b200_generate_lp(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks),
                                     n_steps, C.byref(sp), _ptr(out), C.byref(lp.c)))
        return out, lp.lp, lp.top_ids, lp.top_lp
    check(lib().b200_generate_sample(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks),
                                     n_steps, C.byref(sp), _ptr(out)))
    return out


class SpecStats(C.Structure):
    _fields_ = [("passes", C.c_int32), ("drafted", C.c_int32), ("accepted", C.c_int32)]


def generate_speculative(slices, extra: Extra, session: int, draft_slices, draft_extra: Extra, draft_session: int, prompt,
                         n_steps: int, n_draft: int, temperature: Optional[float] = None, repeat_penalty: float = 1.1,
                         seed: Optional[int] = None, first_draw: int = 0, history=None, top_k: int = 0, top_p: float = 0.0,
                         logprobs: Optional[int] = None):
    """Speculative decoding on the device (b200_generate_speculative): the draft chain proposes n_draft ids per
    iteration, one pass of the target checks them.  temperature None: greedy, the ids of generate_greedy; else the ids of
    generate_sample with the same settings (seed: the session's Philox key; history: the ids it sampled before).
    -> (ids [n_steps] int32, {"passes", "drafted", "accepted"}); with logprobs = n_top (b200_generate_speculative_lp),
    ((ids, lp [n_steps], top_ids, top_lp [n_steps][n_top]), stats), equal to the plain loop's."""
    toks = np.ascontiguousarray([int(t) for t in prompt], dtype=np.int32)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    dhandles = (C.c_void_p * max(len(draft_slices), 1))(*[s.handle for s in draft_slices])
    sp, keep = None, []
    if temperature is not None:
        if seed is None:
            raise ValueError("sampled speculative generation needs a seed")
        sp, keep = _sampling(1, temperature, repeat_penalty, [seed], first_draw, None if history is None else [history],
                             top_k, top_p)
    out = np.zeros(max(n_steps, 0), np.int32)
    stats = SpecStats()
    args = (handles, len(slices), extra.handle, session, dhandles, len(draft_slices), draft_extra.handle, draft_session,
            _ptr(toks), len(toks), n_steps, n_draft, C.byref(sp) if sp is not None else None, _ptr(out), C.byref(stats))
    lp = None
    if logprobs is not None:
        lp = _LpOut(out.shape, _n_top(logprobs, extra.n_vocab))
        check(lib().b200_generate_speculative_lp(*args, C.byref(lp.c)))
    else:
        check(lib().b200_generate_speculative(*args))
    del keep
    st = {"passes": stats.passes, "drafted": stats.drafted, "accepted": stats.accepted}
    return ((out, lp.lp, lp.top_ids, lp.top_lp) if lp is not None else out), st


def score(slices, extra: Extra, sessions, token_lists) -> list:
    """Scoring on the device (b200_score): session sessions[k] is fed token_lists[k][:-1] from its current position, and
    its entry of the result holds -log p(token_lists[k][j + 1] | everything before) for every j, in float64.  `slices`
    are in layer order, all on the extra layers' GPU.  -> one array of len(token_lists[k]) - 1 values per session."""
    ids = np.ascontiguousarray(sessions, dtype=np.int32)
    if len(token_lists) != len(ids):
        raise ValueError("need one token list per listed session")
    counts = np.array([len(t) for t in token_lists], np.int32)
    toks = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int64) for t in token_lists]) if len(token_lists) else [],
                                dtype=np.int32)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    fed = np.maximum(counts.astype(np.int64) - 1, 0)
    out = np.zeros(max(int(fed.sum()), 1), np.float64)
    check(lib().b200_score(handles, len(slices), extra.handle, _ptr(ids), _ptr(counts), len(ids), _ptr(toks), _ptr(out)))
    return np.split(out[:int(fed.sum())], np.cumsum(fed)[:-1])


def ppl_window_rows(n_tokens: int, n_ctx: int, n_batch: int = 512):
    """perplexity.cpp's window rules (:37, :48, :103, :130) -> (n_chunk, n_batch, first, n_scored): n_chunk windows of
    n_ctx ids (a trailing partial window dropped), segments of n_batch = min(n_batch, n_ctx) rows, rows j in
    [first, n_ctx - 1) scored, first = min(512, n_ctx / 2)."""
    n_ctx = _int("n_ctx", n_ctx, 2, 2 ** 31 - 1)
    n_batch = min(_int("n_batch", n_batch, 1, 2 ** 31 - 1), n_ctx)
    first = min(512, n_ctx // 2)
    return n_tokens // n_ctx, n_batch, first, n_ctx - 1 - first


def perplexity_windows(slices, extra: Extra, sessions, tokens, n_ctx: int, n_batch: int = 512,
                       fast: bool = False) -> np.ndarray:
    """llama.cpp's windowed perplexity on the device (b200_perplexity_windows): tokens (the text tokenized with BOS) cut
    into windows of n_ctx ids, each evaluated from n_past 0 with its id 0 replaced by BOS, in segments of n_batch rows,
    len(sessions) windows per wave at most.  -> float32 [n_chunk][n_scored]: row i holds window i's terms -logf(prob)
    for rows first .. n_ctx - 2 (ppl_window_rows).  The sessions are left at n_past 0.  fast: the tensor-core prefill
    on Q4_0 / Q8_0 slices (other formats ignore it)."""
    n_chunk, _, _, n_scored = ppl_window_rows(len(tokens), n_ctx, n_batch)
    ids = np.ascontiguousarray(sessions, dtype=np.int32).reshape(-1)
    if len(ids) < 1:
        raise ValueError("perplexity_windows needs at least one session")
    if len(set(ids.tolist())) != len(ids):
        raise ValueError("session listed twice: %s" % ids.tolist())
    toks = np.ascontiguousarray(np.asarray(tokens, np.int64).reshape(-1), dtype=np.int32)
    if len(toks) and (toks.min() < 0 or toks.max() >= extra.n_vocab):
        raise ValueError("token ids must lie in [0, %d)" % extra.n_vocab)
    handles = (C.c_void_p * max(len(slices), 1))(*[s.handle for s in slices])
    out = np.zeros(max(n_chunk * n_scored, 1), np.float32)
    keep = toks if len(toks) else np.zeros(1, np.int32)
    check(lib().b200_perplexity_windows(handles, len(slices), extra.handle, _ptr(ids), len(ids), _ptr(keep), len(toks),
                                        n_ctx, n_batch, int(bool(fast)), _ptr(out)))
    return out[:n_chunk * n_scored].reshape(n_chunk, n_scored)


def _int(name: str, v, lo: int, hi: int) -> int:
    """v as a Python int in [lo, hi], or ValueError / TypeError naming the argument."""
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise TypeError("%s must be an integer, got %r" % (name, v))
    v = int(v)
    if not lo <= v <= hi:
        raise ValueError("%s must be in [%d, %d], got %d" % (name, lo, hi, v))
    return v


def _ids(name: str, seq, n_vocab: int, min_len: int) -> np.ndarray:
    """A list of token ids as int32, each in [0, n_vocab)."""
    if isinstance(seq, (str, bytes)) or not hasattr(seq, "__len__"):
        raise TypeError("%s must be a sequence of token ids" % name)
    out = np.array([_int("%s[%d]" % (name, i), t, 0, n_vocab - 1) for i, t in enumerate(seq)] or [0], np.int32)
    if len(seq) < min_len:
        raise ValueError("%s needs at least %d id(s)" % (name, min_len))
    return out


class Stream:
    """A generation stream (b200_stream_*) over slices in layer order on the extra layers' GPU.  add() queues a session
    with its prompt and budget; read() returns (session, id) pairs as the device draws them; a session leaves at its
    budget, at a stop id (delivered), on cancel() or at close().  Each session's ids equal generate_greedy /
    generate_sample for it alone.  While the stream is open its handles belong to it.  A context manager (close on exit)
    and an iterator of (session, id) pairs, read one at a time, that ends when no session is left.  prefill_chunk C > 0
    feeds each prompt in chunks of C ids beside the other sessions' decode rows (b200_stream_open_ex): a session's ids
    then equal session_forward of each non-final chunk, then generate_* with the last chunk as its prompt."""

    def __init__(self, slices, extra: Extra, max_rows: int = 0, lookahead: int = 0, prefill_chunk: int = 0):
        self._h = None
        slices = list(slices)
        if not slices:
            raise ValueError("a stream needs at least one slice")
        max_rows = _int("max_rows", max_rows, -2 ** 31, 2 ** 31 - 1)
        lookahead = _int("lookahead", lookahead, -2 ** 31, 2 ** 31 - 1)
        prefill_chunk = _int("prefill_chunk", prefill_chunk, 0, 2 ** 31 - 1)
        self.n_vocab = extra.n_vocab
        handles = (C.c_void_p * len(slices))(*[s.handle for s in slices])
        h = C.c_void_p()
        if prefill_chunk:
            check(lib().b200_stream_open_ex(handles, len(slices), extra.handle, max_rows, lookahead, prefill_chunk,
                                            C.byref(h)))
        else:
            check(lib().b200_stream_open(handles, len(slices), extra.handle, max_rows, lookahead, C.byref(h)))
        self._h = h

    def _handle(self) -> C.c_void_p:
        if not self._h:
            raise ValueError("the stream is closed")
        return self._h

    def add(self, session: int, prompt, max_tokens: int, temperature: Optional[float] = None, repeat_penalty: float = 1.1,
            seed: int = 0, first_draw: int = 0, history=None, stop_ids=(), top_k: int = 0, top_p: float = 0.0,
            logprobs: Optional[int] = None, guidance=None) -> None:
        """Queue `session` with `prompt` (token ids) for at most max_tokens ids.  temperature None: greedy (the argmax of
        the raw logits); else the client's Sampler with repeat_penalty on numpy.random.Philox(key=seed), starting at draw
        first_draw, with history (ids sampled before) penalised, truncated to top_k / top_p (0: off).  The session ends
        after the first id in stop_ids.  logprobs = n_top (0..20): each id's record (read_logprobs) holds its
        log-probability and n_top alternatives (b200_stream_add_lp).  guidance = (guidance session, negative prompt ids,
        scale, smooth_factor): classifier-free guidance (b200_stream_add_cfg); the pair enters and leaves as one."""
        session = _int("session", session, 0, 2 ** 31 - 1)
        p = _ids("prompt", prompt, self.n_vocab, 1)
        max_tokens = _int("max_tokens", max_tokens, 1, 2 ** 31 - 1)
        stops = _ids("stop_ids", stop_ids, self.n_vocab, 0)
        sp, keep = None, None
        if temperature is not None:
            t, rp = float(temperature), float(repeat_penalty)
            if not (np.isfinite(t) and t >= 0):
                raise ValueError("temperature must be finite and >= 0, got %r" % temperature)
            if not (np.isfinite(rp) and rp > 0):
                raise ValueError("repeat_penalty must be finite and > 0, got %r" % repeat_penalty)
            seed = _int("seed", seed, 0, 2 ** 64 - 1)
            first_draw = _int("first_draw", first_draw, 0, 2 ** 63 - 1)
            if history is not None:
                history = [_ids("history", history, self.n_vocab, 0)[:len(history)].tolist()]
            sp, keep = _sampling(1, t, rp, [seed], first_draw, history, top_k, top_p)
        elif history is not None or first_draw or _truncation(top_k, top_p) != (0, 0.0):
            raise ValueError("history, first_draw, top_k and top_p apply to sampled sessions (give a temperature)")
        if guidance is not None:
            try:
                g_session, g_ids, scale, smooth_factor = guidance
            except (TypeError, ValueError):
                raise TypeError("guidance must be (session, negative prompt ids, scale, smooth_factor)") from None
            g_session = _int("guidance session", g_session, 0, 2 ** 31 - 1)
            neg = _ids("negative prompt", g_ids, self.n_vocab, 1)
            n_top = -1 if logprobs is None else _n_top(logprobs, self.n_vocab)
            check(lib().b200_stream_add_cfg(self._handle(), session, _ptr(p), len(prompt), max_tokens,
                                            None if sp is None else C.byref(sp), _ptr(stops), len(stop_ids), n_top,
                                            g_session, _ptr(neg), len(g_ids), float(scale), float(smooth_factor)))
            return
        if logprobs is not None:
            n_top = _n_top(logprobs, self.n_vocab)
            check(lib().b200_stream_add_lp(self._handle(), session, _ptr(p), len(prompt), max_tokens,
                                           None if sp is None else C.byref(sp), _ptr(stops), len(stop_ids), n_top))
            return
        check(lib().b200_stream_add(self._handle(), session, _ptr(p), len(prompt), max_tokens,
                                    None if sp is None else C.byref(sp), _ptr(stops), len(stop_ids)))

    def read(self, cap: int = 64) -> list:
        """Up to cap (session, id) pairs in the order they were drawn; blocks until there is at least one.  [] only when
        no session is active or queued.  An id of -1 ends its session: its logits had no distribution."""
        cap = _int("cap", cap, 1, 2 ** 20)
        h = self._handle()
        sess, ids, n = np.zeros(cap, np.int32), np.zeros(cap, np.int32), C.c_int()
        check(lib().b200_stream_read(h, _ptr(sess), _ptr(ids), cap, C.byref(n)))
        return list(zip(sess[:n.value].tolist(), ids[:n.value].tolist()))

    def read_logprobs(self, cap: int = 64) -> list:
        """read() with each id's record (b200_stream_read_lp): up to cap (session, id, lp, [(id, lp), ...]) tuples, the
        list holding the session's n_top alternatives.  A session added without logprobs gives lp NaN and no
        alternatives."""
        cap = _int("cap", cap, 1, 2 ** 20)
        h = self._handle()
        sess, ids, n = np.zeros(cap, np.int32), np.zeros(cap, np.int32), C.c_int()
        lp = np.zeros(cap, np.float64)
        top_ids, top_lp = np.zeros((cap, MAX_TOP), np.int32), np.zeros((cap, MAX_TOP), np.float64)
        check(lib().b200_stream_read_lp(h, _ptr(sess), _ptr(ids), _ptr(lp), _ptr(top_ids), _ptr(top_lp), cap, C.byref(n)))
        return unpack_records(sess[:n.value], ids[:n.value], lp[:n.value], top_ids[:n.value], top_lp[:n.value])

    def cancel(self, session: int) -> None:
        """End a queued or active session now: its positions reflect the ids read so far."""
        session = _int("session", session, 0, 2 ** 31 - 1)
        check(lib().b200_stream_cancel(self._handle(), session))

    def fork(self, src: int, dst: int, n_keep: int) -> None:
        """Copy rows [0, n_keep) of session src to session dst on every slice, in order behind the steps in flight
        (b200_stream_fork); neither may be queued or active.  A following add(dst, ...) continues from n_keep."""
        src = _int("src", src, 0, 2 ** 31 - 1)
        dst = _int("dst", dst, 0, 2 ** 31 - 1)
        n_keep = _int("n_keep", n_keep, 0, 2 ** 31 - 1)
        check(lib().b200_stream_fork(self._handle(), src, dst, n_keep))

    def stats(self) -> dict:
        """The load so far (b200_stream_stats): steps enqueued, the token rows they carried, and the rows of the largest
        step."""
        steps, rows, most = C.c_int64(), C.c_int64(), C.c_int()
        check(lib().b200_stream_stats(self._handle(), C.byref(steps), C.byref(rows), C.byref(most)))
        return {"steps": steps.value, "rows": rows.value, "most_rows": most.value}

    def close(self) -> None:
        if self._h:
            h, self._h = self._h, None
            check(lib().b200_stream_close(h))

    def __enter__(self) -> "Stream":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __iter__(self):
        while True:
            pairs = self.read(1)
            if not pairs:
                return
            yield pairs[0]

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def unpack_records(sessions, ids, lp, top_ids, top_lp) -> list:
    """b200_stream_read_lp's rows (top_* of stride 20, unused entries -1) -> (session, id, lp, [(id, lp), ...])."""
    out = []
    for k in range(len(ids)):
        alts = [(int(t), float(v)) for t, v in zip(top_ids[k], top_lp[k]) if t >= 0]
        out.append((int(sessions[k]), int(ids[k]), float(lp[k]), alts))
    return out
