"""The Q5_0 / Q5_1 C restatement (tests/q5_port.c on top of oracle/slice_oracle.c), TEST INFRASTRUCTURE.

`Q5PortSlice` mirrors oracle.oracle.PortSlice on a slice file of any type the restatement covers; the library is
compiled on first use into a per-source directory under the system temporary directory (the tree may be read-only).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from distributedllm_b200 import ggjt

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "q5_port.c"), os.path.join(ROOT, "oracle", "slice_oracle.c")]

_lib = None


def lib_path() -> str:
    h = hashlib.sha256()
    for p in SOURCES:
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "b200_q5_port_" + h.hexdigest()[:16])
    return os.path.join(d, "libq5port.so")


def build() -> str:
    """Same flags as oracle/Makefile's liboracle.so."""
    so = lib_path()
    if not os.path.isfile(so):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + ".tmp%d" % os.getpid()
        subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-mfma", "-mavx2", "-ffp-contract=off",
                        "-I" + os.path.join(ROOT, "oracle"), "-o", tmp, SOURCES[0], "-lm"], check=True)
        os.replace(tmp, so)
    return so


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.c_int] * 6
        L.orc_set_layer.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 9
        L.q5_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.q5_forward.restype = C.c_int
        for fn in ("orc_clear", "orc_free"):
            getattr(L, fn).argtypes = [C.c_void_p]
        L.orc_dot_q5_0_q8_0.restype = C.c_float
        L.orc_dot_q5_0_q8_0.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_dot_q5_1_q8_1.restype = C.c_float
        L.orc_dot_q5_1_q8_1.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_quant_q8_0.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.orc_quant_q8_1.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


class Q5PortSlice:
    """The C restatement on one slice file (Q5_0, Q5_1, or any type oracle/slice_oracle.c covers)."""

    def __init__(self, path: str, n_ctx: int = 512):
        self.lib = lib()
        self.file = ggjt.read_file(path, sliced=True)
        hp = self.file.hparams
        self.n_embd, self.n_layer, self.first_layer = hp.n_embd, hp.n_layer, hp.first_layer
        mm = np.memmap(path, dtype=np.uint8, mode="r")
        wt = self.file.tensors["layers.%d.attention.wq.weight" % hp.first_layer].ttype
        self.h = self.lib.orc_create(hp.n_embd, hp.n_head, hp.n_ff, hp.n_layer, n_ctx, wt)
        self._keep = []
        for i in range(hp.n_layer):
            pre = "layers.%d." % (i + hp.first_layer)
            ptrs = []
            for nm in ("attention_norm.weight", "attention.wq.weight", "attention.wk.weight", "attention.wv.weight",
                       "attention.wo.weight", "ffn_norm.weight", "feed_forward.w1.weight", "feed_forward.w2.weight",
                       "feed_forward.w3.weight"):
                t = self.file.tensors[pre + nm]
                a = np.array(mm[t.offset:t.offset + t.nbytes])          # private, aligned copy
                self._keep.append(a)
                ptrs.append(_ptr(a))
            self.lib.orc_set_layer(self.h, i, *ptrs)

    def forward(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        rc = self.lib.q5_forward(self.h, _ptr(x), x.shape[0], _ptr(out))
        if rc != 0:
            raise RuntimeError("oracle forward failed: %d" % rc)
        return out

    def clear_context(self) -> None:
        self.lib.orc_clear(self.h)

    def close(self) -> None:
        if self.h:
            self.lib.orc_free(self.h)
            self.h = None
