"""The Q4_K / Q6_K C restatement (tests/kq_port.c on top of oracle/slice_oracle.c), TEST INFRASTRUCTURE.

`KQPortSlice` mirrors oracle.oracle.PortSlice on a k-quant slice file (every matrix Q4_K or Q6_K, in any mix);
`KQPortExtra` restates the extra layers of a k-quant model (Q4_K tok_embeddings, Q6_K output.weight).  The library is
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
SOURCES = [os.path.join(HERE, "kq_port.c"), os.path.join(ROOT, "oracle", "slice_oracle.c")]

_lib = None


def lib_path() -> str:
    h = hashlib.sha256()
    for p in SOURCES:
        h.update(open(p, "rb").read())
    d = os.path.join(tempfile.gettempdir(), "b200_kq_port_" + h.hexdigest()[:16])
    return os.path.join(d, "libkqport.so")


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
        L.kq_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.kq_forward.restype = C.c_int
        for fn in ("orc_clear", "orc_free"):
            getattr(L, fn).argtypes = [C.c_void_p]
        L.orc_quantize_q8_K.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_dot_q4_K_q8_K.restype = C.c_float
        L.orc_dot_q4_K_q8_K.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_dot_q6_K_q8_K.restype = C.c_float
        L.orc_dot_q6_K_q8_K.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_dequant_q4_K.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.kq_logits.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _lib = L
    return _lib


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


class KQPortSlice:
    """The C restatement on one k-quant slice file."""

    def __init__(self, path: str, n_ctx: int = 512):
        self.lib = lib()
        self.file = ggjt.read_file(path, sliced=True)
        hp = self.file.hparams
        self.n_embd, self.n_layer, self.first_layer = hp.n_embd, hp.n_layer, hp.first_layer
        mm = np.memmap(path, dtype=np.uint8, mode="r")
        self.h = self.lib.orc_create(hp.n_embd, hp.n_head, hp.n_ff, hp.n_layer, n_ctx, ggjt.T_Q4_K)
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
        types = ggjt.check_slice_types(self.file)
        if types[0] not in (ggjt.T_Q4_K, ggjt.T_Q6_K):
            raise ValueError("not a k-quant slice (first matrix %s)" % ggjt.TYPE_NAME.get(types[0], str(types[0])))
        self.types = np.array(types, dtype=np.int32)

    def forward(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        out = np.empty_like(x)
        rc = self.lib.kq_forward(self.h, _ptr(self.types), _ptr(x), x.shape[0], _ptr(out))
        if rc != 0:
            raise RuntimeError("oracle forward failed: %d" % rc)
        return out

    def clear_context(self) -> None:
        self.lib.orc_clear(self.h)

    def close(self) -> None:
        if self.h:
            self.lib.orc_free(self.h)
            self.h = None


class KQPortExtra:
    """Embeddings (Q4_K rows, dequantize_row_q4_K) and logits (RMSNorm + Q6_K lm_head) of a k-quant extra-layers file."""

    def __init__(self, path: str):
        self.lib = lib()
        f = ggjt.read_file(path, sliced=True)
        self.n_vocab, self.n_embd = f.hparams.n_vocab, f.hparams.n_embd
        assert f.tensors["tok_embeddings.weight"].ttype == ggjt.T_Q4_K and f.tensors["output.weight"].ttype == ggjt.T_Q6_K
        self.emb = np.frombuffer(f.read_raw("tok_embeddings.weight"), np.uint8).copy()
        self.norm = np.frombuffer(f.read_raw("norm.weight"), np.float32).copy()
        self.out = np.frombuffer(f.read_raw("output.weight"), np.uint8).copy()

    def embed(self, tokens) -> np.ndarray:
        e = self.n_embd
        row = e // ggjt.QK_K * 144
        out = np.zeros((len(tokens), e), np.float32)
        for i, t in enumerate(tokens):
            if 0 <= t < self.n_vocab:
                self.lib.orc_dequant_q4_K(_ptr(self.emb[t * row:(t + 1) * row]), e, _ptr(out[i]))
        return out

    def logits(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, self.n_embd)
        y = np.empty((x.shape[0], self.n_vocab), np.float32)
        self.lib.kq_logits(_ptr(self.out), self.n_vocab, self.n_embd, _ptr(self.norm), _ptr(x), x.shape[0], _ptr(y))
        return y
