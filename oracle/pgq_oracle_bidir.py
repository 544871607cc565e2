"""ctypes front-end of oracle/pgq_oracle_bidir.c: iterativelengthbidirectional, restated loop for loop.

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_bidir.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_bidir.so")


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_bidir.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_iterativelengthbidirectional.argtypes = [C.c_int64, p64, p64, C.c_int64, p64, p64, pu8, pu8, C.c_int,
                                                         p64, pu8, p64, p64, p64]
        lib.orc_iterativelengthbidirectional.restype = C.c_int
        _lib = lib
    return _lib


@dataclass
class BidirStats:
    batches: int
    iterations: int
    edges_traversed: int


def iterativelengthbidirectional(n: int, v, e, src, dst, src_valid=None, dst_valid=None, lanes: int = 512):
    """(lengths, valid, BidirStats) of the reference's batches of `lanes` (a multiple of 64) over the CSR (v, e).
    NULL destinations give NULL without a lane; ids outside [0, n) raise ValueError."""
    if lanes <= 0 or lanes % 64:
        raise ValueError("lanes must be a positive multiple of 64")
    lib = _load()
    v = np.ascontiguousarray(v, dtype=np.int64)
    e = np.ascontiguousarray(e, dtype=np.int64)
    src = np.ascontiguousarray(src, dtype=np.int64)
    dst = np.ascontiguousarray(dst, dtype=np.int64)
    p = len(src)
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    out = np.full(p, -1, dtype=np.int64)
    valid = np.zeros(p, dtype=np.uint8)
    b, it, w = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    p64 = C.POINTER(C.c_int64)
    pu8 = C.POINTER(C.c_uint8)
    rc = lib.orc_iterativelengthbidirectional(
        n, v.ctypes.data_as(p64), e.ctypes.data_as(p64), p, src.ctypes.data_as(p64), dst.ctypes.data_as(p64),
        None if sv is None else sv.ctypes.data_as(pu8), None if dv is None else dv.ctypes.data_as(pu8), lanes // 64,
        out.ctypes.data_as(p64), valid.ctypes.data_as(pu8), C.byref(b), C.byref(it), C.byref(w))
    if rc == -2:
        raise ValueError("source or destination outside [0, n)")
    if rc != 0:
        raise MemoryError("orc_iterativelengthbidirectional: allocation failed")
    return out, valid, BidirStats(b.value, it.value, w.value)
