"""ctypes front-end of oracle/pgq_oracle_cheapest.c: cheapest_path, an extension (the reference has no such function).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, Stats, _Stats, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_cheapest.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_cheapest.so")

ERR_UNSUPPORTED = 4  # a level beyond 65534 (the device's levels are uint16)


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_cheapest.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC, "-lm"])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8, pf64 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.POINTER(C.c_double)
        for name, pw in (("orc_cheapest_path_i64", p64), ("orc_cheapest_path_f64", pf64)):
            fn = getattr(lib, name)
            fn.argtypes = [C.c_int64, p64, p64, p64, pw, C.c_int64, p64, p64, pu8, pu8, C.c_int, p64, p64, pu8,
                           C.POINTER(p64), p64, C.POINTER(_Stats)]
            fn.restype = C.c_int
        lib.orc_cheapest_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def cheapest_path(n: int, v, e, edge_ids, w, src, dst, src_valid=None, dst_valid=None, lanes: int = 256):
    """The cheapest path as shortestpath's list, `lanes` rows per batch (see orc_cheapest_path_i64).  -> (list of
    python lists or None per row, Stats with levels = tight levels expanded).  A path deeper than 65534 edges raises
    OracleError(ERR_UNSUPPORTED)."""
    lib = _load()
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    w = np.ascontiguousarray(w)
    is_f = w.dtype.kind == "f"
    w = w.astype(np.float64 if is_f else np.int64)
    if e.shape[0] == 0:
        e = np.zeros(1, dtype=np.int64)
        edge_ids = np.zeros(1, dtype=np.int64)
        w = np.zeros(1, dtype=w.dtype)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    offs = np.zeros(max(p, 1), dtype=np.int64)
    lens = np.zeros(max(p, 1), dtype=np.int64)
    ov = np.zeros(max(p, 1), dtype=np.uint8)
    elems = C.POINTER(C.c_int64)()
    total = C.c_int64(0)
    st = _Stats()
    fn = lib.orc_cheapest_path_f64 if is_f else lib.orc_cheapest_path_i64
    wp = w.ctypes.data_as(C.POINTER(C.c_double)) if is_f else _p64(w)
    rc = fn(n, _p64(v), _p64(e), _p64(edge_ids), wp, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), lanes, _p64(offs),
            _p64(lens), _pu8(ov), C.byref(elems), C.byref(total), C.byref(st))
    if rc:
        raise OracleError(rc, "orc_cheapest_path")
    flat = np.ctypeslib.as_array(elems, shape=(max(total.value, 1),)).copy()[: total.value]
    lib.orc_cheapest_free(elems)
    paths = [flat[offs[i]: offs[i] + lens[i]].tolist() if ov[i] else None for i in range(p)]
    return paths, Stats(st.batches, st.levels, st.edges_traversed, st.frontier_vertices)
