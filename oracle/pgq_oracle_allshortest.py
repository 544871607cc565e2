"""ctypes front-end of oracle/pgq_oracle_allshortest.c: shortest_path_count and all_shortest_paths, an extension (the
reference has no such functions: it rejects ALL SHORTEST).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_allshortest.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_allshortest.so")

ERR_RANGE = 3        # an id outside [0, n) in a row whose ids are both valid
ERR_UNSUPPORTED = 4  # a depth beyond 65533, or max_paths = 0 on a saturated count
INT64_MAX = (1 << 63) - 1


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_allshortest.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_all_shortest_paths.argtypes = [C.c_int64, p64, p64, p64, C.c_int64, p64, p64, pu8, pu8, C.c_int64,
                                               C.c_int, p64, p64, p64, p64, pu8, C.POINTER(p64), p64]
        lib.orc_all_shortest_paths.restype = C.c_int
        lib.orc_allshortest_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def _call(n, v, e, edge_ids, src, dst, src_valid, dst_valid, max_paths, lists):
    lib = _load()
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    if e.shape[0] == 0:
        e = np.zeros(1, dtype=np.int64)
        edge_ids = np.zeros(1, dtype=np.int64)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    cnt, npaths, plen, offs = (np.zeros(max(p, 1), dtype=np.int64) for _ in range(4))
    ov = np.zeros(max(p, 1), dtype=np.uint8)
    elems = C.POINTER(C.c_int64)()
    total = C.c_int64(0)
    rc = lib.orc_all_shortest_paths(n, _p64(v), _p64(e), _p64(edge_ids), p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv),
                                    int(max_paths), 1 if lists else 0, _p64(cnt), _p64(npaths), _p64(plen), _p64(offs),
                                    _pu8(ov), C.byref(elems), C.byref(total))
    if rc:
        raise OracleError(rc, "orc_all_shortest_paths")
    if not lists:
        return cnt[:p], ov[:p]
    try:
        flat = np.ctypeslib.as_array(elems, shape=(total.value,)).copy() if elems else np.zeros(0, np.int64)
    finally:
        lib.orc_allshortest_free(elems)
    paths = [flat[offs[i]: offs[i] + npaths[i] * plen[i]].reshape(npaths[i], plen[i]).tolist() if ov[i] else None
             for i in range(p)]
    return paths, cnt[:p]


def shortest_path_count(n: int, v, e, edge_ids, src, dst, src_valid=None, dst_valid=None):
    """-> (counts int64 saturated at INT64_MAX, valid uint8) over the reference CSR layout (v, e, edge_ids)."""
    return _call(n, v, e, edge_ids, src, dst, src_valid, dst_valid, 0, False)


def all_shortest_paths(n: int, v, e, edge_ids, src, dst, max_paths: int = 0, src_valid=None, dst_valid=None):
    """-> (per row: list of [src, e1, v1, ..., dst] lists in step order or None, counts).  Raises
    OracleError(ERR_UNSUPPORTED) for max_paths = 0 on a saturated count or a depth beyond 65533."""
    return _call(n, v, e, edge_ids, src, dst, src_valid, dst_valid, max_paths, True)
