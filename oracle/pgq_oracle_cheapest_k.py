"""ctypes front-end of oracle/pgq_oracle_cheapest_k.c: cheapest_k_paths, the k cheapest paths of a row in the WALK,
TRAIL, ACYCLIC and SIMPLE path modes over a weighted CSR (no reference function).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_cheapest_k.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_cheapest_k.so")

ERR_ARG = 2          # k < 1, a bad lane width or mode
ERR_RANGE = 3        # an id outside [0, n) in a row whose ids are both valid
ERR_UNSUPPORTED = 4  # a weight below zero, a spur search beyond 65534 tight levels, a path longer than 65533 edges
MODES = {"WALK": 0, "TRAIL": 1, "ACYCLIC": 2, "SIMPLE": 3}
STATS = ("batches", "lanes", "searches", "push_levels", "paths")


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_cheapest_k.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_cheapest_k_paths.argtypes = [C.c_int64, p64, p64, p64, p64, C.c_int, C.c_int64, p64, p64, pu8, pu8,
                                             C.c_int64, C.c_int32, C.c_int64, p64, p64, pu8, C.POINTER(p64),
                                             C.POINTER(p64), C.POINTER(p64), p64]
        lib.orc_cheapest_k_paths.restype = C.c_int
        lib.orc_cheapest_k_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def cheapest_k_paths(n: int, v, e, edge_ids, w, src, dst, k: int, mode: str = "WALK", src_valid=None, dst_valid=None,
                     lanes: int = 0):
    """-> (per row: list of [src, e1, v1, ..., dst] paths in order or None, per row: list of costs or None, npaths
    int64, stats dict) over the reference CSR layout (v, e, edge_ids) with weights w in CSR position order (int64 for
    BIGINT, float64 for DOUBLE); costs are ints or floats.  The stats are at opts->lanes = `lanes` (0: the header's
    rule).  Raises OracleError on k < 1 or a bad mode / lane width (ERR_ARG), an id out of range (ERR_RANGE), or a
    weight below zero or a path beyond the limits (ERR_UNSUPPORTED)."""
    lib = _load()
    w = np.asarray(w)
    is_f64 = w.dtype.kind == "f"
    wbits = np.ascontiguousarray(w, dtype=np.float64).view(np.int64) if is_f64 else _i64(w)
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    if e.shape[0] == 0:
        e = np.zeros(1, dtype=np.int64)
        edge_ids = np.zeros(1, dtype=np.int64)
        wbits = np.zeros(1, dtype=np.int64)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    npaths, first = np.zeros(max(p, 1), dtype=np.int64), np.zeros(max(p, 1), dtype=np.int64)
    ov = np.zeros(max(p, 1), dtype=np.uint8)
    offs, elems, costs = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
    st = np.zeros(len(STATS), dtype=np.int64)
    mode_id = MODES.get(str(mode).upper(), -1)
    rc = lib.orc_cheapest_k_paths(n, _p64(v), _p64(e), _p64(edge_ids), _p64(wbits), int(is_f64), p, _p64(src),
                                  _p64(dst), _pu8(sv), _pu8(dv), int(k), mode_id, int(lanes), _p64(npaths), _p64(first),
                                  _pu8(ov), C.byref(offs), C.byref(elems), C.byref(costs), _p64(st))
    if rc:
        raise OracleError(rc, "orc_cheapest_k_paths")
    stats = dict(zip(STATS, st.tolist()))
    try:
        woff = np.ctypeslib.as_array(offs, shape=(stats["paths"] + 1,)).copy()
        flat = np.ctypeslib.as_array(elems, shape=(max(int(woff[-1]), 1),)).copy() if woff[-1] else np.zeros(0, np.int64)
        cbits = np.ctypeslib.as_array(costs, shape=(stats["paths"] + 1,)).copy()[:stats["paths"]]
    finally:
        lib.orc_cheapest_k_free(offs)
        lib.orc_cheapest_k_free(elems)
        lib.orc_cheapest_k_free(costs)
    cvals = (cbits.view(np.float64) if is_f64 else cbits).tolist()
    walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(stats["paths"])]
    paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
    cost_rows = [cvals[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
    return paths, cost_rows, npaths[:p], stats
