"""ctypes front-end of oracle/pgq_oracle_kpaths_modes.c: shortest_k_paths in the TRAIL, ACYCLIC and SIMPLE path modes,
an extension (the reference parses the modes and rejects all but WALK).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_kpaths_modes.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_kpaths_modes.so")

ERR_ARG = 2          # k < 1, a bad lane width or mode
ERR_RANGE = 3        # an id outside [0, n) in a row whose ids are both valid
ERR_UNSUPPORTED = 4  # a spur search beyond 65533 levels, or an accepted path longer than 65533 edges
PATH_MAX = 65533
MODES = {"TRAIL": 1, "ACYCLIC": 2, "SIMPLE": 3}
STATS = ("batches", "lanes", "searches", "levels", "paths")


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_kpaths_modes.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_shortest_k_paths_mode.argtypes = [C.c_int64, p64, p64, p64, C.c_int64, p64, p64, pu8, pu8, C.c_int64,
                                                  C.c_int32, C.c_int64, p64, p64, pu8, C.POINTER(p64), C.POINTER(p64), p64]
        lib.orc_shortest_k_paths_mode.restype = C.c_int
        lib.orc_kpaths_modes_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def shortest_k_paths_mode(n: int, v, e, edge_ids, src, dst, k: int, mode: str, src_valid=None, dst_valid=None,
                          lanes: int = 0):
    """-> (per row: list of [src, e1, v1, ..., dst] paths in order or None, npaths int64, stats dict) for mode "TRAIL",
    "ACYCLIC" or "SIMPLE" over the reference CSR layout (v, e, edge_ids); the stats at opts->lanes = `lanes` (0: the
    header's rule).  Raises OracleError on k < 1 or a bad mode / lane width (ERR_ARG), an id out of range (ERR_RANGE)
    or a path beyond 65533 edges (ERR_UNSUPPORTED)."""
    lib = _load()
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    if e.shape[0] == 0:
        e = np.zeros(1, dtype=np.int64)
        edge_ids = np.zeros(1, dtype=np.int64)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    npaths, first = np.zeros(max(p, 1), dtype=np.int64), np.zeros(max(p, 1), dtype=np.int64)
    ov = np.zeros(max(p, 1), dtype=np.uint8)
    offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
    st = np.zeros(len(STATS), dtype=np.int64)
    rc = lib.orc_shortest_k_paths_mode(n, _p64(v), _p64(e), _p64(edge_ids), p, _p64(src), _p64(dst), _pu8(sv),
                                       _pu8(dv), int(k), MODES.get(str(mode).upper(), 0), int(lanes), _p64(npaths),
                                       _p64(first), _pu8(ov), C.byref(offs), C.byref(elems), _p64(st))
    if rc:
        raise OracleError(rc, "orc_shortest_k_paths_mode")
    stats = dict(zip(STATS, st.tolist()))
    try:
        woff = np.ctypeslib.as_array(offs, shape=(stats["paths"] + 1,)).copy()
        flat = np.ctypeslib.as_array(elems, shape=(max(int(woff[-1]), 1),)).copy() if woff[-1] else np.zeros(0, np.int64)
    finally:
        lib.orc_kpaths_modes_free(offs)
        lib.orc_kpaths_modes_free(elems)
    walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(stats["paths"])]
    paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
    return paths, npaths[:p], stats
