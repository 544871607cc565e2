"""ctypes front-end of oracle/pgq_oracle_kgroups.c: shortest_k_groups, an extension (the reference carries SQL/PGQ's
SHORTEST k GROUP in its AST and rejects it).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_kgroups.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_kgroups.so")

ERR_ARG = 2          # k < 1, max_paths < 0, a bad lane width or mode
ERR_RANGE = 3        # an id outside [0, n) in a row whose ids are both valid
ERR_UNSUPPORTED = 4  # a group past 65533 edges, or WALK with max_paths = 0 and a saturated count
PATH_MAX = 65533
MODES = {"WALK": 0, "TRAIL": 1, "ACYCLIC": 2, "SIMPLE": 3}
STATS = ("batches", "lanes", "searches", "levels", "push_levels", "paths")


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_kgroups.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_shortest_k_groups.argtypes = [C.c_int64, p64, p64, p64, C.c_int64, p64, p64, pu8, pu8, C.c_int64,
                                              C.c_int32, C.c_int64, C.c_int32, C.c_int64, p64, p64, p64, pu8, p64, p64,
                                              pu8, C.POINTER(p64), C.POINTER(p64), p64]
        lib.orc_shortest_k_groups.restype = C.c_int
        lib.orc_kgroups_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def shortest_k_groups(n: int, v, e, edge_ids, src, dst, k: int, max_paths: int = 0, mode: str = "WALK",
                      src_valid=None, dst_valid=None, lanes: int = 0, count_only: bool = False):
    """-> (per row: list of [src, e1, v1, ..., dst] paths in order or None, a dict of per-row int64 arrays "count",
    "ngroups", "last_len", "complete", "npaths", "valid", and a stats dict at opts->lanes = `lanes`, 0 for the header's
    rule) over the reference CSR layout (v, e, edge_ids).  count_only (WALK): no lists, valid = the row has a walk.
    Raises OracleError on bad arguments (ERR_ARG), an id out of range (ERR_RANGE) or ERR_UNSUPPORTED."""
    lib = _load()
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    if e.shape[0] == 0:
        e = np.zeros(1, dtype=np.int64)
        edge_ids = np.zeros(1, dtype=np.int64)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    q = max(p, 1)
    cnt, ng, last, npaths, first = (np.zeros(q, dtype=np.int64) for _ in range(5))
    comp, ov = np.zeros(q, dtype=np.uint8), np.zeros(q, dtype=np.uint8)
    offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
    st = np.zeros(len(STATS), dtype=np.int64)
    rc = lib.orc_shortest_k_groups(n, _p64(v), _p64(e), _p64(edge_ids), p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv),
                                   int(k), MODES.get(str(mode).upper(), -1), int(max_paths), int(bool(count_only)),
                                   int(lanes), _p64(cnt), _p64(ng), _p64(last), _pu8(comp), _p64(npaths), _p64(first),
                                   _pu8(ov), C.byref(offs), C.byref(elems), _p64(st))
    if rc:
        raise OracleError(rc, "orc_shortest_k_groups")
    stats = dict(zip(STATS, st.tolist()))
    try:
        woff = np.ctypeslib.as_array(offs, shape=(stats["paths"] + 1,)).copy()
        flat = np.ctypeslib.as_array(elems, shape=(max(int(woff[-1]), 1),)).copy() if woff[-1] else np.zeros(0, np.int64)
    finally:
        lib.orc_kgroups_free(offs)
        lib.orc_kgroups_free(elems)
    walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(stats["paths"])]
    paths = None if count_only else [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
    rows = {"count": cnt[:p], "ngroups": ng[:p], "last_len": last[:p], "complete": comp[:p], "npaths": npaths[:p],
            "valid": ov[:p]}
    return paths, rows, stats
