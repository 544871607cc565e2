"""ctypes front-end of oracle/pgq_oracle_allcheapest.c: cheapest_path_count and all_cheapest_paths, an extension
(SQL/PGQ's ALL CHEAPEST; the reference has no such functions).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from .pgq_oracle import OracleError, _i64, _p64, _pu8

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_allcheapest.c")
_DEPS = [_SRC, os.path.join(_HERE, "pgq_oracle_cheapest.c")]
_LIB = os.path.join(_HERE, "libpgq_oracle_allcheapest.so")

ERR_ALLOC = 1
ERR_ARG = 2          # lanes <= 0, max_paths < 0, or an id outside [0, n) in a row whose id is valid
ERR_UNSUPPORTED = 4  # a row still counting after 65533 edges, or max_paths = 0 with a count of INT64_MAX
WALK_MAX = 65533
INT64_MAX = (1 << 63) - 1
STATS = ("batches", "push_levels", "pull_levels", "walks")


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_allcheapest.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(_LIB) < os.path.getmtime(d) for d in _DEPS):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC, "-lm"])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        for name, wp in (("orc_all_cheapest_paths_i64", p64), ("orc_all_cheapest_paths_f64", C.POINTER(C.c_double))):
            fn = getattr(lib, name)
            fn.argtypes = [C.c_int64, p64, p64, p64, wp, C.c_int64, p64, p64, pu8, pu8, C.c_int, C.c_int, C.c_int64,
                           p64, p64, p64, pu8, C.POINTER(p64), C.POINTER(p64), p64]
            fn.restype = C.c_int
        lib.orc_cheapest_free.argtypes = [C.c_void_p]
        _lib = lib
    return _lib


def _run(n, v, e, edge_ids, w, src, dst, src_valid, dst_valid, lanes, lists, max_paths):
    lib = _load()
    v, e, edge_ids, src, dst = _i64(v), _i64(e), _i64(edge_ids), _i64(src), _i64(dst)
    is_f = np.asarray(w).dtype.kind == "f"
    w = np.ascontiguousarray(w, dtype=np.float64 if is_f else np.int64)
    if e.shape[0] == 0:
        e, edge_ids = np.zeros(1, dtype=np.int64), np.zeros(1, dtype=np.int64)
        w = np.zeros(1, dtype=w.dtype)
    p = src.shape[0]
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    cnt, npaths, first = (np.zeros(max(p, 1), dtype=np.int64) for _ in range(3))
    ov = np.zeros(max(p, 1), dtype=np.uint8)
    offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
    st = np.zeros(len(STATS), dtype=np.int64)
    fn = lib.orc_all_cheapest_paths_f64 if is_f else lib.orc_all_cheapest_paths_i64
    wp = w.ctypes.data_as(C.POINTER(C.c_double)) if is_f else _p64(w)
    rc = fn(n, _p64(v), _p64(e), _p64(edge_ids), wp, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), int(lanes),
            int(lists), int(max_paths), _p64(cnt), _p64(npaths), _p64(first), _pu8(ov), C.byref(offs), C.byref(elems),
            _p64(st))
    if rc:
        raise OracleError(rc, "orc_all_cheapest_paths")
    stats = dict(zip(STATS, st.tolist()))
    try:
        woff = np.ctypeslib.as_array(offs, shape=(stats["walks"] + 1,)).copy()
        flat = np.ctypeslib.as_array(elems, shape=(max(int(woff[-1]), 1),)).copy() if woff[-1] else np.zeros(0, np.int64)
    finally:
        lib.orc_cheapest_free(offs)
        lib.orc_cheapest_free(elems)
    walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(stats["walks"])]
    paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
    return paths, cnt[:p], ov[:p], stats


def cheapest_path_count(n: int, v, e, edge_ids, w, src, dst, src_valid=None, dst_valid=None, lanes: int = 256):
    """-> (counts int64, valid uint8, stats dict) at `lanes` rows per batch over the reference CSR layout (v, e,
    edge_ids) with weights w in CSR order (int64 or float64).  Raises OracleError (ERR_ARG, ERR_UNSUPPORTED)."""
    _, cnt, ov, stats = _run(n, v, e, edge_ids, w, src, dst, src_valid, dst_valid, lanes, False, 0)
    return cnt, ov, stats


def all_cheapest_paths(n: int, v, e, edge_ids, w, src, dst, max_paths: int = 0, src_valid=None, dst_valid=None,
                       lanes: int = 256):
    """-> (per row: list of [src, e1, v1, ..., dst] paths or None, counts int64, stats dict): the first
    min(count, max_paths) cheapest paths of each row (all for max_paths = 0), in the header's order."""
    paths, cnt, _, stats = _run(n, v, e, edge_ids, w, src, dst, src_valid, dst_valid, lanes, True, max_paths)
    return paths, cnt, stats
