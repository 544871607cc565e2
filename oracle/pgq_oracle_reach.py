"""ctypes front-end of oracle/pgq_oracle_reach.c: reachability, restated loop for loop (both traversals).

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_reach.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_reach.so")

LANE_LIMIT = 512


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_reach.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_reachability.argtypes = [C.c_int64, p64, p64, C.c_int64, C.c_int64, p64, p64, pu8, pu8, C.c_int,
                                         C.c_int, pu8, pu8, p64, p64, p64, p64]
        lib.orc_reachability.restype = C.c_int
        _lib = lib
    return _lib


class ReferenceHang(RuntimeError):
    """The reference's batch loop would never end on this NULL layout (reachability.cpp:194,251)."""


@dataclass
class ReachStats:
    batches: int
    levels: int
    edges_traversed: int
    stale_starts: int  # batches whose first level ran over a visit_list left by an earlier batch (is_variant)


def reachability(n: int, v, e, src, dst, src_valid=None, dst_valid=None, input_size=None, is_variant=False,
                 restart=False):
    """(reachable uint8, written uint8, ReachStats) of ReachabilityFunction over the CSR (v, e) with the search over
    `input_size` vertices (default n).  restart=True is the reference's batch start (NULL sources re-run rows, a
    layout that would hang raises ReferenceHang, NULL destinations are read as given); restart=False is the defined
    one of pgq_reachability's reference batching (NULL destination -> not written).  Ids read outside
    [0, input_size) raise ValueError."""
    lib = _load()
    v = np.ascontiguousarray(v, dtype=np.int64)
    e = np.ascontiguousarray(e, dtype=np.int64)
    src = np.ascontiguousarray(src, dtype=np.int64)
    dst = np.ascontiguousarray(dst, dtype=np.int64)
    p = len(src)
    sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
    dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
    out = np.zeros(max(p, 1), dtype=np.uint8)
    written = np.zeros(max(p, 1), dtype=np.uint8)
    b, lv, w, ss = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
    p64 = C.POINTER(C.c_int64)
    pu8 = C.POINTER(C.c_uint8)
    rc = lib.orc_reachability(
        n, v.ctypes.data_as(p64), e.ctypes.data_as(p64), n if input_size is None else int(input_size), p,
        src.ctypes.data_as(p64), dst.ctypes.data_as(p64), None if sv is None else sv.ctypes.data_as(pu8),
        None if dv is None else dv.ctypes.data_as(pu8), 1 if is_variant else 0, 1 if restart else 0,
        out.ctypes.data_as(pu8), written.ctypes.data_as(pu8), C.byref(b), C.byref(lv), C.byref(w), C.byref(ss))
    if rc == -2:
        raise ValueError("source or destination outside [0, input_size)")
    if rc == -3:
        raise ReferenceHang("the reference's batch loop would not end on this NULL layout")
    if rc != 0:
        raise MemoryError("orc_reachability: allocation failed")
    return out[:p], written[:p], ReachStats(b.value, lv.value, w.value, ss.value)


def reference_batch_starts(src, src_valid=None):
    """The rows at which the reference starts its batches (reachability.cpp:22,194,251): a batch takes rows from its
    start until the row that opens lane 512 (or the end), and the next one starts curr_batch_size rows -- the rows with
    a valid source -- later.  Raises ReferenceHang where a batch would find no valid source."""
    src = np.asarray(src)
    p = len(src)
    ok = np.ones(p, dtype=bool) if src_valid is None else np.asarray(src_valid).astype(bool)
    starts, start = [], 0
    while start < p:
        starts.append(start)
        lanes, cbs, i = set(), 0, start
        while i < p and len(lanes) < LANE_LIMIT:
            if ok[i]:
                lanes.add(int(src[i]))
                cbs += 1
            i += 1
        if cbs == 0:
            raise ReferenceHang(f"a batch starting at row {start} finds no valid source")
        start += cbs
    return starts
