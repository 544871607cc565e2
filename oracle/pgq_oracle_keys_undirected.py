"""ctypes front-end of oracle/pgq_oracle_keys_undirected.c: the undirected CSR CTE of the reference from key columns.

TEST INFRASTRUCTURE ONLY, like pgq_oracle.py: imported by tests/ and tools/, never by duckpgq_extension_b200.
The joins, the GROUP BY and the UNION BY NAME of CreateUndirectedCSRCTE (compressed_sparse_row.cpp:125-130,145-172,
192-223) run in pgq_oracle_keys_undirected.c; what they produce goes through pgq_oracle's restatement of
create_csr_vertex -> prefix sum -> create_csr_edge.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import pgq_oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pgq_oracle_keys_undirected.c")
_LIB = os.path.join(_HERE, "libpgq_oracle_keys_undirected.so")

ConstraintError = orc.ConstraintError
CONSTRAINT_TEXT = orc.CONSTRAINT_TEXT


def build(force: bool = False) -> str:
    """gcc -O2 the restatement into oracle/libpgq_oracle_keys_undirected.so (git-ignored)."""
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", _LIB, _SRC])
    return _LIB


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
        lib.orc_key_join_undirected.argtypes = [C.c_int64, p64, pu8, C.c_int64, p64, p64, pu8, pu8, p64, p64, p64,
                                                C.POINTER(C.c_int), p64, p64, p64]
        lib.orc_key_join_undirected.restype = C.c_int
        _lib = lib
    return _lib


def _p64(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_int64))


def _pu8(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))


def key_join_undirected(vertex_keys, edge_src, edge_dst, vertex_valid=None, src_valid=None, dst_valid=None):
    """The CTE's statements without create_csr_edge: (cnt[n] degrees, S, bad, rows) with rows = (src, dst, edge_id)
    int64 sorted by (src, dst), one per distinct pair, edge_id the smallest edge rowid of the pair."""
    lib = _load()
    vk, sk, dk = (np.ascontiguousarray(a, dtype=np.int64) for a in (vertex_keys, edge_src, edge_dst))
    if sk.shape != dk.shape:
        raise ValueError("edge_src and edge_dst differ in length")
    vv, sv, dv = (None if a is None else np.ascontiguousarray(a, dtype=np.uint8)
                  for a in (vertex_valid, src_valid, dst_valid))
    n, m = vk.shape[0], sk.shape[0]
    vk1, sk1, dk1 = (a if a.shape[0] else np.zeros(1, dtype=np.int64) for a in (vk, sk, dk))
    cnt = np.zeros(max(n, 1), dtype=np.int64)
    s, r, bad = C.c_int64(0), C.c_int64(0), C.c_int(0)
    args = (n, _p64(vk1), _pu8(vv), m, _p64(sk1), _p64(dk1), _pu8(sv), _pu8(dv), _p64(cnt), C.byref(s), C.byref(r),
            C.byref(bad))
    if lib.orc_key_join_undirected(*args, None, None, None):
        raise orc.OracleError(orc.ORC_ERR_ALLOC, "orc_key_join_undirected")
    rows = [np.zeros(max(r.value, 1), dtype=np.int64) for _ in range(3)]
    if lib.orc_key_join_undirected(*args, *(_p64(x) for x in rows)):
        raise orc.OracleError(orc.ORC_ERR_ALLOC, "orc_key_join_undirected")
    return cnt[:n], s.value, bool(bad.value), tuple(x[:r.value] for x in rows)


def csr_build_keys_undirected(vertex_keys, edge_src, edge_dst, vertex_valid=None, src_valid=None, dst_valid=None):
    """The undirected CSR CTE from key columns.  Returns (v[n+2], e, edge_ids) int64 in the reference layout, each
    row's neighbours in ascending rowid order.  Raises ConstraintError when the degree sum differs from the number of
    rows (csr_creation.cpp:121-125) and when some row's pair count differs from its degree."""
    cnt, s, bad, (rsrc, rdst, reid) = key_join_undirected(vertex_keys, edge_src, edge_dst, vertex_valid, src_valid,
                                                          dst_valid)
    if bad or s != rsrc.shape[0]:
        raise ConstraintError(orc.ORC_ERR_CONSTRAINT, CONSTRAINT_TEXT)
    n = cnt.shape[0]
    # create_csr_vertex(rowid, cnt) for every vertex row, then create_csr_edge over the rows (Sigma cnt vs count)
    return orc.csr_build_stepwise(n, np.arange(n, dtype=np.int64), cnt, rsrc.shape[0], rsrc, rdst, reid)
