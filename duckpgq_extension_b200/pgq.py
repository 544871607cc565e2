"""Host-side mirror of DuckPGQ's path-finding scalar functions on top of the C ABI.

Same names, argument meaning and error behaviour as the reference UDFs, so the parity tests read
like the reference's own sqllogictests:

    create_csr_vertex(id, v_size, dense_id, cnt)                      csr_creation.cpp:86-110,200-208
    create_csr_edge(id, v_size, sum_cnt, edge_count, src, dst, edge)  csr_creation.cpp:112-198,210-238
    iterativelength(id, v_size, src, dst)                             iterativelength.cpp:34-152
    shortestpath(id, v_size, src, dst)                                shortest_path.cpp:43-217
    cheapest_path(id, v_size, src, dst)                               (no reference function: the cheapest path's list)
    cheapest_path_count(id, v_size, src, dst)                         (no reference function: ALL CHEAPEST's count)
    all_cheapest_paths(id, v_size, src, dst, max_paths)               (no reference function: ALL CHEAPEST's lists)
    shortest_path_count(id, v_size, src, dst)                         (no reference function: ALL SHORTEST's count)
    all_shortest_paths(id, v_size, src, dst, max_paths)               (no reference function: ALL SHORTEST's lists)
    shortest_k_paths(id, v_size, src, dst, k)                         (no reference function: SHORTEST k's walks)
    shortest_k_groups(id, v_size, src, dst, k, max_paths)             (no reference function: SHORTEST k GROUP's paths)
    delete_csr(id)                                                    csr_deletion.cpp:10-29
    DuckPGQState.{csr_list, csr_to_delete, get_csr, query_end}        duckpgq_state.hpp:12-39, duckpgq_state.cpp:162-186

DataChunk columns are numpy int64 arrays (+ an optional validity array for NULLs).  All compute
happens in libduckpgq_b200.so on the GPU; this file only marshals pointers.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _native

PGQ_OK = 0
PGQ_ERR_INVALID_ARG, PGQ_ERR_CUDA, PGQ_ERR_OOM, PGQ_ERR_CONSTRAINT = 1, 2, 3, 4
PGQ_ERR_RANGE, PGQ_ERR_INVALID_ID, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_UNSUPPORTED = 5, 6, 7, 8
PGQ_PATH_WALK, PGQ_PATH_TRAIL, PGQ_PATH_ACYCLIC, PGQ_PATH_SIMPLE = 0, 1, 2, 3  # pgq_path_mode


def path_mode_id(mode: str) -> int:
    """SQL/PGQ's path mode by name, any case -> PGQ_PATH_*; another name raises InvalidInputException."""
    ids = {"WALK": PGQ_PATH_WALK, "TRAIL": PGQ_PATH_TRAIL, "ACYCLIC": PGQ_PATH_ACYCLIC, "SIMPLE": PGQ_PATH_SIMPLE}
    if not isinstance(mode, str) or mode.upper() not in ids:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"path mode must be WALK, TRAIL, ACYCLIC or SIMPLE, not {mode!r}")
    return ids[mode.upper()]


class PgqError(RuntimeError):
    """Base of all errors raised by this package (status = pgq_status of the C ABI)."""

    def __init__(self, status: int, message: str):
        super().__init__(message)
        self.status = status


class ConstraintException(PgqError):
    """duckdb::ConstraintException with the reference's text."""


class InvalidInputException(PgqError):
    """duckdb::InvalidInputException."""


def _raise(status: int):
    lib = _native.load()
    msg = lib.pgq_last_error().decode()
    if status in (PGQ_ERR_CONSTRAINT, PGQ_ERR_INVALID_ID, PGQ_ERR_NOT_INITIALIZED):
        raise ConstraintException(status, lib.pgq_status_text(status).decode())
    if status in (PGQ_ERR_INVALID_ARG, PGQ_ERR_RANGE):
        raise InvalidInputException(status, msg)
    raise PgqError(status, msg)


def _check(status: int):
    if status != PGQ_OK:
        _raise(status)


def _i64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int64)


def _p64(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_int64))


def _pu8(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))


def _weights(weight):
    """A weight column as create_csr_edge's overloads take it: a float array is DOUBLE (csr_creation.cpp:232-235),
    anything else BIGINT (:227-230).  -> (the contiguous array, its int64 pointer or None, its double pointer or None)."""
    weight = np.ascontiguousarray(weight)
    if weight.dtype.kind == "f":
        weight = weight.astype(np.float64)
        return weight, None, weight.ctypes.data_as(C.POINTER(C.c_double))
    weight = weight.astype(np.int64)
    return weight, _p64(weight), None


def _device_weights(d_weight: int, weight_type: int):
    """A device weight column's address as the (BIGINT, DOUBLE) pointer pair of the C ABI: weight_type 1 = BIGINT,
    2 = DOUBLE.  The address must be non-zero even for no edges: the pointer is what names the type."""
    if weight_type not in (1, 2):
        raise ValueError(f"weight_type must be 1 (BIGINT) or 2 (DOUBLE), not {weight_type!r}")
    return (d_weight or None, None) if weight_type == 1 else (None, d_weight or None)


def _same_length(a: np.ndarray, m: int, what: str):
    if a.shape != (m,):
        raise ValueError(f"{what} holds {a.shape[0] if a.ndim == 1 else a.shape} values for {m} edges")


@dataclass
class Options:
    """pgq_options: lanes 0|64|128|256|512, direction 0 auto | 1 push | 2 pull, alpha 0 = default,
    reference_batching: every non-NULL row takes a lane, as in the reference (PGQ_OPT_REFERENCE_BATCHING)."""
    lanes: int = 0
    direction: int = 0
    alpha: int = 0
    reference_batching: bool = False
    shard_index: int = 0  # multi-GPU: run only the searches with ordinal % shard_count == shard_index
    shard_count: int = 0
    no_dedup: bool = False  # PGQ_OPT_NO_DEDUP: one lane per row even when sources repeat
    no_prune: bool = False  # PGQ_OPT_NO_PRUNE: no degree shortcut

    def c(self) -> _native.PgqOptions:
        flags = (1 if self.reference_batching else 0) | (2 if self.no_dedup else 0) | (4 if self.no_prune else 0)
        return _native.PgqOptions(self.lanes, self.direction, self.alpha, flags, self.shard_index, self.shard_count)


class Context:
    """One per (process, GPU): pgq_ctx."""

    def __init__(self, device: int = 0):
        self._lib = _native.load()
        h = C.c_void_p()
        _check(self._lib.pgq_ctx_create(device, C.byref(h)))
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.pgq_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx: dict[int, Context] = {}


def device_count() -> int:
    c = C.c_int(0)
    _check(_native.load().pgq_device_count(C.byref(c)))
    return c.value


def default_context(device: int = 0) -> Context:
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class DeviceCSR:
    """pgq_csr: the device-resident CSR (class CSR, compressed_sparse_row.hpp:25-47)."""

    def __init__(self, ctx: Context, handle: C.c_void_p, n: int):
        self.ctx = ctx
        self._lib = ctx._lib
        self._h = handle
        self.n = n
        self.initialized_v = True
        self.initialized_e = True  # CsrInitializeEdge has run (csr_creation.cpp:43-61): False until create()'s edges come

    # ---- construction ---------------------------------------------------------------------------
    @classmethod
    def create(cls, ctx: Context, n: int) -> "DeviceCSR":
        h = C.c_void_p()
        _check(ctx._lib.pgq_csr_create(ctx._h, n, C.byref(h)))
        csr = cls(ctx, h, n)
        csr.initialized_e = False
        return csr

    @classmethod
    def build(cls, ctx: Context, n: int, src, dst, edge_id=None, weight=None) -> "DeviceCSR":
        """The CSR of the edge rows (src, dst, edge rowid).  weight (optional): one BIGINT (int) or DOUBLE (float)
        weight per row, which lands at the CSR position its row takes (pgq_csr_build_weighted)."""
        src, dst = _i64(src), _i64(dst)
        eid = None if edge_id is None else _i64(edge_id)
        h = C.c_void_p()
        if weight is None:
            _check(ctx._lib.pgq_csr_build(ctx._h, n, src.shape[0], _p64(src), _p64(dst), _p64(eid), C.byref(h)))
        else:
            w, wi, wf = _weights(weight)
            _same_length(w, src.shape[0], "weight")
            _check(ctx._lib.pgq_csr_build_weighted(ctx._h, n, src.shape[0], _p64(src), _p64(dst), _p64(eid), wi, wf,
                                                   C.byref(h)))
        return cls(ctx, h, n)

    @classmethod
    def build_device(cls, ctx: Context, n: int, m: int, d_src: int, d_dst: int, d_edge_id: int = 0,
                     d_weight: int = 0, weight_type: int = 0) -> "DeviceCSR":
        """Edge columns already in HBM: raw device addresses of int32 src / dst (and int64 edge rowids).  With
        weight_type 1 (BIGINT, int64) or 2 (DOUBLE, float64), d_weight is the address of one weight per row
        (pgq_csr_build_device_weighted)."""
        h = C.c_void_p()
        if not weight_type and not d_weight:
            _check(ctx._lib.pgq_csr_build_device(ctx._h, n, m, d_src, d_dst, d_edge_id or None, C.byref(h)))
        else:
            wi, wf = _device_weights(d_weight, weight_type)
            _check(ctx._lib.pgq_csr_build_device_weighted(ctx._h, n, m, d_src, d_dst, d_edge_id or None, wi, wf,
                                                          C.byref(h)))
        return cls(ctx, h, n)

    @classmethod
    def build_from_keys(cls, ctx: Context, vertex_keys, edge_src, edge_dst, vertex_valid=None, src_valid=None,
                        dst_valid=None, undirected: bool = False, weight=None, weight_valid=None) -> "DeviceCSR":
        """The directed CSR CTE (compressed_sparse_row.cpp:132-143,234-251) from key columns: vertex row i has key
        vertex_keys[i], edge k joins src key edge_src[k] to dst key edge_dst[k]; the *_valid arrays (1 = valid,
        0 = NULL) are optional.  Raises ConstraintException (csr_creation.cpp:121-125) when an edge with a
        matching source has no or several matching destination rows.

        undirected=True builds the undirected CSR CTE instead (compressed_sparse_row.cpp:125-130,145-172,192-223):
        one row per distinct pair of the joined edges and their reverses, its edge id the smallest edge rowid of the
        pair, neighbours in ascending rowid order; ConstraintException when a row's pair count differs from its
        number of distinct other-end keys (NULL and unmatched ones included).

        weight (optional, directed only): the edge table's BIGINT (int) or DOUBLE (float) weight column e.w; every row
        edge k becomes carries weight[k] (pgq_csr_build_keys_weighted).  weight_valid (optional, 0 = NULL) may mark
        NULL weights on edges that join nothing; a NULL weight on an edge that joins raises InvalidInputException."""
        if weight is None and weight_valid is not None:
            raise ValueError("weight_valid without a weight column")
        if undirected and weight is not None:
            raise ValueError("the undirected CSR CTE carries no weights")
        vk, sk, dk = _i64(vertex_keys), _i64(edge_src), _i64(edge_dst)
        if sk.shape != dk.shape:
            raise ValueError("edge_src and edge_dst differ in length")
        vv, sv, dv = (None if a is None else np.ascontiguousarray(a, dtype=np.uint8)
                      for a in (vertex_valid, src_valid, dst_valid))
        for a, want in ((vv, vk), (sv, sk), (dv, dk)):
            if a is not None and a.shape != want.shape:
                raise ValueError("a validity array differs in length from its key column")
        n = vk.shape[0]
        h = C.c_void_p()
        if weight is not None:
            w, wi, wf = _weights(weight)
            _same_length(w, sk.shape[0], "weight")
            wv = None if weight_valid is None else np.ascontiguousarray(weight_valid, dtype=np.uint8)
            if wv is not None:
                _same_length(wv, sk.shape[0], "weight_valid")
            _check(ctx._lib.pgq_csr_build_keys_weighted(ctx._h, n, _p64(vk), _pu8(vv), sk.shape[0], _p64(sk), _p64(dk),
                                                        _pu8(sv), _pu8(dv), wi, wf, _pu8(wv), C.byref(h)))
            return cls(ctx, h, n)
        fn = ctx._lib.pgq_csr_build_keys_undirected if undirected else ctx._lib.pgq_csr_build_keys
        _check(fn(ctx._h, n, _p64(vk), _pu8(vv), sk.shape[0], _p64(sk), _p64(dk), _pu8(sv), _pu8(dv), C.byref(h)))
        return cls(ctx, h, n)

    @classmethod
    def build_from_keys_device(cls, ctx: Context, n: int, m: int, d_vertex_keys: int, d_edge_src: int,
                               d_edge_dst: int, d_vertex_valid: int = 0, d_src_valid: int = 0,
                               d_dst_valid: int = 0, undirected: bool = False, d_weight: int = 0,
                               d_weight_valid: int = 0, weight_type: int = 0) -> "DeviceCSR":
        """build_from_keys for columns already in HBM: raw device addresses of the int64 key columns (n vertex
        keys, m edge src / dst keys) and of the optional uint8 validity columns (0 = all valid).  With weight_type
        1 (BIGINT, int64) or 2 (DOUBLE, float64), d_weight is the address of the weight column and d_weight_valid
        that of its optional validity (pgq_csr_build_keys_weighted_device)."""
        h = C.c_void_p()
        if weight_type or d_weight or d_weight_valid:
            if undirected:
                raise ValueError("the undirected CSR CTE carries no weights")
            wi, wf = _device_weights(d_weight, weight_type)
            _check(ctx._lib.pgq_csr_build_keys_weighted_device(
                ctx._h, n, d_vertex_keys or None, d_vertex_valid or None, m, d_edge_src or None, d_edge_dst or None,
                d_src_valid or None, d_dst_valid or None, wi, wf, d_weight_valid or None, C.byref(h)))
            return cls(ctx, h, n)
        fn = ctx._lib.pgq_csr_build_keys_undirected_device if undirected else ctx._lib.pgq_csr_build_keys_device
        _check(fn(ctx._h, n, d_vertex_keys or None, d_vertex_valid or None, m, d_edge_src or None, d_edge_dst or None,
                  d_src_valid or None, d_dst_valid or None, C.byref(h)))
        return cls(ctx, h, n)

    @classmethod
    def upload(cls, ctx: Context, n: int, v, e, edge_ids=None, weight=None) -> "DeviceCSR":
        """A finished CSR in the reference's layout (v: n + 2 offsets, e: m targets).  weight (optional): one BIGINT
        (int) or DOUBLE (float) weight per CSR position, the reference's w / w_double (pgq_csr_upload_weighted)."""
        v, e = _i64(v), _i64(e)
        ids = None if edge_ids is None else _i64(edge_ids)
        h = C.c_void_p()
        if weight is None:
            _check(ctx._lib.pgq_csr_upload(ctx._h, n, e.shape[0], _p64(v), _p64(e), _p64(ids), C.byref(h)))
        else:
            w, wi, wf = _weights(weight)
            _same_length(w, e.shape[0], "weight")
            _check(ctx._lib.pgq_csr_upload_weighted(ctx._h, n, e.shape[0], _p64(v), _p64(e), _p64(ids), wi, wf,
                                                    C.byref(h)))
        return cls(ctx, h, n)

    def clone(self, ctx: Context) -> "DeviceCSR":
        """A replica of this (finished) CSR in another context / on another device (pgq_csr_clone)."""
        h = C.c_void_p()
        _check(self._lib.pgq_csr_clone(self._h, ctx._h, C.byref(h)))
        return DeviceCSR(ctx, h, self.n)

    def add_vertex_counts(self, dense_id, cnt) -> int:
        dense_id, cnt = _i64(dense_id), _i64(cnt)
        s = C.c_int64(0)
        _check(self._lib.pgq_csr_add_vertex_counts(self._h, dense_id.shape[0], _p64(dense_id), _p64(cnt), C.byref(s)))
        return s.value

    def add_edges(self, edge_size: int, edge_size_count: int, src, dst, edge_id, weight=None):
        src, dst, edge_id = _i64(src), _i64(dst), _i64(edge_id)
        self.initialized_e = True
        if weight is None:
            _check(self._lib.pgq_csr_add_edges(self._h, edge_size, edge_size_count, src.shape[0], _p64(src), _p64(dst),
                                               _p64(edge_id)))
            return
        weight, wi, wf = _weights(weight)
        _check(self._lib.pgq_csr_add_edges_weighted(self._h, edge_size, edge_size_count, src.shape[0], _p64(src),
                                                    _p64(dst), _p64(edge_id), wi, wf))

    def weight_type(self) -> int:
        t = C.c_int(0)
        _check(self._lib.pgq_csr_weight_type(self._h, C.byref(t)))
        return t.value

    def download_weights(self):
        """get_csr_w (pgq_scan.cpp:113-141): the weights in the reference's CSR position order."""
        _, m, _ = self.info()
        kind = self.weight_type()
        w = np.zeros(max(m, 1), dtype=np.float64 if kind == 2 else np.int64)
        _check(self._lib.pgq_csr_download_weights(self._h, w.ctypes.data_as(C.c_void_p)))
        return w[:m]

    def cheapest_path_length(self, src, dst, src_valid=None, dst_valid=None):
        """-> (costs in the CSR's weight type, valid uint8, stats dict)"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        out = np.zeros(max(p, 1), dtype=np.float64 if self.weight_type() == 2 else np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        _check(self._lib.pgq_cheapest_path_length(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv),
                                                  out.ctypes.data_as(C.c_void_p), _pu8(ov), C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    def cheapest_path(self, src, dst, src_valid=None, dst_valid=None):
        """-> (list of [src, e1, v1, ..., dst] lists or None, stats dict): the cheapest path itself, with
        shortestpath's tie-break over the edges the costs make tight (include/duckpgq_b200.h, pgq_cheapest_path)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        offs = np.zeros(max(p, 1), dtype=np.int64)
        lens = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        elems = C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        _check(self._lib.pgq_cheapest_path(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), _p64(offs),
                                           _p64(lens), _pu8(ov), C.byref(elems), C.byref(total), C.byref(st)))
        try:  # (no rows: no element array)
            flat = np.ctypeslib.as_array(elems, shape=(total.value,)).copy() if elems else np.zeros(0, np.int64)
        finally:
            self._lib.pgq_free(elems)
        paths = [flat[offs[i]: offs[i] + lens[i]].tolist() if ov[i] else None for i in range(p)]
        return paths, st.as_dict()

    def cheapest_path_count(self, src, dst, src_valid=None, dst_valid=None):
        """-> (counts int64, valid uint8, stats dict): the number of cheapest paths of each row, the walks of edges its
        costs make tight, saturated at INT64_MAX, which also stands for infinitely many (include/duckpgq_b200.h,
        pgq_cheapest_path_count)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        _check(self._lib.pgq_cheapest_path_count(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), _p64(cnt),
                                                 _pu8(ov), C.byref(st)))
        return cnt[:p], ov[:p], st.as_dict()

    def all_cheapest_paths(self, src, dst, max_paths: int = 0, src_valid=None, dst_valid=None):
        """-> (per row: list of [src, e1, v1, ..., dst] paths or None, counts int64, stats dict): the first
        min(count, max_paths) cheapest paths of each row (all of them for max_paths = 0), fewest edges first, in step
        order within a length; path 0 is cheapest_path's (include/duckpgq_b200.h, pgq_all_cheapest_paths)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt, npaths, first = (np.zeros(max(p, 1), dtype=np.int64) for _ in range(3))
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        _check(self._lib.pgq_all_cheapest_paths(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), int(max_paths),
                                                _p64(cnt), _p64(npaths), _p64(first), _pu8(ov), C.byref(offs),
                                                C.byref(elems), C.byref(total), C.byref(st)))
        try:
            woff = np.ctypeslib.as_array(offs, shape=(total.value + 1,)).copy()
            flat = np.ctypeslib.as_array(elems, shape=(int(woff[-1]),)).copy() if woff[-1] else np.zeros(0, np.int64)
        finally:
            self._lib.pgq_free(offs)
            self._lib.pgq_free(elems)
        walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(total.value)]
        paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
        return paths, cnt[:p], st.as_dict()

    def finalize(self):
        _check(self._lib.pgq_csr_finalize(self._h))

    # ---- the other consumers of the CSR (ids n and n + 1 are the reference's two entries behind the vertices) ---
    def local_clustering_coefficient(self, src, src_valid=None):
        """-> (float32 coefficients, valid uint8, stats dict).  An id outside [0, n) raises (PGQ_ERR_RANGE)."""
        src = _i64(src)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        out = np.zeros(max(p, 1), dtype=np.float32)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        _check(self._lib.pgq_local_clustering_coefficient(self._h, p, _p64(src), _pu8(sv),
                                                          out.ctypes.data_as(C.POINTER(C.c_float)), _pu8(ov),
                                                          C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    def pagerank(self, src, src_valid=None):
        """-> (float64 ranks, valid uint8, iterations, stats dict).  Computed on the first call, cached after."""
        src = _i64(src)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        out = np.zeros(max(p, 1), dtype=np.float64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        it = C.c_int64(0)
        st = _native.PgqStats()
        _check(self._lib.pgq_pagerank(self._h, p, _p64(src), _pu8(sv), out.ctypes.data_as(C.POINTER(C.c_double)),
                                      _pu8(ov), C.byref(it), C.byref(st)))
        return out[:p], ov[:p], int(it.value), st.as_dict()

    def weakly_connected_component(self, src, src_valid=None):
        """-> (int64 component ids, valid uint8, stats dict).  Computed on the first call, cached after."""
        src = _i64(src)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        out = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        _check(self._lib.pgq_weakly_connected_component(self._h, p, _p64(src), _pu8(sv), _p64(out), _pu8(ov),
                                                        C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    # ---- introspection (get_csr_v / get_csr_e, pgq_scan.cpp:84-111) ------------------------------
    def info(self):
        n, m, b = C.c_int64(), C.c_int64(), C.c_int64()
        _check(self._lib.pgq_csr_info(self._h, C.byref(n), C.byref(m), C.byref(b)))
        return n.value, m.value, b.value

    def download(self):
        n, m, _ = self.info()
        v = np.zeros(n + 2, dtype=np.int64)
        e = np.zeros(max(m, 1), dtype=np.int64)
        ids = np.zeros(max(m, 1), dtype=np.int64)
        _check(self._lib.pgq_csr_download(self._h, _p64(v), _p64(e), _p64(ids)))
        return v, e[:m], ids[:m]

    def download_ve(self):
        """download() without the edge-id column (half the host memory for a full-size CSR)."""
        n, m, _ = self.info()
        v = np.zeros(n + 2, dtype=np.int64)
        e = np.zeros(max(m, 1), dtype=np.int64)
        _check(self._lib.pgq_csr_download(self._h, _p64(v), _p64(e), None))
        return v, e[:m], None

    # ---- path functions ---------------------------------------------------------------------------
    def iterativelength(self, src, dst, src_valid=None, options: Optional[Options] = None):
        """-> (lengths int64 [-1 where NULL], valid uint8, stats dict)"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        out = np.full(max(p, 1), -1, dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_iterativelength(self._h, p, _p64(src), _p64(dst), _pu8(sv), C.byref(opts), _p64(out),
                                             _pu8(ov), C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    def iterativelengthbidirectional(self, src, dst, src_valid=None, dst_valid=None,
                                     options: Optional[Options] = None):
        """-> (lengths int64 [-1 where NULL], valid uint8, stats dict): the reference's 512-lane batches, each lane
        searching from both ends along out-edges (include/duckpgq_b200.h, pgq_iterativelength_bidirectional)"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        out = np.full(max(p, 1), -1, dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_iterativelength_bidirectional(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv),
                                                           C.byref(opts), _p64(out), _pu8(ov), C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    def reachability(self, src, dst, src_valid=None, dst_valid=None, options: Optional[Options] = None):
        """-> (reachable uint8 [0 where NULL], valid uint8, stats dict): the rows of pgq_iterativelength, or with
        reference_batching the reference's 512-lane batches (include/duckpgq_b200.h, pgq_reachability)"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        out = np.zeros(max(p, 1), dtype=np.uint8)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_reachability(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                          _pu8(out), _pu8(ov), C.byref(st)))
        return out[:p], ov[:p], st.as_dict()

    def iterativelength_device(self, d_src: int, d_dst: int, p: int, d_out_len: int, d_out_valid: int,
                               d_src_valid: int = 0, stream: int = 0, options: Optional[Options] = None) -> dict:
        """Device-pointer form (raw addresses, e.g. torch.Tensor.data_ptr()); work runs on `stream`."""
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_iterativelength_device(self._h, p, d_src, d_dst, d_src_valid or None, C.byref(opts),
                                                    d_out_len, d_out_valid, stream or None, C.byref(st)))
        return st.as_dict()

    def shortestpath(self, src, dst, src_valid=None, options: Optional[Options] = None):
        """-> (list of [src, e1, v1, ..., dst] lists or None, stats dict)"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        offs = np.zeros(max(p, 1), dtype=np.int64)
        lens = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        elems = C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_shortestpath(self._h, p, _p64(src), _p64(dst), _pu8(sv), C.byref(opts), _p64(offs),
                                          _p64(lens), _pu8(ov), C.byref(elems), C.byref(total), C.byref(st)))
        try:
            flat = np.ctypeslib.as_array(elems, shape=(max(total.value, 1),)).copy()[: total.value]
        finally:
            self._lib.pgq_free(elems)
        paths = [flat[offs[i]: offs[i] + lens[i]].tolist() if ov[i] else None for i in range(p)]
        return paths, st.as_dict()

    def shortest_path_count(self, src, dst, src_valid=None, dst_valid=None, options: Optional[Options] = None):
        """-> (counts int64, valid uint8, stats dict): the number of shortest paths of each row, saturated at
        INT64_MAX, 0 under NULL (include/duckpgq_b200.h, pgq_shortest_path_count)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_shortest_path_count(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                                 _p64(cnt), _pu8(ov), C.byref(st)))
        return cnt[:p], ov[:p], st.as_dict()

    def all_shortest_paths(self, src, dst, max_paths: int = 0, src_valid=None, dst_valid=None,
                           options: Optional[Options] = None):
        """-> (per row: list of [src, e1, v1, ..., dst] lists or None, counts int64, stats dict): the first
        min(count, max_paths) shortest paths of each row in step order, all of them for max_paths = 0
        (include/duckpgq_b200.h, pgq_all_shortest_paths)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt = np.zeros(max(p, 1), dtype=np.int64)
        npaths = np.zeros(max(p, 1), dtype=np.int64)
        plen = np.zeros(max(p, 1), dtype=np.int64)
        offs = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        elems = C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_all_shortest_paths(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                                int(max_paths), _p64(cnt), _p64(npaths), _p64(plen), _p64(offs),
                                                _pu8(ov), C.byref(elems), C.byref(total), C.byref(st)))
        try:  # (no rows: no element array)
            flat = np.ctypeslib.as_array(elems, shape=(total.value,)).copy() if elems else np.zeros(0, np.int64)
        finally:
            self._lib.pgq_free(elems)
        paths = [flat[offs[i]: offs[i] + npaths[i] * plen[i]].reshape(npaths[i], plen[i]).tolist() if ov[i] else None
                 for i in range(p)]
        return paths, cnt[:p], st.as_dict()

    def shortest_k_paths(self, src, dst, k: int, src_valid=None, dst_valid=None, options: Optional[Options] = None,
                         mode: str = "WALK"):
        """-> (per row: list of [src, e1, v1, ..., dst] paths or None, npaths int64, stats dict): the first min(k,
        total) paths of each row in the path mode ("WALK", "TRAIL", "ACYCLIC" or "SIMPLE", any case), shortest first,
        in step order within a length (include/duckpgq_b200.h, pgq_shortest_k_paths / pgq_shortest_k_paths_mode)."""
        path_mode = path_mode_id(mode)
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        npaths = np.zeros(max(p, 1), dtype=np.int64)
        first = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_shortest_k_paths_mode(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                                   int(k), path_mode, _p64(npaths), _p64(first), _pu8(ov),
                                                   C.byref(offs), C.byref(elems), C.byref(total), C.byref(st)))
        try:
            woff = np.ctypeslib.as_array(offs, shape=(total.value + 1,)).copy()
            flat = np.ctypeslib.as_array(elems, shape=(int(woff[-1]),)).copy() if woff[-1] else np.zeros(0, np.int64)
        finally:
            self._lib.pgq_free(offs)
            self._lib.pgq_free(elems)
        walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(total.value)]
        paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
        return paths, npaths[:p], st.as_dict()

    def cheapest_k_paths(self, src, dst, k: int, src_valid=None, dst_valid=None, options: Optional[Options] = None,
                         mode: str = "WALK"):
        """-> (per row: list of [src, e1, v1, ..., dst] paths or None, per row: list of costs (int for BIGINT weights,
        float for DOUBLE) or None, npaths int64, stats dict): the first min(k, total) paths of each row in the path mode
        ("WALK", "TRAIL", "ACYCLIC" or "SIMPLE", any case), cheapest first, then by length and step order, over a CSR
        with weights >= 0 (include/duckpgq_b200.h, pgq_cheapest_k_paths)."""
        path_mode = path_mode_id(mode)
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        npaths = np.zeros(max(p, 1), dtype=np.int64)
        first = np.zeros(max(p, 1), dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        costs = C.c_void_p()
        total = C.c_int64(0)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_cheapest_k_paths(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                              int(k), path_mode, _p64(npaths), _p64(first), _pu8(ov), C.byref(offs),
                                              C.byref(elems), C.byref(costs), C.byref(total), C.byref(st)))
        try:
            woff = np.ctypeslib.as_array(offs, shape=(total.value + 1,)).copy()
            flat = np.ctypeslib.as_array(elems, shape=(int(woff[-1]),)).copy() if woff[-1] else np.zeros(0, np.int64)
            cbits = (np.ctypeslib.as_array(C.cast(costs, C.POINTER(C.c_int64)), shape=(total.value,)).copy()
                     if total.value else np.zeros(0, np.int64))
        finally:
            self._lib.pgq_free(offs)
            self._lib.pgq_free(elems)
            self._lib.pgq_free(costs)
        cvals = (cbits.view(np.float64) if self.weight_type() == 2 else cbits).tolist()
        walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(total.value)]
        paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
        cost_rows = [cvals[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
        return paths, cost_rows, npaths[:p], st.as_dict()

    def shortest_k_groups(self, src, dst, k: int, max_paths: int = 0, src_valid=None, dst_valid=None,
                          options: Optional[Options] = None, mode: str = "WALK"):
        """-> (per row: list of [src, e1, v1, ..., dst] paths or None, counts int64, ngroups int64, last_len int64,
        complete uint8, stats dict): every path of the k shortest lengths of each row in the path mode, in
        shortest_k_paths' order, the first max_paths of them for max_paths > 0.  counts is N, the number of such paths
        (-1 when a mode's row was cut by max_paths); last_len is the last group's length, -1 for none
        (include/duckpgq_b200.h, pgq_shortest_k_groups)."""
        path_mode = path_mode_id(mode)
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt, ngroups, last_len, npaths, first = (np.zeros(max(p, 1), dtype=np.int64) for _ in range(5))
        complete = np.zeros(max(p, 1), dtype=np.uint8)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        offs, elems = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)()
        total = C.c_int64(0)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_shortest_k_groups(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv), C.byref(opts),
                                               int(k), path_mode, int(max_paths), _p64(cnt), _p64(ngroups),
                                               _p64(last_len), _pu8(complete), _p64(npaths), _p64(first), _pu8(ov),
                                               C.byref(offs), C.byref(elems), C.byref(total), C.byref(st)))
        try:
            woff = np.ctypeslib.as_array(offs, shape=(total.value + 1,)).copy()
            flat = np.ctypeslib.as_array(elems, shape=(int(woff[-1]),)).copy() if woff[-1] else np.zeros(0, np.int64)
        finally:
            self._lib.pgq_free(offs)
            self._lib.pgq_free(elems)
        walks = [flat[woff[j]: woff[j + 1]].tolist() for j in range(total.value)]
        paths = [walks[first[i]: first[i] + npaths[i]] if ov[i] else None for i in range(p)]
        return paths, cnt[:p], ngroups[:p], last_len[:p], complete[:p], st.as_dict()

    def shortest_k_groups_count(self, src, dst, k: int, src_valid=None, dst_valid=None,
                                options: Optional[Options] = None):
        """-> (counts int64, ngroups int64, last_len int64, valid uint8, stats dict): WALK's N, saturated at INT64_MAX,
        with the groups found and the last group's length, from the counting pass alone
        (include/duckpgq_b200.h, pgq_shortest_k_groups_count)."""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        dv = None if dst_valid is None else np.ascontiguousarray(dst_valid, dtype=np.uint8)
        cnt, ngroups, last_len = (np.zeros(max(p, 1), dtype=np.int64) for _ in range(3))
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        st = _native.PgqStats()
        opts = (options or Options()).c()
        _check(self._lib.pgq_shortest_k_groups_count(self._h, p, _p64(src), _p64(dst), _pu8(sv), _pu8(dv),
                                                     C.byref(opts), int(k), _p64(cnt), _p64(ngroups), _p64(last_len),
                                                     _pu8(ov), C.byref(st)))
        return cnt[:p], ngroups[:p], last_len[:p], ov[:p], st.as_dict()

    def free(self):
        if getattr(self, "_h", None):
            self._lib.pgq_csr_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class MultiDeviceCSR:
    """pgq_multi_csr: a finished DeviceCSR replicated on several GPUs of the box (peer copies over NVLink); the
    search lanes of every call are dealt over the devices, one host thread each, no collective (SURVEY 8e)."""

    def __init__(self, primary: DeviceCSR, devices):
        self._lib = primary._lib
        self.primary = primary
        devs = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        _check(self._lib.pgq_multi_csr_create(primary._h, devs, len(devices), C.byref(h)))
        self._h = h
        self.n_devices = len(devices)

    def iterativelength(self, src, dst, src_valid=None, options: Optional[Options] = None):
        """-> (lengths, valid, [stats dict per device])"""
        src, dst = _i64(src), _i64(dst)
        p = src.shape[0]
        sv = None if src_valid is None else np.ascontiguousarray(src_valid, dtype=np.uint8)
        out = np.full(max(p, 1), -1, dtype=np.int64)
        ov = np.zeros(max(p, 1), dtype=np.uint8)
        sts = (_native.PgqStats * self.n_devices)()
        opts = (options or Options()).c()
        _check(self._lib.pgq_multi_iterativelength(self._h, p, _p64(src), _p64(dst), _pu8(sv), C.byref(opts), _p64(out),
                                                   _pu8(ov), sts))
        return out[:p], ov[:p], [s.as_dict() for s in sts]

    def free(self):
        if getattr(self, "_h", None):
            self._lib.pgq_multi_csr_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DuckPGQState:
    """Per-connection CSR registry (DuckPGQState, duckpgq_state.hpp:12-39)."""

    def __init__(self, ctx: Optional[Context] = None, device: int = 0):
        self.ctx = ctx or default_context(device)
        self.csr_list: dict[int, DeviceCSR] = {}
        self.csr_to_delete: set[int] = set()

    def get_csr(self, csr_id: int) -> DeviceCSR:
        # DuckPGQState::GetCSR, duckpgq_state.cpp:180-186
        if csr_id not in self.csr_list:
            raise ConstraintException(PGQ_ERR_INVALID_ID, f"CSR not found with ID {csr_id}")
        return self.csr_list[csr_id]

    def query_end(self):
        # DuckPGQState::QueryEnd, duckpgq_state.cpp:162-170
        for csr_id in list(self.csr_to_delete):
            csr = self.csr_list.pop(csr_id, None)
            if csr is not None:
                csr.free()
        self.csr_to_delete.clear()


def create_csr_vertex(state: DuckPGQState, csr_id: int, v_size: int, dense_id, cnt) -> np.ndarray:
    """create_csr_vertex(INT, BIGINT, BIGINT, BIGINT) -> BIGINT: stores the out-degree of each
    vertex, returns cnt per row (the SQL caller sum()s it)."""
    csr = state.csr_list.get(csr_id)
    if csr is None or not csr.initialized_v:  # CsrInitializeVertex, csr_creation.cpp:14-41
        csr = DeviceCSR.create(state.ctx, int(v_size))
        state.csr_list[csr_id] = csr
    cnt = _i64(cnt)
    csr.add_vertex_counts(dense_id, cnt)
    return cnt.copy()


def create_csr_edge(state: DuckPGQState, csr_id: int, v_size: int, edge_size: int, edge_size_count: int, src_rowid,
                    dst_rowid, edge_rowid, weight=None) -> np.ndarray:
    """create_csr_edge(INT, BIGINT x6 [, BIGINT | DOUBLE]) -> INT (1, or the weight cast to int32).  Raises the
    reference's ConstraintException when sum(cnt) != count(*) of the edge join and marks the id for deletion
    (csr_creation.cpp:121-125)."""
    if int(edge_size) != int(edge_size_count):
        state.csr_to_delete.add(csr_id)
        raise ConstraintException(PGQ_ERR_CONSTRAINT, _native.load().pgq_status_text(PGQ_ERR_CONSTRAINT).decode())
    csr = state.csr_list.get(csr_id)
    if csr is None:
        raise ConstraintException(PGQ_ERR_INVALID_ID, "Invalid ID")
    src_rowid = _i64(src_rowid)
    csr.add_edges(int(edge_size), int(edge_size_count), src_rowid, dst_rowid, edge_rowid, weight)
    if weight is not None:
        return np.asarray(weight).astype(np.int32)  # result_data[i] = static_cast<int32_t>(weight), csr_creation.cpp:167,193
    return np.ones(src_rowid.shape[0], dtype=np.int32)


def cheapest_path_length(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None, dst_valid=None):
    """cheapest_path_length(INT, BIGINT, BIGINT, BIGINT) -> BIGINT | DOUBLE (cheapest_path_length.cpp:138-166)."""
    csr = state.csr_list.get(csr_id)
    if csr is None:  # DuckPGQState::GetCSR, duckpgq_state.cpp:180-186
        raise ConstraintException(PGQ_ERR_INVALID_ID, f"CSR not found with ID {csr_id}")
    state.csr_to_delete.add(csr_id)  # the bind marks it, cheapest_path_length_function_data.cpp:20
    csr.finalize()
    cost, valid, _ = csr.cheapest_path_length(src, dst, src_valid, dst_valid)
    state.csr_to_delete.add(csr_id)  # cheapest_path_length.cpp:160
    return cost, valid


def cheapest_path(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None, dst_valid=None):
    """cheapest_path(INT, BIGINT, BIGINT, BIGINT) -> LIST(BIGINT): the cheapest path as [src, e1, v1, ..., ek, dst]
    rowids or None (no reference function; looked up and marked as cheapest_path_length is)."""
    csr = state.csr_list.get(csr_id)
    if csr is None:  # DuckPGQState::GetCSR, duckpgq_state.cpp:180-186
        raise ConstraintException(PGQ_ERR_INVALID_ID, f"CSR not found with ID {csr_id}")
    state.csr_to_delete.add(csr_id)
    csr.finalize()
    if csr.weight_type() == 0:  # CheapestPathLengthBind's check, cheapest_path_length_function_data.cpp:22-24
        raise ConstraintException(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path")
    paths, _ = csr.cheapest_path(src, dst, src_valid, dst_valid)
    state.csr_to_delete.add(csr_id)
    return paths


def _lookup_weighted(state: DuckPGQState, csr_id: int) -> DeviceCSR:
    csr = state.csr_list.get(csr_id)
    if csr is None:  # DuckPGQState::GetCSR, duckpgq_state.cpp:180-186
        raise ConstraintException(PGQ_ERR_INVALID_ID, f"CSR not found with ID {csr_id}")
    state.csr_to_delete.add(csr_id)
    csr.finalize()
    if csr.weight_type() == 0:  # CheapestPathLengthBind's check, cheapest_path_length_function_data.cpp:22-24
        raise ConstraintException(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing cheapest path")
    return csr


def cheapest_path_count(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None, dst_valid=None):
    """cheapest_path_count(INT, BIGINT, BIGINT, BIGINT) -> BIGINT: the number of cheapest paths, saturated at INT64_MAX
    (also for infinitely many), or NULL (no reference function; looked up and marked as cheapest_path is).  Returns
    (counts, valid)."""
    csr = _lookup_weighted(state, csr_id)
    counts, valid, _ = csr.cheapest_path_count(src, dst, src_valid, dst_valid)
    state.csr_to_delete.add(csr_id)
    return counts, valid


def all_cheapest_paths(state: DuckPGQState, csr_id: int, v_size: int, src, dst, max_paths: int = 0, src_valid=None,
                       dst_valid=None):
    """all_cheapest_paths(INT, BIGINT, BIGINT, BIGINT, BIGINT max_paths) -> LIST(LIST(BIGINT)): per row the first
    min(count, max_paths) cheapest paths (every one for max_paths = 0) or None (no reference function; looked up and
    marked as cheapest_path is)."""
    csr = _lookup_weighted(state, csr_id)
    paths, _, _ = csr.all_cheapest_paths(src, dst, max_paths, src_valid, dst_valid)
    state.csr_to_delete.add(csr_id)
    return paths


def cheapest_k_paths(state: DuckPGQState, csr_id: int, v_size: int, src, dst, k: int, src_valid=None, dst_valid=None,
                     options: Optional[Options] = None, mode: str = "WALK"):
    """cheapest_k_paths(INT, BIGINT, BIGINT, BIGINT, BIGINT k[, VARCHAR mode]) -> LIST(LIST(BIGINT)): per row the first
    min(k, total) paths of the path mode, cheapest first, or None (no reference function; looked up and marked as
    cheapest_path is).  Returns (paths, costs): costs per row in the CSR's weight type, or None."""
    path_mode_id(mode)
    csr = _lookup_weighted(state, csr_id)
    paths, costs, _, _ = csr.cheapest_k_paths(src, dst, k, src_valid, dst_valid, options, mode)
    state.csr_to_delete.add(csr_id)
    return paths, costs


def _lookup_for_path(state: DuckPGQState, csr_id: int, lengths: bool) -> DeviceCSR:
    state.csr_to_delete.add(csr_id)  # IterativeLengthBind marks at bind time, iterative_length_function_data.cpp:27
    if lengths and csr_id + 1 > len(state.csr_list):  # iterativelength.cpp:41-43
        raise ConstraintException(PGQ_ERR_INVALID_ID, "Invalid ID")
    csr = state.csr_list.get(csr_id)
    if csr is None:
        if lengths:  # iterativelength.cpp:44-47
            raise ConstraintException(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing shortest path")
        raise ConstraintException(PGQ_ERR_INVALID_ID, "Invalid ID")  # shortest_path.cpp:49-52
    if not csr.initialized_v:
        raise ConstraintException(PGQ_ERR_NOT_INITIALIZED, "Need to initialize CSR before doing shortest path")
    csr.finalize()  # no-op once built; the reference's CSR is complete when the CTE has been drained
    return csr


def iterativelength(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None,
                    options: Optional[Options] = None):
    """iterativelength(INT, BIGINT, BIGINT, BIGINT) -> BIGINT.  Returns (lengths, valid): hop count or
    NULL (valid 0, value -1) per row."""
    csr = _lookup_for_path(state, csr_id, lengths=True)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    out, valid, _ = csr.iterativelength(src, dst, src_valid, options)
    state.csr_to_delete.add(csr_id)  # iterativelength.cpp:142
    return out, valid


def iterativelengthbidirectional(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None,
                                 dst_valid=None, options: Optional[Options] = None):
    """iterativelengthbidirectional(INT, BIGINT, BIGINT, BIGINT) -> BIGINT.  Returns (lengths, valid): the meeting
    iteration + 1, 0 for src == dst, or NULL (valid 0, value -1) per row.  A missing or uninitialised CSR raises the
    texts of iterativelength (the reference only asserts)."""
    csr = _lookup_for_path(state, csr_id, lengths=True)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    out, valid, _ = csr.iterativelengthbidirectional(src, dst, src_valid, dst_valid, options)
    state.csr_to_delete.add(csr_id)  # iterativelength_bidirectional.cpp:152
    return out, valid


def reachability(state: DuckPGQState, csr_id: int, is_variant: bool, input_size: int, src, dst, src_valid=None,
                 dst_valid=None, options: Optional[Options] = None):
    """reachability(INTEGER, BOOLEAN, BIGINT, BIGINT, BIGINT) -> BOOLEAN (reachability.cpp:165-264).  Returns
    (reachable, valid): True / False per row, NULL (valid 0) for a NULL source or destination.  is_variant picks the
    reference's traversal, which does not change the answers: it is ignored.  A missing CSR raises GetCSR's text."""
    del is_variant
    csr = state.get_csr(csr_id)  # "CSR not found with ID %d", duckpgq_state.cpp:180-186
    if int(input_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG,
                                    f"input_size {input_size} does not match the CSR ({csr.n} vertices)")
    csr.finalize()
    out, valid, _ = csr.reachability(src, dst, src_valid, dst_valid, options)
    state.csr_to_delete.add(csr_id)  # l.253
    return out.astype(bool), valid


def shortestpath(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None,
                 options: Optional[Options] = None):
    """shortestpath(INT, BIGINT, BIGINT, BIGINT) -> LIST(BIGINT): [src, e1, v1, ..., ek, dst] rowids or None."""
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    paths, _ = csr.shortestpath(src, dst, src_valid, options)
    state.csr_to_delete.add(csr_id)  # shortest_path.cpp:206
    return paths


def shortest_path_count(state: DuckPGQState, csr_id: int, v_size: int, src, dst, src_valid=None, dst_valid=None,
                        options: Optional[Options] = None):
    """shortest_path_count(INT, BIGINT, BIGINT, BIGINT) -> BIGINT: the number of shortest paths, saturated at
    INT64_MAX (no reference function; looked up and marked as shortestpath is).  Returns (counts, valid)."""
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    counts, valid, _ = csr.shortest_path_count(src, dst, src_valid, dst_valid, options)
    state.csr_to_delete.add(csr_id)
    return counts, valid


def all_shortest_paths(state: DuckPGQState, csr_id: int, v_size: int, src, dst, max_paths: int = 0, src_valid=None,
                       dst_valid=None, options: Optional[Options] = None):
    """all_shortest_paths(INT, BIGINT, BIGINT, BIGINT, BIGINT max_paths) -> LIST(LIST(BIGINT)): per row the first
    min(count, max_paths) shortest paths (every one for max_paths = 0) or None (no reference function; looked up and
    marked as shortestpath is)."""
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    paths, _, _ = csr.all_shortest_paths(src, dst, max_paths, src_valid, dst_valid, options)
    state.csr_to_delete.add(csr_id)
    return paths


def shortest_k_paths(state: DuckPGQState, csr_id: int, v_size: int, src, dst, k: int, src_valid=None, dst_valid=None,
                     options: Optional[Options] = None, mode: str = "WALK"):
    """shortest_k_paths(INT, BIGINT, BIGINT, BIGINT, BIGINT k[, VARCHAR mode]) -> LIST(LIST(BIGINT)): per row the first
    min(k, total) paths of the path mode, shortest first, or None (no reference function; looked up and marked as
    shortestpath is)."""
    path_mode_id(mode)
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    paths, _, _ = csr.shortest_k_paths(src, dst, k, src_valid, dst_valid, options, mode)
    state.csr_to_delete.add(csr_id)
    return paths


def shortest_k_groups(state: DuckPGQState, csr_id: int, v_size: int, src, dst, k: int, max_paths: int = 0,
                      src_valid=None, dst_valid=None, options: Optional[Options] = None, mode: str = "WALK"):
    """shortest_k_groups(INT, BIGINT, BIGINT, BIGINT, BIGINT k, BIGINT max_paths[, VARCHAR mode]) ->
    LIST(LIST(BIGINT)): per row every path of the path mode whose length is among the row's k shortest, shortest first
    (the first max_paths of them for max_paths > 0), or None (no reference function; looked up and marked as
    shortestpath is)."""
    path_mode_id(mode)
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    paths = csr.shortest_k_groups(src, dst, k, max_paths, src_valid, dst_valid, options, mode)[0]
    state.csr_to_delete.add(csr_id)
    return paths


def shortest_k_groups_count(state: DuckPGQState, csr_id: int, v_size: int, src, dst, k: int, src_valid=None,
                            dst_valid=None, options: Optional[Options] = None):
    """shortest_k_groups_count(INT, BIGINT, BIGINT, BIGINT, BIGINT k) -> BIGINT: the number of walks whose length is
    among the row's k shortest, saturated at INT64_MAX (no reference function; looked up and marked as shortestpath
    is).  Returns (counts, valid)."""
    csr = _lookup_for_path(state, csr_id, lengths=False)
    if int(v_size) != csr.n:
        raise InvalidInputException(PGQ_ERR_INVALID_ARG, f"v_size {v_size} does not match the CSR ({csr.n} vertices)")
    counts, _, _, valid, _ = csr.shortest_k_groups_count(src, dst, k, src_valid, dst_valid, options)
    state.csr_to_delete.add(csr_id)
    return counts, valid


_NOT_INITIALIZED_TEXT = {  # the binds' texts: local_clustering_coefficient.cpp:22, pagerank.cpp:23,
    "lcc": "Need to initialize CSR before doing local clustering coefficient.",  # weakly_connected_component.cpp:47
    "pagerank": "Need to initialize CSR before running PageRank.",
    "wcc": "Need to initialize CSR before doing weakly connected components.",
}


def _lookup_for_analytics(state: DuckPGQState, csr_id: int, what: str) -> DeviceCSR:
    csr = state.csr_list.get(csr_id)
    if csr is None:
        raise ConstraintException(PGQ_ERR_INVALID_ID, "CSR not found. Is the graph populated?")
    if not (csr.initialized_v and csr.initialized_e):  # e.g. pagerank.cpp:22-24
        raise ConstraintException(PGQ_ERR_NOT_INITIALIZED, _NOT_INITIALIZED_TEXT[what])
    csr.finalize()
    return csr


def local_clustering_coefficient(state: DuckPGQState, csr_id: int, src, src_valid=None):
    """local_clustering_coefficient(INT, BIGINT) -> FLOAT (local_clustering_coefficient.cpp:14-70):
    (coefficients, valid)."""
    csr = _lookup_for_analytics(state, csr_id, "lcc")
    out, valid, _ = csr.local_clustering_coefficient(src, src_valid)
    state.csr_to_delete.add(csr_id)  # l.71
    return out, valid


def pagerank(state: DuckPGQState, csr_id: int, src, src_valid=None):
    """pagerank(INT, BIGINT) -> DOUBLE (pagerank.cpp:14-107): (ranks, valid)."""
    csr = _lookup_for_analytics(state, csr_id, "pagerank")
    out, valid, _, _ = csr.pagerank(src, src_valid)
    state.csr_to_delete.add(csr_id)
    return out, valid


def weakly_connected_component(state: DuckPGQState, csr_id: int, src, src_valid=None):
    """weakly_connected_component(INT, BIGINT) -> BIGINT (weakly_connected_component.cpp:37-104):
    (component ids, valid)."""
    csr = _lookup_for_analytics(state, csr_id, "wcc")
    out, valid, _ = csr.weakly_connected_component(src, src_valid)
    state.csr_to_delete.add(csr_id)
    return out, valid


def delete_csr(state: DuckPGQState, csr_id: int) -> bool:
    """delete_csr(INT) -> BOOLEAN (csr_deletion.cpp:10-20)."""
    csr = state.csr_list.pop(csr_id, None)
    if csr is None:
        return False
    csr.free()
    return True
