"""Build + ctypes binding of libduckpgq_b200.so (the C ABI declared in include/duckpgq_b200.h).

The library is compiled in-tree (duckpgq_extension_b200/lib/) for sm_90a (H100) only.  There is no CPU
fallback: if the shared library is missing or cannot be loaded, load() raises.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_PKG)
CSRC = os.path.join(_PKG, "csrc")
INCLUDE = os.path.join(ROOT, "include")
LIB_DIR = os.path.join(_PKG, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libduckpgq_b200.so")
SOURCES = ["pgq_csr.cu", "pgq_bfs.cu", "pgq_api.cu", "pgq_cheapest.cu", "pgq_allshortest.cu", "pgq_kshortest.cu",
           "pgq_kpaths_modes.cu", "pgq_cheapest_k.cu",
           "pgq_multi.cu", "pgq_analytics.cu"]
HEADERS = ["pgq_internal.h", "pgq_tile.cuh", "pgq_pull.cuh", "pgq_count.cuh", "pgq_bf.cuh", "pgq_kpaths.cuh"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libduckpgq_b200.so")


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.join(INCLUDE, "duckpgq_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc -gencode arch=compute_90a,code=sm_90a ... ->duckpgq_extension_b200/lib/libduckpgq_b200.so"""
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + ["-I", INCLUDE, "-I", CSRC, "-o", LIB_PATH] + [os.path.join(CSRC, f) for f in SOURCES]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    subprocess.check_call(cmd)
    return LIB_PATH


class PgqOptions(C.Structure):
    _fields_ = [("lanes", C.c_int32), ("direction", C.c_int32), ("alpha", C.c_int32), ("flags", C.c_int32),
                ("shard_index", C.c_int32), ("shard_count", C.c_int32)]


class PgqStats(C.Structure):
    _fields_ = [
        ("batches", C.c_int64), ("levels", C.c_int64), ("edges_traversed", C.c_int64),
        ("frontier_vertices", C.c_int64), ("push_levels", C.c_int64), ("pull_levels", C.c_int64),
        ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
        ("expand_ms", C.c_double), ("total_ms", C.c_double), ("lanes", C.c_int32), ("reserved", C.c_int32),
        ("searches", C.c_int64), ("pruned", C.c_int64), ("search_rows", C.c_int64),
        ("pull_ms", C.c_double), ("pull_edges", C.c_int64),
    ]

    def as_dict(self) -> dict:
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


# every symbol include/duckpgq_b200.h declares: name -> (restype, argtypes)
_P64 = C.POINTER(C.c_int64)
_PU8 = C.POINTER(C.c_uint8)
_VP = C.c_void_p
SYMBOLS = {
    "pgq_abi_version": (C.c_int, []),
    "pgq_last_error": (C.c_char_p, []),
    "pgq_status_text": (C.c_char_p, [C.c_int]),
    "pgq_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "pgq_ctx_create": (C.c_int, [C.c_int, C.POINTER(_VP)]),
    "pgq_ctx_destroy": (None, [_VP]),
    "pgq_csr_create": (C.c_int, [_VP, C.c_int64, C.POINTER(_VP)]),
    "pgq_csr_add_vertex_counts": (C.c_int, [_VP, C.c_int64, _P64, _P64, _P64]),
    "pgq_csr_add_edges": (C.c_int, [_VP, C.c_int64, C.c_int64, C.c_int64, _P64, _P64, _P64]),
    "pgq_csr_add_edges_weighted": (C.c_int, [_VP, C.c_int64, C.c_int64, C.c_int64, _P64, _P64, _P64, _P64,
                                             C.POINTER(C.c_double)]),
    "pgq_csr_finalize": (C.c_int, [_VP]),
    "pgq_csr_free": (None, [_VP]),
    "pgq_csr_build": (C.c_int, [_VP, C.c_int64, C.c_int64, _P64, _P64, _P64, C.POINTER(_VP)]),
    "pgq_csr_upload": (C.c_int, [_VP, C.c_int64, C.c_int64, _P64, _P64, _P64, C.POINTER(_VP)]),
    "pgq_csr_build_device": (C.c_int, [_VP, C.c_int64, C.c_int64, _VP, _VP, _VP, C.POINTER(_VP)]),
    "pgq_csr_build_keys": (C.c_int, [_VP, C.c_int64, _P64, _PU8, C.c_int64, _P64, _P64, _PU8, _PU8, C.POINTER(_VP)]),
    "pgq_csr_build_keys_device": (C.c_int, [_VP, C.c_int64, _VP, _VP, C.c_int64, _VP, _VP, _VP, _VP, C.POINTER(_VP)]),
    "pgq_csr_build_keys_undirected": (C.c_int, [_VP, C.c_int64, _P64, _PU8, C.c_int64, _P64, _P64, _PU8, _PU8,
                                                C.POINTER(_VP)]),
    "pgq_csr_build_keys_undirected_device": (C.c_int, [_VP, C.c_int64, _VP, _VP, C.c_int64, _VP, _VP, _VP, _VP,
                                                       C.POINTER(_VP)]),
    "pgq_csr_build_weighted": (C.c_int, [_VP, C.c_int64, C.c_int64, _P64, _P64, _P64, _P64, C.POINTER(C.c_double),
                                         C.POINTER(_VP)]),
    "pgq_csr_build_device_weighted": (C.c_int, [_VP, C.c_int64, C.c_int64, _VP, _VP, _VP, _VP, _VP, C.POINTER(_VP)]),
    "pgq_csr_upload_weighted": (C.c_int, [_VP, C.c_int64, C.c_int64, _P64, _P64, _P64, _P64, C.POINTER(C.c_double),
                                          C.POINTER(_VP)]),
    "pgq_csr_build_keys_weighted": (C.c_int, [_VP, C.c_int64, _P64, _PU8, C.c_int64, _P64, _P64, _PU8, _PU8, _P64,
                                              C.POINTER(C.c_double), _PU8, C.POINTER(_VP)]),
    "pgq_csr_build_keys_weighted_device": (C.c_int, [_VP, C.c_int64, _VP, _VP, C.c_int64, _VP, _VP, _VP, _VP, _VP, _VP,
                                                     _VP, C.POINTER(_VP)]),
    "pgq_csr_download": (C.c_int, [_VP, _P64, _P64, _P64]),
    "pgq_csr_info": (C.c_int, [_VP, _P64, _P64, _P64]),
    "pgq_csr_weight_type": (C.c_int, [_VP, C.POINTER(C.c_int)]),
    "pgq_csr_download_weights": (C.c_int, [_VP, _VP]),
    "pgq_iterativelength": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, C.POINTER(PgqOptions), _P64, _PU8,
                                      C.POINTER(PgqStats)]),
    "pgq_iterativelength_bidirectional": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, C.POINTER(PgqOptions),
                                                    _P64, _PU8, C.POINTER(PgqStats)]),
    "pgq_reachability": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, C.POINTER(PgqOptions), _PU8, _PU8,
                                   C.POINTER(PgqStats)]),
    "pgq_shortestpath": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, C.POINTER(PgqOptions), _P64, _P64, _PU8,
                                   C.POINTER(_P64), _P64, C.POINTER(PgqStats)]),
    "pgq_free": (None, [_VP]),
    "pgq_cheapest_path_length": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, _PU8, C.POINTER(PgqStats)]),
    "pgq_cheapest_path": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _P64, _P64, _PU8, C.POINTER(_P64), _P64,
                                    C.POINTER(PgqStats)]),
    "pgq_cheapest_path_count": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _P64, _PU8, C.POINTER(PgqStats)]),
    "pgq_all_cheapest_paths": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, C.c_int64, _P64, _P64, _P64, _PU8,
                                         C.POINTER(_P64), C.POINTER(_P64), _P64, C.POINTER(PgqStats)]),
    "pgq_shortest_path_count": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, _P64, _PU8,
                                          C.POINTER(PgqStats)]),
    "pgq_all_shortest_paths": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, _P64, _P64, _P64, _P64,
                                         _PU8, C.POINTER(_P64), _P64, C.POINTER(PgqStats)]),
    "pgq_shortest_k_paths": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, _P64, _P64, _PU8,
                                       C.POINTER(_P64), C.POINTER(_P64), _P64, C.POINTER(PgqStats)]),
    "pgq_shortest_k_paths_mode": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, C.c_int32, _P64,
                                            _P64, _PU8, C.POINTER(_P64), C.POINTER(_P64), _P64, C.POINTER(PgqStats)]),
    "pgq_cheapest_k_paths": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, C.c_int32, _P64, _P64,
                                       _PU8, C.POINTER(_P64), C.POINTER(_P64), C.POINTER(_VP), _P64,
                                       C.POINTER(PgqStats)]),
    "pgq_shortest_k_groups": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, C.c_int32, C.c_int64,
                                        _P64, _P64, _P64, _PU8, _P64, _P64, _PU8, C.POINTER(_P64), C.POINTER(_P64),
                                        _P64, C.POINTER(PgqStats)]),
    "pgq_shortest_k_groups_count": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, _PU8, _VP, C.c_int64, _P64, _P64, _P64,
                                              _PU8, C.POINTER(PgqStats)]),
    "pgq_local_clustering_coefficient": (C.c_int, [_VP, C.c_int64, _P64, _PU8, C.POINTER(C.c_float), _PU8,
                                                   C.POINTER(PgqStats)]),
    "pgq_pagerank": (C.c_int, [_VP, C.c_int64, _P64, _PU8, C.POINTER(C.c_double), _PU8, _P64, C.POINTER(PgqStats)]),
    "pgq_weakly_connected_component": (C.c_int, [_VP, C.c_int64, _P64, _PU8, _P64, _PU8, C.POINTER(PgqStats)]),
    "pgq_csr_clone": (C.c_int, [_VP, _VP, C.POINTER(_VP)]),
    "pgq_multi_csr_create": (C.c_int, [_VP, C.POINTER(C.c_int), C.c_int, C.POINTER(_VP)]),
    "pgq_multi_csr_devices": (C.c_int, [_VP, C.POINTER(C.c_int)]),
    "pgq_multi_csr_free": (None, [_VP]),
    "pgq_multi_iterativelength": (C.c_int, [_VP, C.c_int64, _P64, _P64, _PU8, C.POINTER(PgqOptions), _P64, _PU8,
                                            C.POINTER(PgqStats)]),
    "pgq_iterativelength_device": (C.c_int, [_VP, C.c_int64, _VP, _VP, _VP, C.POINTER(PgqOptions), _VP, _VP, _VP,
                                             C.POINTER(PgqStats)]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree library and bind every declared symbol.  Raises if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA library has not been built "
            "(run `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the export is missing
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib
