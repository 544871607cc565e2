"""duckpgq_extension_b200 -- H100-native path-finding hot path of DuckPGQ (iterativelength /
shortestpath over the create_csr_* CSR) behind the reference's scalar-function interface.

  include/duckpgq_b200.h   the C ABI (drop-in boundary)
  csrc/                    sm_90a CUDA kernels + the C ABI implementation -> lib/libduckpgq_b200.so
  pgq.py                   host-side mirror of the reference UDFs (same names / arguments / errors)
  datagen.py               synthetic inputs of BASELINE.json's configs (R-MAT, SNB-shaped, pairs)
  sharding.py              multi-GPU: pairs sharded over ranks, CSR replicated, results gathered
"""
from .pgq import (  # noqa: F401
    ConstraintException, Context, DeviceCSR, DuckPGQState, InvalidInputException, Options, PgqError,
    create_csr_edge, create_csr_vertex, default_context, delete_csr, iterativelength, shortestpath,
)
