#!/usr/bin/env python
"""Golden vectors for the CSR built from key columns (pgq_csr_build_keys), produced by the UNMODIFIED reference
(oracle/_ref/duckdb, threads = 1) with the directed CSR CTE of make_golden_next4.py.  Run in the build container
only:

    python tests/golden/make_golden_keys.py

Writes tests/golden/refk_<name>.npz:
    vkey                  the vertex table's key column v.id (rowid = position)
    src, dst, src_valid, dst_valid    the edge table's key columns e.src / e.dst (rowid = position, 0 = NULL)
    constraint            1 if the reference raised the ConstraintException of csr_creation.cpp:121-125
    csr_v, csr_e          get_csr_v(0) / get_csr_e(0) (pgq_scan.cpp:84-111) when it did not
The vertex keys are never NULL here: the reference sizes the CSR by count(v.id) (compressed_sparse_row.cpp:106-111)
but writes v[rowid + 2] for every vertex row, so a NULL vertex key makes it write past its array."""
import os
import sys
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_next4 import BUILD, datagen, run_sql  # noqa: E402

CONSTRAINT_TEXT = "Non-existent/non-unique vertices detected"
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def save(name, vkey, src, dst, src_valid=None, dst_valid=None):
    vkey, src, dst = (np.asarray(x, dtype=np.int64) for x in (vkey, src, dst))
    m = src.shape[0]
    sv = np.ones(m, dtype=np.uint8) if src_valid is None else np.asarray(src_valid, dtype=np.uint8)
    dv = np.ones(m, dtype=np.uint8) if dst_valid is None else np.asarray(dst_valid, dtype=np.uint8)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": pa.array(vkey, type=pa.int64())}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": pa.array(src, type=pa.int64(), mask=sv == 0),
                                 "dst": pa.array(dst, type=pa.int64(), mask=dv == 0)}), f"{td}/e.parquet")
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
{BUILD.format(id=0)}
.print ---V
SELECT csrv FROM get_csr_v(0);
.print ---E
SELECT csre FROM get_csr_e(0);
"""
        try:
            txt = run_sql(sql)
            constraint = 0
        except RuntimeError as ex:
            if CONSTRAINT_TEXT not in str(ex):
                raise
            constraint = 1
    if constraint:
        csr_v = csr_e = np.zeros(0, dtype=np.int64)
    else:
        csr_v = np.array([int(x) for x in txt.split("---V\n")[1].split("---E\n")[0].split()], dtype=np.int64)
        csr_e = np.array([int(x) for x in txt.split("---E\n")[1].split()], dtype=np.int64)
    out = os.path.join(HERE, f"refk_{name}.npz")
    np.savez_compressed(out, vkey=vkey, src=src, dst=dst, src_valid=sv, dst_valid=dv, constraint=np.int64(constraint),
                        csr_v=csr_v, csr_e=csr_e)
    print(f"{name}: n={vkey.shape[0]} m={m} constraint={constraint} rows={csr_e.shape[0]} -> {os.path.getsize(out)} bytes")


def main():
    rng = np.random.default_rng(2024)
    # keys = a shuffled range: every edge matches exactly one source and one destination row
    n = 500
    keys = rng.permutation(n)
    save("shuffled500", keys, rng.choice(keys, 2500), rng.choice(keys, 2500))
    # sparse keys of both signs
    keys = rng.choice(np.arange(-10**12, 10**12, 7919), 300, replace=False)
    save("sparse_signed300", keys, rng.choice(keys, 1500), rng.choice(keys, 1500))
    # the int64 extremes and their neighbours next to small keys
    keys = np.array([I64_MAX, 0, I64_MIN, -1, I64_MAX - 1, 1, I64_MIN + 1, 42, -42, 2**32, -(2**32)], dtype=np.int64)
    save("extremes11", keys, rng.choice(keys, 120), rng.choice(keys, 120))
    # duplicated source keys: vertex rows 0..39 hold keys 0..19 twice, rows 40..59 hold unique keys 100..119;
    # destinations only use unique keys, so every edge is legal and lands under each matching source row
    keys = np.concatenate([np.arange(20), rng.permutation(20), 100 + np.arange(20)])
    src = rng.choice(keys, 400)
    save("dupsrc60", keys, src, 100 + rng.integers(0, 20, 400))
    # NULL and dangling keys that the joins drop: a NULL or unmatched source (whatever its destination) and a NULL
    # destination behind a NULL source
    n = 200
    keys = rng.permutation(n) * 3
    m = 1200
    src, dst = rng.choice(keys, m), rng.choice(keys, m)
    src_valid = (rng.random(m) > 0.15).astype(np.uint8)
    src[rng.random(m) < 0.1] = 1  # no vertex has key 1 (all keys are multiples of 3)
    dst_valid = np.where(src_valid == 0, (rng.random(m) > 0.5), 1).astype(np.uint8)
    dst[(src == 1) & (rng.random(m) < 0.5)] = 2  # unmatched source with unmatched destination
    save("nulls200", keys, src, dst, src_valid, dst_valid)
    # an R-MAT graph (duplicates and self-loops kept) under a random sparse relabelling
    n, s, d = datagen.rmat_edges(9)
    keys = rng.choice(np.arange(-(2**40), 2**40, 104729), n, replace=False)
    save("rmat9_relabelled", keys, keys[s], keys[d])
    # (an edge table that joins to no row -- empty, or no key matching -- leaves this statement without a CSR: the
    # reference creates it in the first create_csr_edge call, and there is none)
    # what the reference rejects: a dangling destination, a duplicated destination
    keys = np.arange(30)
    src, dst = rng.choice(keys, 60), rng.choice(keys, 60)
    dst[17] = 1000
    save("dangling_dst", keys, src, dst)
    keys = np.concatenate([np.arange(30), [4]])
    src, dst = rng.choice(np.arange(5, 30), 60), rng.choice(np.arange(5, 30), 60)
    dst[9] = 4
    save("duplicate_dst", keys, src, dst)


if __name__ == "__main__":
    main()
