#!/usr/bin/env python
"""Generate golden vectors of iterativelengthbidirectional with the UNMODIFIED reference (oracle/_ref/duckdb, built by
oracle/build_ref.sh).  Run in the build container only:

    python tests/golden/make_golden_bidir.py

The reference reads the key columns of this function through UnifiedVectorFormat::data, a byte pointer
(iterativelength_bidirectional.cpp:61-62,104-110): row r's source is the BYTE at offset r of the column's data, not the
row's value.  So every case chooses the ids the searches should use (`eff_src` / `eff_dst`, each < min(n, 256), so that
no byte indexes past the reference's masks) and spells them into the first ceil(P / 8) int64 values of the columns,
little-endian; the remaining values are noise.  NULL sources only sit in rows >= ceil(P / 8), whose values are never
read as bytes.  One statement per case, threads = 1 and P <= 2048 rows: one DataChunk, one flat vector, rows in order.

Each refb_<name>.npz holds the graph (n, edge rows src / dst), the column values handed to SQL (col_src, col_dst),
the source validity, the ids the reference searched (eff_src, eff_dst = the byte view) and what it returned
(length, length_valid).  tests/test_oracle_bidir_golden.py checks that the byte view of the columns is eff_* and that
the restatement of oracle/pgq_oracle_bidir.c returns the reference's rows on it.
"""
import csv
import io
import os
import subprocess
import sys
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from duckpgq_extension_b200 import datagen  # noqa: E402

DUCKDB = os.path.join(ROOT, "oracle", "_ref", "duckdb")

CSR_CTE = """
WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid) AS temp
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst)
"""


def run_sql(sql: str) -> str:
    out = subprocess.run([DUCKDB, "-csv", "-noheader"], input=sql, capture_output=True, text=True)
    if out.returncode != 0 or "Error" in out.stderr:
        raise RuntimeError(out.stderr + out.stdout)
    return out.stdout


def spell(eff, rng):
    """int64 column whose byte view starts with eff (uint8 values), noise behind"""
    p = len(eff)
    words = (p + 7) // 8
    col = rng.integers(-(1 << 62), 1 << 62, p, dtype=np.int64)
    packed = np.zeros(words * 8, dtype=np.uint8)
    packed[:p] = eff
    col[:words] = packed.view("<i8")
    assert np.array_equal(col.view(np.uint8)[:p], eff)
    return col


def reference_rows(n, src, dst, col_src, col_dst, src_valid):
    p = len(col_src)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": np.arange(n, dtype=np.int64)}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": np.asarray(src, np.int64), "dst": np.asarray(dst, np.int64)}), f"{td}/e.parquet")
        ps = pa.array(col_src, mask=~src_valid.astype(bool))
        pq.write_table(pa.table({"i": np.arange(p, dtype=np.int64), "src": ps, "dst": col_dst}), f"{td}/p.parquet")
        # the CSR statement binds no path function, so the CSR outlives it (SURVEY 8b); the second statement is
        # a plain scan of p: one flat DataChunk of p rows
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
CREATE TABLE p AS SELECT * FROM read_parquet('{td}/p.parquet');
CREATE TABLE t AS {CSR_CTE} SELECT count(cte1.temp) AS c FROM cte1;
SELECT p.i, iterativelengthbidirectional(0, {n}, p.src, p.dst) FROM p;
"""
        rows = list(csv.reader(io.StringIO(run_sql(sql))))
    assert len(rows) == p, (len(rows), p)
    length = np.full(p, -1, dtype=np.int64)
    valid = np.zeros(p, dtype=np.uint8)
    for r in rows:
        i = int(r[0])
        if r[1] not in ("", "NULL"):
            length[i] = int(r[1])
            valid[i] = 1
    return length, valid


def save(name, n, src, dst, eff_src, eff_dst, null_rows=(), seed=0):
    rng = np.random.default_rng(seed)
    eff_src = np.asarray(eff_src, dtype=np.uint8)
    eff_dst = np.asarray(eff_dst, dtype=np.uint8)
    p = len(eff_src)
    assert 0 < p <= 2048 and len(eff_dst) == p
    assert int(eff_src.max()) < n and int(eff_dst.max()) < n
    src_valid = np.ones(p, dtype=np.uint8)
    null_rows = np.asarray(null_rows, dtype=np.int64)
    assert np.all(null_rows >= (p + 7) // 8), "a NULL element would be read as bytes"
    src_valid[null_rows] = 0
    col_src, col_dst = spell(eff_src, rng), spell(eff_dst, rng)
    length, valid = reference_rows(n, src, dst, col_src, col_dst, src_valid)
    out = os.path.join(HERE, f"refb_{name}.npz")
    np.savez_compressed(out, n=np.int64(n), src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32),
                        col_src=col_src, col_dst=col_dst, src_valid=src_valid, eff_src=eff_src, eff_dst=eff_dst,
                        length=length.astype(np.int32), length_valid=valid)
    print(f"{name}: n={n} m={len(src)} rows={p} met={int((valid & (length > 0)).sum())} "
          f"zero={int((valid & (length == 0)).sum())} -> {os.path.getsize(out)} bytes")


def pairs(rng, n, p, trivial=True, repeat=True):
    k = min(n, 256)
    s = rng.integers(0, k, p)
    d = rng.integers(0, k, p)
    if trivial:
        d[::9] = s[::9]  # src == dst: 0 without a lane
    if repeat and p > 20:
        s[5::13], d[5::13] = s[1], d[1]  # repeated pairs
    return s, d


def nulls(rng, p, frac=0.08):
    lo = (p + 7) // 8
    return np.nonzero(rng.random(p - lo) < frac)[0] + lo


def coupling_graph():
    """X = (0, 1): 0 is a sink and 1 -> 0, so X's source side dies at once; Y = (2, 9): 2 -> 3 -> 4 -> 5 keeps growing."""
    return 10, np.array([1, 2, 3, 4]), np.array([0, 3, 4, 5])


def main():
    rng = np.random.default_rng(20261016)
    # the ref_* graphs, directed
    for g in ("student8", "student9", "rand40_nulls", "rand600_1300pairs", "chain200", "rmat10", "rmat12",
              "snb0003_allpairs", "edgeless4"):
        z = np.load(os.path.join(HERE, f"ref_{g}.npz"))
        n = int(z["n"])
        p = 600 if n > 8 else 25
        s, d = pairs(rng, n, p)
        save(g, n, z["src"], z["dst"], s, d, nulls(rng, p), seed=len(g))
    # an undirected R-MAT-9 (both directions of every edge)
    n, s0, d0 = datagen.rmat_edges(9, seed=9)
    src, dst = np.concatenate([s0, d0]), np.concatenate([d0, s0])
    s, d = pairs(rng, n, 1500)
    save("rmat9_undirected", n, src, dst, s, d, nulls(rng, 1500), seed=9)
    # the coupling across lanes: X alone is NULL, X behind Y is 2
    n, src, dst = coupling_graph()
    save("coupling_alone", n, src, dst, [0], [1])
    save("coupling_with_y", n, src, dst, [2, 0], [9, 1])
    # 513..2048 rows (512 lanes; rows with src == dst and NULL rows take none): X as row 513 is alone in the second
    # batch (NULL); as row 514 it shares the second batch with a growing row (2); behind 511 lane rows and 300 trivial
    # rows it is the last lane of the first batch (2)
    fill_s, fill_d = np.full(600, 2), np.full(600, 8)
    save("coupling_x_alone_in_batch_2_513", n, src, dst, np.concatenate([[2], fill_s[:511], [0]]),
         np.concatenate([[9], fill_d[:511], [1]]))
    save("coupling_x_with_y_in_batch_2_514", n, src, dst, np.concatenate([[2], fill_s[:512], [0]]),
         np.concatenate([[9], fill_d[:512], [1]]))
    s = np.concatenate([[2], fill_s[:510], np.full(300, 7), [0]])
    d = np.concatenate([[9], fill_d[:510], np.full(300, 7), [1]])
    save("coupling_trivial_rows_812", n, src, dst, s, d, nulls(rng, len(s), 0.2))
    # exactly 1024 lane rows followed by trivial and NULL rows: the reference's empty third batch
    s = np.concatenate([np.full(1024, 2), np.full(200, 5)])
    d = np.concatenate([np.full(1024, 8), np.full(200, 5)])
    save("full_batches_1224", n, src, dst, s, d, np.arange(1100, 1224, 3))
    # 2048 rows on R-MAT-10, several batches
    z = np.load(os.path.join(HERE, "ref_rmat10.npz"))
    s, d = pairs(rng, 1024, 2048)
    save("rmat10_2048rows", 1024, z["src"], z["dst"], s, d, nulls(rng, 2048), seed=2048)


if __name__ == "__main__":
    main()
