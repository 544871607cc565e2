#!/usr/bin/env python
"""Generate golden vectors of reachability with the UNMODIFIED reference (oracle/_ref/duckdb, built by
oracle/build_ref.sh).  Run in the build container only:

    python tests/golden/make_golden_reach.py

The reference reads both key columns of this function through UnifiedVectorFormat::data, a byte pointer
(reachability.cpp:177,181,26,241-242): row r searches from the BYTE at offset r of the column's data.  So, as in
make_golden_bidir.py, every case chooses the ids the searches use (`eff_src` / `eff_dst`, each < min(n, 256)) and spells
them into the first ceil(P / 8) int64 values of the columns, little-endian; the remaining values are noise.  NULLs only
sit in rows >= ceil(P / 8), whose values are never read as bytes; the byte of a row with a NULL destination is still
eff_dst (the reference reads it).  One statement per case and traversal, threads = 1 and P <= 2048 rows: one DataChunk,
one flat vector, rows in order.

The reference starts its next batch curr_batch_size rows -- the rows with a valid source -- after the last one
(l.251), so NULL sources make it re-run the last rows, and a batch that finds no valid source never ends.  Before a
statement runs, the generator replays that recurrence over the validity column (oracle/pgq_oracle_reach.py,
reference_batch_starts) and refuses a layout that would hang.

Each refr_<name>.npz holds the graph (n, edge rows src / dst), the column values handed to SQL (col_src, col_dst),
both validity columns, the ids the reference searched (eff_src, eff_dst = the byte view) and what it returned for
is_variant = false (reach0, reach0_valid) and true (reach1, reach1_valid).  Rows with a NULL source or destination
hold whatever the reference printed: their result is never written, or read through a NULL.
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
from oracle import pgq_oracle_reach as orr  # noqa: E402

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
    out = subprocess.run([DUCKDB, "-csv", "-noheader"], input=sql, capture_output=True, text=True, timeout=600)
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


def reference_rows(n, src, dst, col_src, col_dst, src_valid, dst_valid, is_variant):
    p = len(col_src)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": np.arange(n, dtype=np.int64)}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": np.asarray(src, np.int64), "dst": np.asarray(dst, np.int64)}), f"{td}/e.parquet")
        ps = pa.array(col_src, mask=~src_valid.astype(bool))
        pd = pa.array(col_dst, mask=~dst_valid.astype(bool))
        pq.write_table(pa.table({"i": np.arange(p, dtype=np.int64), "src": ps, "dst": pd}), f"{td}/p.parquet")
        # the CSR statement binds no path function, so the CSR outlives it; the second statement is a plain scan of
        # p: one flat DataChunk of p rows
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
CREATE TABLE p AS SELECT * FROM read_parquet('{td}/p.parquet');
CREATE TABLE t AS {CSR_CTE} SELECT count(cte1.temp) AS c FROM cte1;
SELECT p.i, reachability(0, {'true' if is_variant else 'false'}, {n}, p.src, p.dst) FROM p;
"""
        rows = list(csv.reader(io.StringIO(run_sql(sql))))
    assert len(rows) == p, (len(rows), p)
    reach = np.zeros(p, dtype=np.uint8)
    valid = np.zeros(p, dtype=np.uint8)
    for r in rows:
        i = int(r[0])
        if r[1] not in ("", "NULL"):
            reach[i] = 1 if r[1] == "true" else 0
            valid[i] = 1
    return reach, valid


def save(name, n, src, dst, eff_src, eff_dst, src_nulls=(), dst_nulls=(), seed=0):
    rng = np.random.default_rng(seed)
    eff_src = np.asarray(eff_src, dtype=np.uint8)
    eff_dst = np.asarray(eff_dst, dtype=np.uint8)
    p = len(eff_src)
    assert 0 < p <= 2048 and len(eff_dst) == p
    assert int(eff_src.max()) < n and int(eff_dst.max()) < n
    src_valid = np.ones(p, dtype=np.uint8)
    dst_valid = np.ones(p, dtype=np.uint8)
    for valid, rows in ((src_valid, src_nulls), (dst_valid, dst_nulls)):
        rows = np.asarray(rows, dtype=np.int64)
        assert np.all(rows >= (p + 7) // 8), "a NULL element would be read as bytes"
        valid[rows] = 0
    starts = orr.reference_batch_starts(eff_src, src_valid)  # raises ReferenceHang: the statement would never end
    col_src, col_dst = spell(eff_src, rng), spell(eff_dst, rng)
    res = {}
    for variant in (0, 1):
        reach, valid = reference_rows(n, src, dst, col_src, col_dst, src_valid, dst_valid, variant)
        res[f"reach{variant}"], res[f"reach{variant}_valid"] = reach, valid
    out = os.path.join(HERE, f"refr_{name}.npz")
    np.savez_compressed(out, n=np.int64(n), src=np.asarray(src, np.int32), dst=np.asarray(dst, np.int32),
                        col_src=col_src, col_dst=col_dst, src_valid=src_valid, dst_valid=dst_valid, eff_src=eff_src,
                        eff_dst=eff_dst, **res)
    ok = (src_valid & dst_valid).astype(bool)
    print(f"{name}: n={n} m={len(src)} rows={p} batch starts={starts} true={int(res['reach0'][ok].sum())}/"
          f"{int(ok.sum())} variant differs in {int((res['reach0'] != res['reach1'])[ok].sum())} rows "
          f"-> {os.path.getsize(out)} bytes")


def pairs(rng, n, p):
    k = min(n, 256)
    s = rng.integers(0, k, p)
    d = rng.integers(0, k, p)
    d[::9] = s[::9]  # src == dst
    if p > 20:
        s[5::13], d[5::13] = s[1], d[1]  # repeated pairs
    return s, d


def early_nulls(rng, p, count):
    """`count` NULL rows just behind the rows read as bytes: the reference re-runs the last `count` rows"""
    lo = (p + 7) // 8
    return np.sort(rng.choice(np.arange(lo, min(p - 1, lo + max(count * 4, 16))), count, replace=False))


def main():
    rng = np.random.default_rng(20261016)
    # the ref_* graphs, directed
    for g in ("student8", "student9", "rand40_nulls", "rand600_1300pairs", "chain200", "rmat10", "rmat12",
              "snb0003_allpairs", "edgeless4"):
        z = np.load(os.path.join(HERE, f"ref_{g}.npz"))
        n = int(z["n"])
        p = 600 if n > 8 else 40
        s, d = pairs(rng, n, p)
        save(g, n, z["src"], z["dst"], s, d, early_nulls(rng, p, 5), early_nulls(rng, p, 3), seed=len(g))
    # an undirected R-MAT-9 (both directions of every edge), a full chunk of 2048 rows
    n, s0, d0 = datagen.rmat_edges(9, seed=9)
    src, dst = np.concatenate([s0, d0]), np.concatenate([d0, s0])
    s, d = pairs(rng, n, 2048)
    save("rmat9_undirected", n, src, dst, s, d, early_nulls(rng, 2048, 40), early_nulls(rng, 2048, 20), seed=9)
    s, d = pairs(rng, n, 2048)
    save("rmat9_undirected_no_nulls", n, src, dst, s, d, seed=10)
    # a sink: every vertex points at 0, which has no out-edge
    n = 60
    s, d = pairs(rng, n, 300)
    save("sink", n, np.arange(1, n), np.zeros(n - 1, np.int64), s, d, early_nulls(rng, 300, 4), seed=60)
    # a directed cycle of 50 and a tail of 10 vertices leading into it
    n = 60
    cs = np.concatenate([np.arange(50), np.arange(50, 60)])
    cd = np.concatenate([(np.arange(50) + 1) % 50, np.concatenate([np.arange(51, 60), [0]])])
    s, d = pairs(rng, n, 500)
    save("cycle", n, cs, cd, s, d, early_nulls(rng, 500, 6), early_nulls(rng, 500, 6), seed=61)
    # the visit_list kept across batches (is_variant): 0 -> 1 -> {2 .. 9}; the first batch ends in mode 2 with
    # visit_list = {2 .. 9}; the NULL row 5 makes the reference start a second batch at row 23, which runs in mode 1
    # over that list and answers (0, 5) false
    n = 10
    p = 24
    s = np.zeros(p, np.int64)
    d = np.arange(p) % n
    d[-1] = 5
    save("stale_visit_list", n, np.array([0] + [1] * 8), np.arange(1, 10), s, d, [5], seed=62)


if __name__ == "__main__":
    main()
