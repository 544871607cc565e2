#!/usr/bin/env python
"""Golden vectors for the weighted CSR, cheapest_path_length and iterativelength2, produced by the UNMODIFIED
reference (oracle/_ref/duckdb).  Run in the build container only:

    python tests/golden/make_golden_weighted.py

Writes tests/golden/refw_<name>.npz: the inputs (n, edge rows with a BIGINT or DOUBLE weight, pairs) and what the
reference returned:
    w_type                csr_get_w_type(0)                               (csr_get_w_type.cpp)
    csr_v, csr_e, csr_w   get_csr_v(0) / get_csr_e(0) / get_csr_w(0)      (pgq_scan.cpp:84-141); the order of a vertex's
                          edges is the order in which DuckDB's join handed them to create_csr_edge -- compare per vertex
    cost, cost_valid      cheapest_path_length(0, n, src, dst)            (cheapest_path_length.cpp)
    length2, length2_valid  iterativelength2(0, n, src, dst)              (iterativelength2.cpp)
The weighted CSR is built by one statement (the 8-argument create_csr_edge overloads, csr_creation.cpp:227-235)
and queried by the next ones of the same CLI session, the way test/sql/scalar/get_csr_w_type.test does.
threads = 1: deterministic single-thread edge order.  All pairs have non-NULL sources (a NULL source shifts the
lanes of the reference's batch, cheapest_path_length.cpp:18-25 vs 88-93 -- see DESIGN.md section 7)."""
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

BUILD = """
SELECT count(CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid, k.w))
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst;
"""
PLAIN_CTE = """
WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(1, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(1, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
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


def save(name, n, src, dst, w, psrc, pdst, pdst_valid=None):
    src, dst, psrc, pdst = (np.asarray(x, dtype=np.int64) for x in (src, dst, psrc, pdst))
    w = np.asarray(w)
    is_f = w.dtype.kind == "f"
    P = len(psrc)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": np.arange(n, dtype=np.int64)}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": src, "dst": dst, "w": w.astype(np.float64 if is_f else np.int64)}), f"{td}/e.parquet")
        pdm = pa.array(pdst, mask=None if pdst_valid is None else ~pdst_valid.astype(bool))
        pq.write_table(pa.table({"i": np.arange(P, dtype=np.int64), "src": psrc, "dst": pdm}), f"{td}/p.parquet")
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
CREATE TABLE p AS SELECT * FROM read_parquet('{td}/p.parquet');
{BUILD}
.print ---T
SELECT csr_get_w_type(0);
.print ---V
SELECT csrv FROM get_csr_v(0);
.print ---E
SELECT csre FROM get_csr_e(0);
.print ---W
SELECT csrw FROM get_csr_w(0);
.print ---C
SELECT p.i, cheapest_path_length(0, (SELECT count(*) FROM v), p.src, p.dst) FROM p ORDER BY p.i;
.print ---L
{PLAIN_CTE} SELECT p.i, iterativelength2(1, (SELECT count(*) FROM v), p.src, p.dst) + __x.temp
  FROM p, (SELECT count(cte1.temp) * 0 AS temp FROM cte1) __x ORDER BY p.i;
"""
        txt = run_sql(sql)
    w_type = int(txt.split("---T\n")[1].split("---V\n")[0].strip())
    csr_v = np.array([int(x) for x in txt.split("---V\n")[1].split("---E\n")[0].split()], dtype=np.int64)
    csr_e = np.array([int(x) for x in txt.split("---E\n")[1].split("---W\n")[0].split()], dtype=np.int64)
    wpart = txt.split("---W\n")[1].split("---C\n")[0].split()
    cpart = txt.split("---C\n")[1].split("---L\n")[0]
    lpart = txt.split("---L\n")[1]
    csr_w = np.array([float(x) if is_f else int(x) for x in wpart], dtype=np.float64 if is_f else np.int64)
    cost = np.zeros(P, dtype=np.float64 if is_f else np.int64)
    cvalid = np.zeros(P, dtype=np.uint8)
    for r in csv.reader(io.StringIO(cpart)):
        if r[1] not in ("", "NULL"):
            cost[int(r[0])] = float(r[1]) if is_f else int(r[1])
            cvalid[int(r[0])] = 1
    l2 = np.full(P, -1, dtype=np.int64)
    l2v = np.zeros(P, dtype=np.uint8)
    for r in csv.reader(io.StringIO(lpart)):
        if r[1] not in ("", "NULL"):
            l2[int(r[0])] = int(r[1])
            l2v[int(r[0])] = 1
    out = os.path.join(HERE, f"refw_{name}.npz")
    np.savez_compressed(out, n=np.int64(n), src=src.astype(np.int32), dst=dst.astype(np.int32), w=w,
                        psrc=psrc.astype(np.int32), pdst=pdst.astype(np.int32),
                        pdst_valid=(np.ones(P, np.uint8) if pdst_valid is None else pdst_valid.astype(np.uint8)),
                        w_type=np.int64(w_type), csr_v=csr_v.astype(np.int32), csr_e=csr_e.astype(np.int32), csr_w=csr_w, cost=cost, cost_valid=cvalid, length2=l2.astype(np.int32),
                        length2_valid=l2v)
    print(f"{name}: n={n} m={len(src)} pairs={P} w_type={w_type} reachable={int(cvalid.sum())} -> {os.path.getsize(out)} bytes")


def main():
    rng = np.random.default_rng(77)
    # the 6-vertex example of the raw-UDF form, parallel edges with different weights
    save("tiny_i64", 6, [0, 1, 0, 2, 4, 0], [1, 2, 2, 3, 5, 1], np.array([5, 7, 20, 1, 2, 3]), [0, 0, 0, 4, 3, 1],
         [2, 3, 5, 5, 0, 1])
    # random multigraph, integer weights, 700 pairs (batches 256 + 256 + 128 + 32 + 16 + 8 + 4).  No NULL targets:
    # the reference indexes dists[] with the value under the NULL (cheapest_path_length.cpp:95-96) and aborts
    n = 300
    src, dst = datagen.random_graph(n, 1500, seed=5)
    ps, pd = rng.integers(0, n, 700), rng.integers(0, n, 700)
    save("rand300_i64", n, src, dst, rng.integers(1, 100, len(src)), ps, pd)
    # double weights (sums depend on the path order -> the bit-exactness claim), R-MAT shape
    n, src, dst = datagen.rmat_edges(9, edge_factor=6)
    ps, pd = datagen.hashed_pairs(400, n)
    save("rmat9_f64", n, src, dst, rng.random(len(src)) * 10.0 + 0.001, ps, pd)
    # a chain with shortcuts: many relaxation sweeps
    n = 150
    src = np.concatenate([np.arange(0, 149), rng.integers(0, 150, 40)])
    dst = np.concatenate([np.arange(1, 150), rng.integers(0, 150, 40)])
    save("chain150_f64", n, src, dst, rng.random(len(src)) + 0.5, rng.integers(0, n, 200), rng.integers(0, n, 200))
    # negative BIGINT weights on a DAG (no cycle can form: every edge runs from a lower to a higher rank of a random
    # permutation).  The reference relaxes from unreached vertices too, so a target that only an unreached vertex
    # reaches at a negative cost gets max/2 + that cost, a valid result; half of the pairs start at low ranks so
    # that many targets are reachable from their source as well
    n = 400
    src, dst, rank = dag_edges(rng, n, 1200)
    ps, pd = dag_pairs(rng, rank, 300)
    save("dagneg_i64", n, src, dst, rng.integers(-50, 51, len(src)), ps, pd)
    # dyadic doubles k/1024 (every path sum is exact), plus one -1e300 edge out of a vertex without in-edges: every
    # row whose target that edge reaches ends near 8.99e307 instead of NULL
    n = 300
    src, dst, rank = dag_edges(rng, n, 900)
    w = rng.integers(-(1 << 20) + 1, 1 << 20, len(src)) / 1024.0
    tail = int(np.argmin(rank))
    head = int(np.argsort(rank)[n // 10])
    src, dst, w = np.append(src, tail), np.append(dst, head), np.append(w, -1e300)
    ps, pd = dag_pairs(rng, rank, 300)
    save("dagdyadic_f64", n, src, dst, w, ps, pd)


def dag_edges(rng, n, m):
    """m random edges (plus a tenth as parallel twins), each oriented from the lower to the higher rank of a random
    permutation, self-loops dropped: a DAG, so negative weights cannot form a negative cycle."""
    rank = rng.permutation(n)
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    a, b = a[a != b], b[a != b]
    fwd = rank[a] < rank[b]
    src, dst = np.where(fwd, a, b), np.where(fwd, b, a)
    twin = rng.integers(0, len(src), len(src) // 10)
    return np.concatenate([src, src[twin]]), np.concatenate([dst, dst[twin]]), rank


def dag_pairs(rng, rank, p):
    """p pairs: the first half uniform, the second half from the lowest quarter of the ranks to the highest half."""
    n = len(rank)
    by_rank = np.argsort(rank)
    h = p // 2
    return (np.concatenate([rng.integers(0, n, h), by_rank[rng.integers(0, n // 4, p - h)]]),
            np.concatenate([rng.integers(0, n, h), by_rank[rng.integers(n // 2, n, p - h)]]))


if __name__ == "__main__":
    main()
