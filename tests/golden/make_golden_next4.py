#!/usr/bin/env python
"""Golden vectors for the reference's other CSR consumers (SURVEY section 8f NEXT-4), produced by the UNMODIFIED
reference (oracle/_ref/duckdb).  Run in the build container only:

    python tests/golden/make_golden_next4.py

Writes tests/golden/refn4_<name>.npz: the inputs (n, edge rows) and what the reference returned for EVERY vertex:
    csr_v, csr_e          get_csr_v(0) / get_csr_e(0)                     (pgq_scan.cpp)
    lcc                   local_clustering_coefficient(0, rowid)  FLOAT   (local_clustering_coefficient.cpp)
    wcc                   weakly_connected_component(1, rowid)    BIGINT  (weakly_connected_component.cpp)
    pagerank              pagerank(2, rowid)                      DOUBLE  (pagerank.cpp)
Each function marks its CSR for deletion, so three CSRs are built from the same statement (threads = 1: the same
edge order in all of them).  The scalar functions are called directly, on whatever CSR the statement built -- the
reference's table-function wrappers (which build an undirected CSR for the first two) are not involved."""
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
SELECT count(CREATE_CSR_EDGE({id}, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX({id}, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid))
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst;
"""


def run_sql(sql: str) -> str:
    out = subprocess.run([DUCKDB, "-csv", "-noheader"], input=sql, capture_output=True, text=True)
    if out.returncode != 0 or "Error" in out.stderr:
        raise RuntimeError(out.stderr + out.stdout)
    return out.stdout


def column(part, n, conv, dtype):
    out = np.zeros(n, dtype=dtype)
    seen = 0
    for r in csv.reader(io.StringIO(part)):
        if len(r) == 2:
            out[int(r[0])] = conv(r[1])
            seen += 1
    assert seen == n, (seen, n)
    return out


def save(name, n, src, dst):
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": np.arange(n, dtype=np.int64)}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": src, "dst": dst}), f"{td}/e.parquet")
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
{BUILD.format(id=0)}
{BUILD.format(id=1)}
{BUILD.format(id=2)}
.print ---V
SELECT csrv FROM get_csr_v(0);
.print ---E
SELECT csre FROM get_csr_e(0);
.print ---L
SELECT a.rowid, local_clustering_coefficient(0, a.rowid) FROM v a ORDER BY a.rowid;
.print ---W
SELECT a.rowid, weakly_connected_component(1, a.rowid) FROM v a ORDER BY a.rowid;
.print ---P
SELECT a.rowid, pagerank(2, a.rowid) FROM v a ORDER BY a.rowid;
"""
        txt = run_sql(sql)
    csr_v = np.array([int(x) for x in txt.split("---V\n")[1].split("---E\n")[0].split()], dtype=np.int64)
    csr_e = np.array([int(x) for x in txt.split("---E\n")[1].split("---L\n")[0].split()], dtype=np.int64)
    lcc = column(txt.split("---L\n")[1].split("---W\n")[0], n, np.float32, np.float32)
    wcc = column(txt.split("---W\n")[1].split("---P\n")[0], n, int, np.int64)
    pr = column(txt.split("---P\n")[1], n, float, np.float64)
    out = os.path.join(HERE, f"refn4_{name}.npz")
    np.savez_compressed(out, n=np.int64(n), src=src.astype(np.int32), dst=dst.astype(np.int32),
                        csr_v=csr_v.astype(np.int32), csr_e=csr_e.astype(np.int32), lcc=lcc, wcc=wcc.astype(np.int32),
                        pagerank=pr)
    print(f"{name}: n={n} m={len(src)} components={len(set(wcc.tolist()))} max_lcc={lcc.max():.3f} "
          f"sum_pr={pr.sum():.6f} -> {os.path.getsize(out)} bytes")


def undirected(n, src, dst):
    """both directions of every distinct non-loop edge (what the reference's undirected CSR holds)"""
    keep = src != dst
    a, b = np.minimum(src[keep], dst[keep]), np.maximum(src[keep], dst[keep])
    key = np.unique(a.astype(np.int64) * n + b)
    a, b = key // n, key % n
    return np.concatenate([a, b]), np.concatenate([b, a])


def main():
    # the Student / know graph of test/sql/scalar/local_clustering_coefficient.test, directed as inserted
    save("student_know", 5, [0, 0, 0, 3, 1, 1, 2, 4], [1, 2, 3, 0, 2, 3, 3, 3])
    n, src, dst = datagen.rmat_edges(9)  # directed, duplicates and self-loops kept
    save("rmat9_directed", n, src, dst)
    us, ud = undirected(n, src.astype(np.int64), dst.astype(np.int64))
    save("rmat9_undirected", n, us, ud)
    n, src, dst, _ = datagen.snb_shaped_edges(600, 12.0, seed=4)  # undirected by construction
    save("snb600", n, src, dst)
    rng = np.random.default_rng(11)  # many small components, isolated vertices
    s = rng.integers(0, 300, 260)
    d = np.clip(s + rng.integers(-3, 4, 260), 0, 299)
    us, ud = undirected(300, s, d)
    save("bands300", 300, us, ud)
    # the smallest shapes of tests/test_analytics_boundaries.py that sit on a kernel boundary of csrc/pgq_analytics.cu
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_analytics_boundaries as tab
    for name in tab.GOLDEN_SHAPES:
        save(name, *tab.shape(name))


if __name__ == "__main__":
    main()
