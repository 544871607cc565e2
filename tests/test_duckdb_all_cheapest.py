"""cheapest_path_count and all_cheapest_paths through the DuckDB shim: raw UDFs over the weighted CSR CTE, as a
statement would call them.  The rows must be the oracle's (oracle/pgq_oracle_allcheapest.c over the same edges and
weights): the counts exactly, the lists as a set (their order follows the CSR's adjacency order, which the statement's
join decides), and path 0 must be the cheapest_path UDF's list.  Skipped where the shim binary has not been built
(duckdb_ext/build.sh)."""
import csv
import io
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allcheapest as oac

pytestmark = pytest.mark.gpu

B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
needs_shim = pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")

N, M, P = 300, 1200, 600
SQL = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT i::BIGINT AS id FROM range(0, {N}) t(i);
CREATE TABLE e AS SELECT (hash(i * 2 + 1) % {N})::BIGINT AS src, (hash(i * 2 + 2) % {N})::BIGINT AS dst,
                         (1 + hash(i * 3 + 7) % 3)::BIGINT AS w FROM range(0, {M}) t(i);
CREATE TABLE p AS SELECT i AS i, CASE WHEN i % 17 = 0 THEN NULL ELSE (hash(i * 7) % {N})::BIGINT END AS src,
                         CASE WHEN i % 19 = 0 THEN NULL WHEN i % 13 = 0 THEN (hash(i * 7) % {N})::BIGINT
                              ELSE (hash(i * 5 + 1) % {N})::BIGINT END AS dst
                  FROM range(0, {P}) t(i);
.print ----EDGES----
SELECT rowid, src, dst, w FROM e ORDER BY rowid;
.print ----PAIRS----
SELECT i, src, dst FROM p ORDER BY i;
.print ----ROWS----
WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid, k.w) AS temp
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst)
SELECT p.i, cheapest_path_count(0, (SELECT count(*) FROM v), p.src, p.dst) + __x.temp AS cnt,
       all_cheapest_paths(0, (SELECT count(*) FROM v), p.src, p.dst, 0) AS paths,
       cheapest_path(0, (SELECT count(*) FROM v), p.src, p.dst) AS path
FROM p, (SELECT count(cte1.temp) * 0 AS temp FROM cte1) __x ORDER BY p.i;
.print ----STATS----
SELECT duckpgq_b200_stats();
"""


def section(text, name):
    body = text.split(f"----{name}----\n")[1].split("----")[0]
    rows = list(csv.reader(io.StringIO(body)))
    return rows[1:]  # (the header)


def opt_int(x):
    return None if x == "" else int(x)


@needs_shim
def test_raw_udfs_return_the_oracles_rows():
    out = subprocess.run([B200, "-csv"], input=SQL, capture_output=True, text=True, timeout=600)
    assert "----STATS----" in out.stdout, (out.stdout[-2000:], out.stderr[-2000:])
    edges = np.array([[int(x) for x in r] for r in section(out.stdout, "EDGES")], dtype=np.int64)
    pairs = [(int(r[0]), opt_int(r[1]), opt_int(r[2])) for r in section(out.stdout, "PAIRS")]
    rows = section(out.stdout, "ROWS")
    assert len(rows) == P
    v, e, ids, w = orc.csr_build_weighted(N, edges[:, 1], edges[:, 2], edges[:, 3], edges[:, 0])
    ps = np.array([0 if s is None else s for _, s, _ in pairs])
    pd = np.array([0 if d is None else d for _, _, d in pairs])
    sv = np.array([s is not None for _, s, _ in pairs], np.uint8)
    dv = np.array([d is not None for _, _, d in pairs], np.uint8)
    opaths, ocnt, _ = oac.all_cheapest_paths(N, v, e, ids, w, ps, pd, 0, sv, dv)
    assert sum(x is not None and len(x) > 1 for x in opaths) > 10  # rows with several cheapest paths
    for (i, cnt, paths, path), exp, ec in zip(rows, opaths, ocnt):
        if exp is None:
            assert cnt == "" and paths == "" and path == "", i
            continue
        got = json.loads(paths)
        assert int(cnt) == ec == len(got), i
        assert sorted(map(tuple, got)) == sorted(map(tuple, exp)), i
        assert got[0] == json.loads(path), i
    stats = section(out.stdout, "STATS")[0][0]
    assert "cheapest_path_count_calls=" in stats and "all_cheapest_paths_calls=" in stats
    assert "cheapest_path_count_calls=0" not in stats and "all_cheapest_paths_calls=0" not in stats
