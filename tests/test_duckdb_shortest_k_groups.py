"""shortest_k_groups and shortest_k_groups_count through the DuckDB shim: raw UDFs over the CSR CTE, as a statement
would call them (the MATCH rewriter stays the reference's, which rejects SHORTEST k GROUP).  The rows must be the
oracle's (oracle/pgq_oracle_kgroups.c over the same edges): the same NULLs and, with max_paths = 0, the same paths as a
set (their order within a length follows the CSR's adjacency order, which the statement's join decides); the counts
must be the oracle's.  The 6- and 7-argument overloads are both called, the binds must reject non-constant or invalid
arguments, and the stats must count the calls.  Skipped where the shim binary has not been built (duckdb_ext/build.sh)."""
import csv
import io
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_kgroups as okg

pytestmark = pytest.mark.gpu

B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
needs_shim = pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")

N, M, P, K = 200, 500, 300, 2
SETUP = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT i::BIGINT AS id FROM range(0, {N}) t(i);
CREATE TABLE e AS SELECT (hash(i * 2 + 1) % {N})::BIGINT AS src, (hash(i * 2 + 2) % {N})::BIGINT AS dst FROM range(0, {M}) t(i);
CREATE TABLE p AS SELECT i AS i, CASE WHEN i % 17 = 0 THEN NULL ELSE (hash(i * 7) % {N})::BIGINT END AS src,
                         CASE WHEN i % 19 = 0 THEN NULL WHEN i % 13 = 0 THEN (hash(i * 7) % {N})::BIGINT
                              ELSE (hash(i * 5 + 1) % {N})::BIGINT END AS dst
                  FROM range(0, {P}) t(i);
"""
CTE = """WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid) AS temp
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst)"""
SQL = SETUP + f"""
.print ----EDGES----
SELECT rowid, src, dst FROM e ORDER BY rowid;
.print ----PAIRS----
SELECT i, src, dst FROM p ORDER BY i;
.print ----ROWS----
{CTE}
SELECT p.i, shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 0) AS walks,
       shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 0, 'Acyclic') AS paths,
       shortest_k_groups_count(0, (SELECT count(*) FROM v), p.src, p.dst, {K}) AS n
FROM p, (SELECT count(cte1.temp) * 0 AS temp FROM cte1) __x ORDER BY p.i;
.print ----STATS----
SELECT duckpgq_b200_stats();
"""


def section(text, name):
    body = text.split(f"----{name}----\n")[1].split("----")[0]
    return list(csv.reader(io.StringIO(body)))[1:]  # (the header)


def is_null(x):  # (the CLI's CSV writes NULL as an empty field or as NULL, by version)
    return x in ("", "NULL")


def opt_int(x):
    return None if is_null(x) else int(x)


@needs_shim
def test_raw_group_udfs_return_the_oracles_rows():
    out = subprocess.run([B200, "-csv"], input=SQL, capture_output=True, text=True, timeout=600)
    assert "----STATS----" in out.stdout, (out.stdout[-2000:], out.stderr[-2000:])
    edges = np.array([[int(x) for x in r] for r in section(out.stdout, "EDGES")], dtype=np.int64)
    pairs = [(int(r[0]), opt_int(r[1]), opt_int(r[2])) for r in section(out.stdout, "PAIRS")]
    rows = section(out.stdout, "ROWS")
    assert len(rows) == P
    v, e, ids = orc.csr_build(N, edges[:, 1], edges[:, 2], edges[:, 0])
    ps = np.array([0 if s is None else s for _, s, _ in pairs])
    pd = np.array([0 if d is None else d for _, _, d in pairs])
    sv = np.array([s is not None for _, s, _ in pairs], np.uint8)
    dv = np.array([d is not None for _, _, d in pairs], np.uint8)
    owalks, orows, _ = okg.shortest_k_groups(N, v, e, ids, ps, pd, K, 0, "WALK", sv, dv)
    opaths, _, _ = okg.shortest_k_groups(N, v, e, ids, ps, pd, K, 0, "ACYCLIC", sv, dv)
    for (i, walks, paths, n), ew, ep, cnt, ok in zip(rows, owalks, opaths, orows["count"], orows["valid"]):
        for got, exp in ((walks, ew), (paths, ep)):
            if exp is None:
                assert is_null(got), i
            else:
                assert sorted(map(tuple, json.loads(got))) == sorted(map(tuple, exp)), i
        assert opt_int(n) == (int(cnt) if ok else None), i
    stats = section(out.stdout, "STATS")[0][0]
    assert "shortest_k_groups_calls=0" not in stats and "shortest_k_groups_calls=" in stats
    assert "shortest_k_groups_count_calls=0" not in stats and "shortest_k_groups_count_calls=" in stats


@needs_shim
@pytest.mark.parametrize("call, text", [
    ("shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, 0, 5)", "k must be 1 or more"),
    ("shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, 2, p.i)", "max_paths must be constant"),
    ("shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, 2, -1)", "max_paths must be 0"),
    ("shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, 2, 5, 'any')", "the path mode must be WALK"),
    ("shortest_k_groups(0, (SELECT count(*) FROM v), p.src, p.dst, 2, 5, CAST(p.i AS VARCHAR))",
     "the path mode must be constant"),
    ("shortest_k_groups_count(0, (SELECT count(*) FROM v), p.src, p.dst, p.i)", "k must be constant"),
])
def test_constant_argument_errors(call, text):
    sql = SETUP + f"{CTE}\nSELECT {call} FROM p, (SELECT count(cte1.temp) * 0 AS temp FROM cte1) __x;\n"
    out = subprocess.run([B200, "-csv"], input=sql, capture_output=True, text=True, timeout=600)
    assert text in out.stdout + out.stderr
