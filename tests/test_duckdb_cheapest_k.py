"""cheapest_k_paths and cheapest_k_costs through the DuckDB shim: raw UDFs over a weighted CSR CTE, as a statement would
call them, in WALK (5 arguments) and with a path mode (a 6th).  The costs must be the oracle's exactly
(oracle/pgq_oracle_cheapest_k.c over the same edges and weights); the lists are compared as paths rather than by
position, since the statement's join decides the CSR's adjacency order and so the order among equal-cost paths: each
listed path must be a path of the mode along the table's edges, with its listed cost, and path 0 must be the
cheapest_path UDF's list.  Skipped where the shim binary has not been built (duckdb_ext/build.sh)."""
import csv
import io
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_cheapest_k as ock

pytestmark = pytest.mark.gpu

B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
needs_shim = pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")

N, M, P, K = 200, 700, 300, 4
MODES = ("WALK", "ACYCLIC", "TRAIL")
CSR_CTE = f"""
WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid, k.w) AS temp
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst)"""
SQL = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT i::BIGINT AS id FROM range(0, {N}) t(i);
CREATE TABLE e AS SELECT (hash(i * 2 + 1) % {N})::BIGINT AS src, (hash(i * 2 + 2) % {N})::BIGINT AS dst,
                         (hash(i * 3 + 7) % 4)::BIGINT AS w FROM range(0, {M}) t(i);
CREATE TABLE p AS SELECT i AS i, CASE WHEN i % 17 = 0 THEN NULL ELSE (hash(i * 7) % {N})::BIGINT END AS src,
                         CASE WHEN i % 19 = 0 THEN NULL WHEN i % 13 = 0 THEN (hash(i * 7) % {N})::BIGINT
                              ELSE (hash(i * 5 + 1) % {N})::BIGINT END AS dst
                  FROM range(0, {P}) t(i);
.print ----EDGES----
SELECT rowid, src, dst, w FROM e ORDER BY rowid;
.print ----PAIRS----
SELECT i, src, dst FROM p ORDER BY i;
.print ----ROWS----
{CSR_CTE}
SELECT p.i, cheapest_k_paths(0, (SELECT count(*) FROM v), p.src, p.dst, {K}) AS walk,
       cheapest_k_costs(0, (SELECT count(*) FROM v), p.src, p.dst, {K}) AS walk_costs,
       cheapest_k_paths(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 'acyclic') AS acyclic,
       cheapest_k_costs(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 'ACYCLIC') AS acyclic_costs,
       cheapest_k_paths(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 'TRAIL') AS trail,
       cheapest_k_costs(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, 'TRAIL') AS trail_costs,
       cheapest_path(0, (SELECT count(*) FROM v), p.src, p.dst) AS path, __x.temp AS z
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


def check_path(path, cost, mode, edge_of):
    """path is [s, e1, v1, ..., t] along the table's edges, admitted by the mode, and its weights sum to cost"""
    verts, eids = path[0::2], path[1::2]
    total = 0
    for a, eid, b in zip(verts, eids, verts[1:]):
        src, dst, w = edge_of[eid]
        assert (src, dst) == (a, b), path
        total += w
    assert total == cost, (path, cost)
    if mode == "ACYCLIC":
        assert len(set(verts)) == len(verts), path
    if mode == "TRAIL":
        assert len(set(eids)) == len(eids), path


@needs_shim
def test_raw_udfs_return_the_oracles_rows():
    out = subprocess.run([B200, "-csv"], input=SQL, capture_output=True, text=True, timeout=600)
    assert "----STATS----" in out.stdout, (out.stdout[-2000:], out.stderr[-2000:])
    edges = np.array([[int(x) for x in r] for r in section(out.stdout, "EDGES")], dtype=np.int64)
    edge_of = {int(r[0]): (int(r[1]), int(r[2]), int(r[3])) for r in edges}
    pairs = [(int(r[0]), opt_int(r[1]), opt_int(r[2])) for r in section(out.stdout, "PAIRS")]
    rows = section(out.stdout, "ROWS")
    assert len(rows) == P
    v, e, ids, w = orc.csr_build_weighted(N, edges[:, 1], edges[:, 2], edges[:, 3], edges[:, 0])
    ps = np.array([0 if s is None else s for _, s, _ in pairs])
    pd = np.array([0 if d is None else d for _, _, d in pairs])
    sv = np.array([s is not None for _, s, _ in pairs], np.uint8)
    dv = np.array([d is not None for _, _, d in pairs], np.uint8)
    listed = 0
    for col, mode in enumerate(MODES):
        _, ocosts, _, _ = ock.cheapest_k_paths(N, v, e, ids, w, ps, pd, K, mode, sv, dv)
        for row, exp in zip(rows, ocosts):
            paths, costs, path = row[1 + 2 * col], row[2 + 2 * col], row[7]
            if exp is None:
                assert paths == "" and costs == "", (mode, row[0])
                continue
            got, got_costs = json.loads(paths), json.loads(costs)
            assert got_costs == exp, (mode, row[0])
            assert len(got) == len(exp) and len(set(map(tuple, got))) == len(got), (mode, row[0])
            for q, c in zip(got, got_costs):
                check_path(q, c, mode, edge_of)
            assert got[0] == json.loads(path), (mode, row[0])  # path 0 is cheapest_path's
            listed += len(got)
    assert listed > 3 * P // 2
    stats = section(out.stdout, "STATS")[0][0]
    assert "cheapest_k_paths_calls=" in stats and "cheapest_k_paths_calls=0" not in stats


@needs_shim
@pytest.mark.parametrize("call,text", [("cheapest_k_paths(0, 1, 0, 0, 0)", "k must be 1 or more"),
                                       ("cheapest_k_costs(0, 1, 0, 0, 2, 'SHORTEST')", "path mode must be")])
def test_binds_check_k_and_mode(call, text):
    out = subprocess.run([B200, "-csv"], input=f"SELECT {call};\n", capture_output=True, text=True, timeout=120)
    assert text in out.stdout + out.stderr
