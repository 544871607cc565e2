"""shortest_k_paths' 6-argument overload (a VARCHAR path mode) through the DuckDB shim: a raw UDF over the CSR CTE, as
a statement would call it (the MATCH rewriter stays the reference's, which rejects every path mode but WALK).  The rows
must be the oracle's (oracle/pgq_oracle_kpaths_modes.c over the same edges): the same NULLs and the same path lengths;
the paths of every length before the last as a set, and those of the last length as paths of the mode in the graph
(which paths of a length come first follows the CSR's adjacency order, which the statement's join decides).  Path 0
must be the shortestpath UDF's list, and the stats must count the calls.  Skipped where the shim binary has not been
built (duckdb_ext/build.sh)."""
import csv
import io
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_kpaths_modes as okm

pytestmark = pytest.mark.gpu

B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
needs_shim = pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")

N, M, P, K = 200, 500, 400, 6
MODE = "trail"
SQL = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT i::BIGINT AS id FROM range(0, {N}) t(i);
CREATE TABLE e AS SELECT (hash(i * 2 + 1) % {N})::BIGINT AS src, (hash(i * 2 + 2) % {N})::BIGINT AS dst FROM range(0, {M}) t(i);
CREATE TABLE p AS SELECT i AS i, CASE WHEN i % 17 = 0 THEN NULL ELSE (hash(i * 7) % {N})::BIGINT END AS src,
                         CASE WHEN i % 19 = 0 THEN NULL WHEN i % 13 = 0 THEN (hash(i * 7) % {N})::BIGINT
                              ELSE (hash(i * 5 + 1) % {N})::BIGINT END AS dst
                  FROM range(0, {P}) t(i);
.print ----EDGES----
SELECT rowid, src, dst FROM e ORDER BY rowid;
.print ----PAIRS----
SELECT i, src, dst FROM p ORDER BY i;
.print ----ROWS----
WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM v a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM v a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.src) AS cnt FROM v a LEFT JOIN e k ON k.src = a.id
                     GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst),
         a.rowid, c.rowid, k.rowid) AS temp
  FROM e k JOIN v a ON a.id = k.src JOIN v c ON c.id = k.dst)
SELECT p.i, shortest_k_paths(0, (SELECT count(*) FROM v), p.src, p.dst, {K}, '{MODE}') AS walks,
       shortestpath(0, (SELECT count(*) FROM v), p.src, p.dst) AS path
FROM p, (SELECT count(cte1.temp) * 0 AS temp FROM cte1) __x ORDER BY p.i;
.print ----STATS----
SELECT duckpgq_b200_stats();
"""


def section(text, name):
    body = text.split(f"----{name}----\n")[1].split("----")[0]
    return list(csv.reader(io.StringIO(body)))[1:]  # (the header)


def opt_int(x):
    return None if x == "" else int(x)


@needs_shim
def test_raw_mode_udf_returns_the_oracles_rows():
    out = subprocess.run([B200, "-csv"], input=SQL, capture_output=True, text=True, timeout=600)
    assert "----STATS----" in out.stdout, (out.stdout[-2000:], out.stderr[-2000:])
    edges = np.array([[int(x) for x in r] for r in section(out.stdout, "EDGES")], dtype=np.int64)
    ends = {int(r[0]): (int(r[1]), int(r[2])) for r in edges}
    pairs = [(int(r[0]), opt_int(r[1]), opt_int(r[2])) for r in section(out.stdout, "PAIRS")]
    rows = section(out.stdout, "ROWS")
    assert len(rows) == P
    v, e, ids = orc.csr_build(N, edges[:, 1], edges[:, 2], edges[:, 0])
    ps = np.array([0 if s is None else s for _, s, _ in pairs])
    pd = np.array([0 if d is None else d for _, _, d in pairs])
    sv = np.array([s is not None for _, s, _ in pairs], np.uint8)
    dv = np.array([d is not None for _, _, d in pairs], np.uint8)
    opaths, _, _ = okm.shortest_k_paths_mode(N, v, e, ids, ps, pd, K, MODE, sv, dv)
    for (i, walks, path), exp in zip(rows, opaths):
        if exp is None:
            assert walks == "", i
            continue
        got = json.loads(walks)
        lens = [(len(w) - 1) // 2 for w in got]
        assert lens == [(len(w) - 1) // 2 for w in exp], i
        last = lens[-1]
        assert sorted(tuple(w) for w in got if len(w) < 2 * last + 1) == \
            sorted(tuple(w) for w in exp if len(w) < 2 * last + 1), i
        for w in got:  # a trail of the graph from src to dst
            assert w[0] == ps[int(i)] and w[-1] == pd[int(i)] and len(set(w[1::2])) == len(w[1::2])
            assert all(ends[w[j]] == (w[j - 1], w[j + 1]) for j in range(1, len(w), 2)), i
        assert got[0] == json.loads(path), i
    stats = section(out.stdout, "STATS")[0][0]
    assert "shortest_k_paths_mode_calls=" in stats and "shortest_k_paths_mode_calls=0" not in stats
    assert "shortest_k_paths_calls=0" in stats
