"""reachability through the DuckDB surface on SNB0.003, run by the shim binary (duckdb_ext/build/duckdb_b200) with the
host CSR left empty (PGQ_B200_HOST_CSR unset = skip).  It must be served from the device CSR -- its call counter grows
and no host CSR is materialised -- and, where the reference binary (oracle/_ref/duckdb) is present, return its rows for
both traversals.  (Both binaries read the key columns byte by byte, DESIGN §3; the Person rowids are < 256, so every
byte is a vertex id, and without NULLs there is no batch restart.)  Skipped where the shim binary was not built (it
needs the reference's DuckDB sources)."""
import os
import re
import subprocess

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "duckdb")
B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
SUITE = os.path.join(ROOT, "tests", "golden", "sqllogic")  # data/SNB0.003 is relative to it

CSR = """
SET threads TO 1;
import database 'data/SNB0.003';
CREATE TABLE pairs AS SELECT a.rowid * 1000 + b.rowid AS i, a.rowid AS s, b.rowid AS d FROM Person a, Person b
  WHERE (a.rowid + 3 * b.rowid) % 2 = 0;
CREATE TABLE csr_done AS WITH cte1 AS (
  SELECT CREATE_CSR_EDGE(0, (SELECT count(a.id) FROM Person a),
         CAST((SELECT sum(CREATE_CSR_VERTEX(0, (SELECT count(a.id) FROM Person a), sub.dense_id, sub.cnt))
               FROM (SELECT a.rowid AS dense_id, count(k.Person1Id) AS cnt FROM Person a
                     LEFT JOIN Person_knows_person k ON k.Person1Id = a.id GROUP BY a.rowid) sub) AS BIGINT),
         (SELECT count(*) FROM Person_knows_person k JOIN Person a ON a.id = k.Person1Id
                                                     JOIN Person c ON c.id = k.Person2Id),
         a.rowid, c.rowid, k.rowid) AS temp
  FROM Person_knows_person k JOIN Person a ON a.id = k.Person1Id JOIN Person c ON c.id = k.Person2Id)
SELECT count(cte1.temp) AS c FROM cte1;
.print ---
SELECT i, reachability(0, false, (SELECT count(*) FROM Person), s, d),
          reachability(0, true, (SELECT count(*) FROM Person), s, d) FROM pairs ORDER BY i;
.print ---
"""


def run(binary, sql):
    env = dict(os.environ)
    env.pop("PGQ_B200_HOST_CSR", None)
    env["LD_LIBRARY_PATH"] = os.path.dirname(binary) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([binary, "-csv"], input=sql, capture_output=True, text=True, timeout=600, cwd=SUITE, env=env)
    assert "Error" not in out.stderr, out.stderr
    return out.stdout


@pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")
def test_reachability_runs_on_the_device_csr():
    parts = run(B200, CSR + "SELECT duckpgq_b200_stats();\n").split("---\n")
    assert len(parts) == 3
    rows = parts[1].strip().splitlines()
    assert len(rows) > 1000
    assert {r.split(",")[1] for r in rows[1:]} == {"true", "false"}
    assert all(r.split(",")[1] == r.split(",")[2] for r in rows[1:])  # is_variant changes nothing here
    stats = dict(re.findall(r"(\w+)=(\d+)", parts[2]))
    assert stats["host_csr_materialisations"] == "0", parts[2]
    assert int(stats["reachability_calls"]) > 0, parts[2]
    if os.path.exists(REF):
        assert parts[:2] == run(REF, CSR).split("---\n")[:2]
