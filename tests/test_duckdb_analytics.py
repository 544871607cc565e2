"""pagerank, weakly_connected_component and local_clustering_coefficient through the DuckDB surface: the reference's
table functions (which expand to SQL calling the scalar functions by name) on SNB0.003, run by the shim binary
(duckdb_ext/build/duckdb_b200).  The shim must serve the scalar functions from the device CSR -- its call counters
grow and no host CSR is materialised -- and, where the reference binary (oracle/_ref/duckdb) is present, return
the same rows.  Skipped where the shim binary was not built (it needs the reference's DuckDB sources)."""
import os
import re
import subprocess

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "duckdb")
B200 = os.path.join(ROOT, "duckpgq_extension_b200", "duckdb_ext", "build", "duckdb_b200")
SUITE = os.path.join(ROOT, "tests", "golden", "sqllogic")  # data/SNB0.003 is relative to it

SETUP = """
import database 'data/SNB0.003';
CREATE PROPERTY GRAPH snb VERTEX TABLES (Person LABEL Person)
  EDGE TABLES (Person_knows_person SOURCE KEY (Person1Id) REFERENCES Person (id)
               DESTINATION KEY (Person2Id) REFERENCES Person (id) LABEL Knows);
"""

QUERIES = [
    "SELECT * FROM pagerank('snb', 'Person', 'Knows') ORDER BY 1;",
    "SELECT * FROM weakly_connected_component('snb', 'Person', 'Knows') ORDER BY 1;",
    "SELECT * FROM local_clustering_coefficient('snb', 'Person', 'Knows') ORDER BY 1;",
]


def run(binary, sql):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = os.path.dirname(binary) + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    out = subprocess.run([binary, "-csv"], input=sql, capture_output=True, text=True, timeout=600, cwd=SUITE, env=env)
    assert "Error" not in out.stderr, out.stderr
    return out.stdout


@pytest.mark.skipif(not os.path.exists(B200), reason="shim DuckDB binary not built")
def test_table_functions_run_on_the_device_csr():
    marker = "---"
    sql = SETUP + "".join(q + f"\n.print {marker}\n" for q in QUERIES) + "SELECT duckpgq_b200_stats();\n"
    parts = run(B200, sql).split(marker + "\n")
    assert len(parts) == len(QUERIES) + 1
    for rows in parts[:-1]:
        assert len(rows.strip().splitlines()) > 10  # a header and one row per person
    stats = dict(re.findall(r"(\w+)=(\d+)", parts[-1]))
    assert stats["host_csr_materialisations"] == "0"
    for name in ("pagerank_calls", "weakly_connected_component_calls", "local_clustering_coefficient_calls"):
        assert int(stats[name]) > 0, parts[-1]
    if os.path.exists(REF):
        expect = run(REF, SETUP + "".join(q + f"\n.print {marker}\n" for q in QUERIES)).split(marker + "\n")
        assert parts[:-1] == expect[:-1]  # DuckDB prints the shortest exact text of a DOUBLE / FLOAT

