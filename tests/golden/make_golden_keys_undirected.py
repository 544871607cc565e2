#!/usr/bin/env python
"""Golden vectors for the undirected CSR built from key columns (pgq_csr_build_keys_undirected), produced by the
UNMODIFIED reference (oracle/_ref/duckdb, threads = 1) with the undirected CSR CTE the reference emits
(CreateUndirectedCSRCTE, compressed_sparse_row.cpp:125-130,145-172,192-223) over tables v(id) and e(src, dst).  Run
in the build container only:

    python tests/golden/make_golden_keys_undirected.py

Writes tests/golden/refu_<name>.npz:
    vkey                  the vertex table's key column v.id (rowid = position)
    src, dst, src_valid, dst_valid    the edge table's key columns e.src / e.dst (rowid = position, 0 = NULL)
    constraint            1 if the reference raised the ConstraintException of csr_creation.cpp:121-125
    ill_formed            1 if it did not, but scattered out of place: a row's offsets decrease, or a row differs from
                          its SQL neighbour set (some row's pair count differs from its degree)
    csr_v, csr_e          get_csr_v(0) / get_csr_e(0) (pgq_scan.cpp:84-111) when it did not raise; get_csr_e returns
                          the 2R entries e is sized by, of which the first R are kept (the rest are checked to be 0)
The vertex keys are never NULL (see make_golden_keys.py)."""
import os
import sys
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_next4 import datagen, run_sql  # noqa: E402

CONSTRAINT_TEXT = "Non-existent/non-unique vertices detected"
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max

# the statement the reference's MATCH rewriter builds for an undirected edge, with v = source = destination table
BUILD = """
WITH edges_cte AS (SELECT src_table.rowid AS src, dst_table.rowid AS dst, e.rowid AS edges
                   FROM e INNER JOIN v src_table ON e.src = src_table.id INNER JOIN v dst_table ON e.dst = dst_table.id),
csr_cte AS (
SELECT create_csr_edge(0, (SELECT count(v.id) FROM v v),
    CAST((SELECT multiply(2, sum(create_csr_vertex(0, (SELECT count(v.id) FROM v v), sub.dense_id, sub.cnt)))
          FROM (SELECT dense_id, count(outgoing_edges) AS cnt FROM (
                SELECT v.rowid AS dense_id, e.src AS outgoing_edges, e.dst AS incoming_edges FROM e INNER JOIN v ON e.src = v.id
                UNION BY NAME
                SELECT v.rowid AS dense_id, e.dst AS outgoing_edges, e.src AS incoming_edges FROM e INNER JOIN v ON e.dst = v.id
                ) unique_edges GROUP BY dense_id) sub) AS BIGINT),
    (SELECT multiply(2, count()) FROM (SELECT src, dst FROM edges_cte UNION BY NAME SELECT dst AS src, src AS dst FROM edges_cte)),
    src, dst, edge) AS temp
FROM (SELECT src, dst, any_value(edges) AS edge FROM (
      SELECT src, dst, edges FROM edges_cte UNION ALL SELECT dst, src, edges FROM edges_cte) GROUP BY src, dst))
SELECT count(temp) FROM csr_cte;
"""


def sql_neighbours(vkey, src, dst, sv, dv):
    """row p -> sorted distinct rows q of edges_cte UNION ALL its reverse"""
    out = [set() for _ in range(len(vkey))]
    for k in range(len(src)):
        if sv[k] and dv[k]:
            for a in np.nonzero(vkey == src[k])[0]:
                for c in np.nonzero(vkey == dst[k])[0]:
                    out[a].add(int(c))
                    out[c].add(int(a))
    return [sorted(x) for x in out]


def save(name, vkey, src, dst, src_valid=None, dst_valid=None):
    vkey, src, dst = (np.asarray(x, dtype=np.int64) for x in (vkey, src, dst))
    m = src.shape[0]
    sv = np.ones(m, dtype=np.uint8) if src_valid is None else np.asarray(src_valid, dtype=np.uint8)
    dv = np.ones(m, dtype=np.uint8) if dst_valid is None else np.asarray(dst_valid, dtype=np.uint8)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": pa.array(vkey, type=pa.int64())}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": pa.array(src, type=pa.int64(), mask=sv == 0),
                                 "dst": pa.array(dst, type=pa.int64(), mask=dv == 0)}), f"{td}/e.parquet")
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
{BUILD}
.print ---V
SELECT csrv FROM get_csr_v(0);
.print ---E
SELECT csre FROM get_csr_e(0);
"""
        try:
            txt = run_sql(sql)
            constraint = 0
        except RuntimeError as ex:
            if CONSTRAINT_TEXT not in str(ex):
                raise
            constraint = 1
    ill_formed = 0
    if constraint:
        csr_v = csr_e = np.zeros(0, dtype=np.int64)
    else:
        csr_v = np.array([int(x) for x in txt.split("---V\n")[1].split("---E\n")[0].split()], dtype=np.int64)
        csr_e = np.array([int(x) for x in txt.split("---E\n")[1].split()], dtype=np.int64)
        n = vkey.shape[0]
        want = sql_neighbours(vkey, src, dst, sv, dv)
        r = sum(len(x) for x in want)
        assert csr_v.shape[0] == n + 2 and csr_e.shape[0] == 2 * r, (csr_v.shape, csr_e.shape)
        assert not csr_e[r:].any()
        csr_e = csr_e[:r]
        ill_formed = int(bool(np.any(np.diff(csr_v[:n + 1]) < 0)) or csr_v[n] != r or
                         [sorted(csr_e[csr_v[i]:csr_v[i + 1]].tolist()) for i in range(n)] != want)
    out = os.path.join(HERE, f"refu_{name}.npz")
    np.savez_compressed(out, vkey=vkey, src=src, dst=dst, src_valid=sv, dst_valid=dv, constraint=np.int64(constraint),
                        ill_formed=np.int64(ill_formed), csr_v=csr_v, csr_e=csr_e)
    print(f"{name}: n={vkey.shape[0]} m={m} constraint={constraint} ill_formed={ill_formed} rows={csr_e.shape[0]} "
          f"-> {os.path.getsize(out)} bytes")


def main():
    rng = np.random.default_rng(2025)
    # shuffled keys; parallel, reciprocal and self-loop edges
    n = 400
    keys = rng.permutation(n)
    src, dst = rng.choice(keys, 1500), rng.choice(keys, 1500)
    src = np.concatenate([src, src[:200], dst[200:400], keys[:50]])
    dst = np.concatenate([dst, dst[:200], src[200:400], keys[:50]])
    save("shuffled400", keys, src, dst)
    # sparse keys of both signs, and the int64 extremes
    keys = rng.choice(np.arange(-10**12, 10**12, 7919), 300, replace=False)
    save("sparse_signed300", keys, rng.choice(keys, 1200), rng.choice(keys, 1200))
    keys = np.array([I64_MAX, 0, I64_MIN, -1, I64_MAX - 1, 1, I64_MIN + 1, 42, -42, 2**32, -(2**32)], dtype=np.int64)
    save("extremes11", keys, rng.choice(keys, 100), rng.choice(keys, 100))
    # self-loops alone (some repeated)
    keys = rng.permutation(30) * 2
    loops = rng.choice(keys, 40)
    save("self_loops", keys, loops, loops)
    # NULL and unmatched ends of both kinds: each adds to its key's degree and not to R, so the reference refuses
    keys = np.concatenate([np.arange(10), [3, 7]])
    save("null_and_unmatched_ends", keys, [3, 1, 7, 2, 100, 5], [4, 2, 50, 1, 6, 8], [1, 1, 1, 1, 1, 1],
         [1, 1, 1, 1, 1, 1])
    keys = np.arange(20)
    m = 200
    src, dst = rng.choice(keys, m), rng.choice(keys, m)
    sv, dv = (rng.random(m) > 0.1).astype(np.uint8), (rng.random(m) > 0.1).astype(np.uint8)
    src[rng.random(m) < 0.05] = 99
    dst[rng.random(m) < 0.05] = -99
    save("nulls_and_unmatched_random", keys, src, dst, sv, dv)
    # a dangling destination; a duplicated key
    keys = np.arange(30)
    src, dst = rng.choice(keys, 60), rng.choice(keys, 60)
    dst[17] = 1000
    save("dangling_dst", keys, src, dst)
    keys = np.concatenate([np.arange(30), [4]])
    src, dst = rng.choice(np.arange(5, 30), 60), rng.choice(np.arange(5, 30), 60)
    dst[9] = 4
    save("duplicate_key", keys, src, dst)
    # the two balanced examples: well-formed, and ill-formed (S = R, R(row 2) = 2 != cnt = 1)
    save("balanced_well_formed", [1, 1, 2], [1, 2], [2, 9])
    save("balanced_ill_formed", [1, 1, 2, 3], [1, 3], [2, 9])
    save("null_end_balanced", [1, 1, 2], [1, 2], [2, 0], None, [1, 0])  # key 2's NULL end balances its second row
    # the Student / know graph of test/sql/path_finding/undirected_paths.test (Student ids 0..4, know pairs as inserted)
    save("student_know", [0, 1, 2, 3, 4], [0, 0, 0, 3, 1, 1, 2, 4, 2], [1, 2, 3, 0, 2, 3, 3, 3, 4])
    # R-MAT-9 under a sparse relabelling (duplicates and self-loops kept); an SNB-shaped graph
    n, s, d = datagen.rmat_edges(9)
    keys = rng.choice(np.arange(-(2**40), 2**40, 104729), n, replace=False)
    save("rmat9_relabelled", keys, keys[s], keys[d])
    n, s, d, _ = datagen.snb_shaped_edges(600, 12.0, seed=5)
    keys = rng.permutation(n).astype(np.int64) * 11 + 933
    save("snb600", keys, keys[s], keys[d])


if __name__ == "__main__":
    main()
