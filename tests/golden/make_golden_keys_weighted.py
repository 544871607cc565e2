#!/usr/bin/env python
"""Golden vectors for the weighted CSR built from key columns (pgq_csr_build_keys_weighted), produced by the UNMODIFIED
reference (oracle/_ref/duckdb, threads = 1) with the directed CSR CTE of make_golden_keys.py and k.w as the last
argument of create_csr_edge (its 8-argument overloads, csr_creation.cpp:141-198,227-235).  Run in the build container
only:

    python tests/golden/make_golden_keys_weighted.py

Writes tests/golden/refkw_<name>.npz:
    vkey                  the vertex table's key column v.id (rowid = position, never NULL: see make_golden_keys.py)
    src, dst, src_valid, dst_valid    the edge table's key columns e.src / e.dst (rowid = position, 0 = NULL)
    w, w_valid            the edge table's weight column e.w, BIGINT (int64) or DOUBLE (float64), 0 = NULL
    w_type                csr_get_w_type(0)
    csr_v, csr_e, csr_w   get_csr_v(0) / get_csr_e(0) / get_csr_w(0); within a vertex the order is DuckDB's join order
    psrc, pdst            vertex rowid pairs (never NULL)
    cost, cost_valid      cheapest_path_length(0, n, psrc, pdst)
The script refuses what the reference cannot build well: a NULL weight on an edge that joins (the reference skips its
row and leaves a malformed CSR), a NULL vertex key, and an edge table that joins to no row (no CSR at all).  Negative
weights only enter where they close no cycle: the reference's Bellman-Ford loops until nothing changes."""
import csv
import io
import os
import sys
import tempfile

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_next4 import BUILD, datagen, run_sql  # noqa: E402

BUILD_W = BUILD.replace("a.rowid, c.rowid, k.rowid))", "a.rowid, c.rowid, k.rowid, k.w))")
assert BUILD_W != BUILD
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def save(name, vkey, src, dst, w, rng, src_valid=None, dst_valid=None, w_valid=None, pairs=300):
    vkey, src, dst = (np.asarray(x, dtype=np.int64) for x in (vkey, src, dst))
    w = np.asarray(w)
    is_f = w.dtype.kind == "f"
    w = w.astype(np.float64 if is_f else np.int64)
    n, m = vkey.shape[0], src.shape[0]
    sv = np.ones(m, dtype=np.uint8) if src_valid is None else np.asarray(src_valid, dtype=np.uint8)
    dv = np.ones(m, dtype=np.uint8) if dst_valid is None else np.asarray(dst_valid, dtype=np.uint8)
    wv = np.ones(m, dtype=np.uint8) if w_valid is None else np.asarray(w_valid, dtype=np.uint8)
    joins = (sv == 1) & np.isin(src, vkey)
    if np.any(joins & (wv == 0)):
        raise ValueError(f"{name}: a NULL weight on an edge that joins leaves the reference's CSR malformed")
    if not np.any(joins & (dv == 1) & np.isin(dst, vkey)):
        raise ValueError(f"{name}: an edge table that joins to no row gives the reference no CSR")
    psrc, pdst = rng.integers(0, n, pairs), rng.integers(0, n, pairs)
    with tempfile.TemporaryDirectory() as td:
        pq.write_table(pa.table({"id": pa.array(vkey, type=pa.int64())}), f"{td}/v.parquet")
        pq.write_table(pa.table({"src": pa.array(src, type=pa.int64(), mask=sv == 0),
                                 "dst": pa.array(dst, type=pa.int64(), mask=dv == 0),
                                 "w": pa.array(w, type=pa.float64() if is_f else pa.int64(), mask=wv == 0)}),
                       f"{td}/e.parquet")
        pq.write_table(pa.table({"i": np.arange(pairs, dtype=np.int64), "src": psrc, "dst": pdst}), f"{td}/p.parquet")
        sql = f"""
SET threads TO 1;
CREATE TABLE v AS SELECT * FROM read_parquet('{td}/v.parquet');
CREATE TABLE e AS SELECT * FROM read_parquet('{td}/e.parquet');
CREATE TABLE p AS SELECT * FROM read_parquet('{td}/p.parquet');
{BUILD_W.format(id=0)}
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
"""
        txt = run_sql(sql)
    w_type = int(txt.split("---T\n")[1].split("---V\n")[0].strip())
    csr_v = np.array([int(x) for x in txt.split("---V\n")[1].split("---E\n")[0].split()], dtype=np.int64)
    csr_e = np.array([int(x) for x in txt.split("---E\n")[1].split("---W\n")[0].split()], dtype=np.int64)
    wpart = txt.split("---W\n")[1].split("---C\n")[0].split()
    csr_w = np.array([float(x) if is_f else int(x) for x in wpart], dtype=np.float64 if is_f else np.int64)
    cost = np.zeros(pairs, dtype=np.float64 if is_f else np.int64)
    cvalid = np.zeros(pairs, dtype=np.uint8)
    for r in csv.reader(io.StringIO(txt.split("---C\n")[1])):
        if r[1] not in ("", "NULL"):
            cost[int(r[0])] = float(r[1]) if is_f else int(r[1])
            cvalid[int(r[0])] = 1
    out = os.path.join(HERE, f"refkw_{name}.npz")
    np.savez_compressed(out, vkey=vkey, src=src, dst=dst, src_valid=sv, dst_valid=dv, w=w, w_valid=wv,
                        w_type=np.int64(w_type), csr_v=csr_v, csr_e=csr_e, csr_w=csr_w, psrc=psrc, pdst=pdst,
                        cost=cost, cost_valid=cvalid)
    print(f"{name}: n={n} m={m} w_type={w_type} rows={csr_e.shape[0]} reachable={int(cvalid.sum())} "
          f"-> {os.path.getsize(out)} bytes")


def main():
    rng = np.random.default_rng(4242)
    # keys = a shuffled range, BIGINT weights; the last 12 vertex rows are sinks, and only edges into a sink carry the
    # int64 extremes and the negative weights (no cycle runs through them)
    n, m = 300, 1500
    keys = rng.permutation(n) + 1000
    inner, sinks = keys[:-12], keys[-12:]
    src, dst = rng.choice(inner, m), rng.choice(inner, m)
    w = rng.integers(1, 1000, m)
    ext = rng.choice(m, 12, replace=False)
    dst[ext] = sinks
    w[ext] = [I64_MAX, I64_MIN, I64_MAX - 1, I64_MIN + 1, 0, -1, I64_MAX, -7, I64_MIN, 2**62, -(2**62), 1]
    save("perm300_extremes_i64", keys, src, dst, w, rng)
    # the same vertex keys, DOUBLE weights in (0, 100] with -0.0 and NaNs anywhere and negatives into the sinks
    src, dst = rng.choice(inner, m), rng.choice(inner, m)
    w = rng.random(m) * 100.0 + 1e-3
    w[rng.choice(m, 20, replace=False)] = -0.0
    w[rng.choice(m, 5, replace=False)] = np.nan
    ext = rng.choice(m, 6, replace=False)
    dst[ext] = sinks[:6]
    w[ext] = [-2.5, -1e300, -0.0, np.nan, -np.inf, 0.0]
    save("perm300_specials_f64", keys, src, dst, w, rng)
    # duplicated source keys: vertex rows 0..39 hold keys 0..19 twice, rows 40..59 hold 100..119; destinations use
    # only those unique keys, which are never sources (no cycle), so every edge becomes two rows of the same weight
    keys = np.concatenate([np.arange(20), rng.permutation(20), 100 + np.arange(20)])
    src, dst = rng.choice(keys[:40], 400), 100 + rng.integers(0, 20, 400)
    save("dupsrc60_i64", keys, src, dst, rng.integers(-50, 51, 400), rng)
    w = rng.integers(-(1 << 20), 1 << 20, 400) / 1024.0
    w[:3] = [-0.0, np.nan, -3.75]
    save("dupsrc60_f64", keys, rng.choice(keys[:40], 400), 100 + rng.integers(0, 20, 400), w, rng)
    # NULL keys on either end and dangling rows that join nothing; the edges that join nothing may carry NULL weights
    n, m = 200, 1200
    keys = rng.permutation(n) * 3
    for kind in ("i64", "f64"):
        src, dst = rng.choice(keys, m), rng.choice(keys, m)
        src_valid = (rng.random(m) > 0.15).astype(np.uint8)
        src[rng.random(m) < 0.1] = 1  # no vertex has key 1 (all keys are multiples of 3)
        dst_valid = np.where(src_valid == 0, rng.random(m) > 0.5, 1).astype(np.uint8)
        dst[(src == 1) & (rng.random(m) < 0.5)] = 2
        joins = (src_valid == 1) & (src != 1)
        w_valid = np.where(joins, 1, rng.random(m) > 0.5).astype(np.uint8)
        if kind == "i64":
            w = rng.integers(0, 60, m)
        else:
            w = rng.random(m) * 8.0
            w[rng.choice(np.flatnonzero(joins), 8, replace=False)] = -0.0
            w[rng.choice(np.flatnonzero(joins), 2, replace=False)] = np.nan
        save(f"nulls200_{kind}", keys, src, dst, w, rng, src_valid, dst_valid, w_valid)
    # an R-MAT graph (duplicates and self-loops kept) under a random sparse relabelling, DOUBLE weights
    n, s, d = datagen.rmat_edges(9)
    keys = rng.choice(np.arange(-(2**40), 2**40, 104729), n, replace=False)
    save("rmat9_relabelled_f64", keys, keys[s], keys[d], rng.random(len(s)) * 10.0 + 1e-3, rng, pairs=400)


if __name__ == "__main__":
    main()
