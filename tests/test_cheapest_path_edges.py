"""cheapest_path_length (csrc/pgq_cheapest.cu) beyond strictly positive weights: negative BIGINT and DOUBLE weights,
zero, infinite and NaN weights, the unreached sentinel max/2 at both types, every batch shape, a lane count shrunk by
the vertex count, shapes that stress the sweep, and concurrent callers.

Every device result is compared bit for bit with the CPU restatement of the reference (oracle/pgq_oracle.c) and,
where the semantics allow it, with an exact reference written here: integer Bellman-Ford in numpy, or scipy's
Dijkstra for weights >= 1.

The reference starts every vertex but the source at max/2 and relaxes from all of them, reached or not.  So for a
BIGINT row (s, t) it ends at  min(dist(s, t), max/2 + h[t])  with  h[t] = min over all u of dist(u, t) <= 0: a target
that only an unreached vertex reaches at a negative cost gets a valid, huge cost, whatever else is in the batch.

No test graph holds a negative cycle, reachable or not: the reference, the restatement and the device would all sweep
about 2^62 times before it stopped improving.  Negative weights only appear on DAGs (every edge runs from a lower to
a higher rank of a random permutation, no self-loops); graphs with cycles carry weights >= 0 only."""
from concurrent.futures import ThreadPoolExecutor
from functools import lru_cache

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc
from test_gpu_csr_weighted import build_chunked

INF_I64 = (2**63 - 1) // 2            # the reference's "unreached" for BIGINT: max / 2
INF_F64 = 1.7976931348623157e308 / 2  # ... and for DOUBLE
NO_PATH = np.iinfo(np.int64).max      # "no path" in the exact references below (never a path cost here)
NEG_NAN = (np.array([np.nan]).view(np.uint64) | np.uint64(1 << 63)).view(np.float64)[0]  # NaN with the sign bit


# ---- graphs ---------------------------------------------------------------------------------------------------------
def random_dag(rng, n, m):
    """m random edges (plus a tenth as parallel twins) oriented from the lower to the higher rank of a random
    permutation, self-loops dropped -> (src, dst, rank)."""
    rank = rng.permutation(n)
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    a, b = a[a != b], b[a != b]
    fwd = rank[a] < rank[b]
    src, dst = np.where(fwd, a, b), np.where(fwd, b, a)
    twin = rng.integers(0, len(src), len(src) // 10)
    return np.concatenate([src, src[twin]]).astype(np.int64), np.concatenate([dst, dst[twin]]).astype(np.int64), rank


def exact_bellman_ford(n, src, dst, w, init):
    """Plain Bellman-Ford in int64 (every sum here stays far from overflow).  init: [k, n] start costs, NO_PATH for
    "no path yet" -> [k, n] least path costs, NO_PATH where there is none."""
    d = np.ascontiguousarray(np.asarray(init, dtype=np.int64).T)  # [n, k]
    w = np.asarray(w, dtype=np.int64)[:, None]
    for _ in range(n + 1):
        du = d[src]
        reached = du != NO_PATH
        cand = np.where(reached, np.where(reached, du, 0) + w, NO_PATH)
        new = d.copy()
        np.minimum.at(new, dst, cand)
        if np.array_equal(new, d):
            return d.T
        d = new
    raise AssertionError("negative cycle")


def exact_from(n, src, dst, w, sources):
    init = np.full((len(sources), n), NO_PATH, dtype=np.int64)
    init[np.arange(len(sources)), sources] = 0
    return exact_bellman_ford(n, src, dst, w, init)


def reference_fixed_point_i64(dist_st, h_t):
    """The reference's BIGINT result for one row, in Python ints: min(dist(s, t), max/2 + h[t]); None = NULL (the value
    is max/2 itself)."""
    v = INF_I64 + int(h_t)
    if dist_st != NO_PATH:
        v = min(v, int(dist_st))
    return None if v == INF_I64 else v


@lru_cache(maxsize=None)
def dag_case(n, m, seed, kind):
    """A random DAG and 600 rows of three kinds, shuffled: t reachable from s; t unreachable from s but reached at a
    negative cost by some other vertex (h[t] < 0); t reached at a negative cost by nothing (h[t] = 0).
    kind "i64": BIGINT weights in [-50, 50], expected = the closed form above.
    kind "dyadic": DOUBLE weights k/1024, |k| < 2^20; every path sum is exact in float64, and max/2 plus such a
    sum rounds back to max/2, so expected = dist(s, t) / 1024, NULL where there is no path."""
    rng = np.random.default_rng(seed)
    src, dst, _ = random_dag(rng, n, m)
    wi = rng.integers(-50, 51, len(src)) if kind == "i64" else rng.integers(-(1 << 20) + 1, 1 << 20, len(src))
    sources = rng.choice(n, size=min(n, 150), replace=False)
    D = exact_from(n, src, dst, wi, sources)
    h = exact_bellman_ford(n, src, dst, wi, np.zeros((1, n), dtype=np.int64))[0]
    p = 600
    j = rng.integers(0, len(sources), p)
    ps, pd, rkind = sources[j], rng.integers(0, n, p), np.zeros(p, dtype=np.int64)
    for i in range(p):
        reach = D[j[i]] != NO_PATH
        for k, cand in enumerate((reach, ~reach & (h < 0), ~reach & (h == 0))):
            if i % 3 == k and cand.any():
                pd[i] = rng.choice(np.flatnonzero(cand))
        rkind[i] = 0 if reach[pd[i]] else (1 if h[pd[i]] < 0 else 2)
    dist = D[j, pd]
    if kind == "i64":
        fp = [reference_fixed_point_i64(dist[i], h[pd[i]]) for i in range(p)]
        exp_valid = np.array([x is not None for x in fp], dtype=np.uint8)
        exp_cost = np.array([0 if x is None else x for x in fp], dtype=np.int64)
        w = wi.astype(np.int64)
    else:
        exp_valid = (dist != NO_PATH).astype(np.uint8)
        exp_cost = np.where(exp_valid == 1, dist, 0) / 1024.0
        w = wi / 1024.0
    return dict(n=n, src=src, dst=dst, w=w, ps=ps, pd=pd, rkind=rkind, exp_cost=exp_cost, exp_valid=exp_valid)


DAGS = [(300, 700, 11), (2000, 3000, 12)]


# ---- comparisons ----------------------------------------------------------------------------------------------------
def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a.astype(np.int64)


def assert_rows(got, exp, what=""):
    """valid equal; costs equal bit for bit on valid rows (a -0.0 is not a +0.0)."""
    (gc, gv), (ec, ev) = got[:2], exp[:2]
    gv, ev = np.asarray(gv), np.asarray(ev)
    bad = np.flatnonzero(gv != ev)
    assert bad.size == 0, f"{what}: NULL-ness differs in {bad.size} rows, e.g. rows {bad[:5].tolist()}: got valid " \
                          f"{gv[bad[:5]].tolist()}, expected {ev[bad[:5]].tolist()}"
    ok = np.flatnonzero(ev == 1)
    bad = ok[bits(np.asarray(gc)[ok]) != bits(np.asarray(ec)[ok])]
    assert bad.size == 0, f"{what}: cost differs in {bad.size} rows, e.g. rows {bad[:5].tolist()}: got " \
                          f"{np.asarray(gc)[bad[:5]].tolist()}, expected {np.asarray(ec)[bad[:5]].tolist()}"


def oracle_rows(n, src, dst, w, ps, pd, sv=None, dv=None):
    v, e, _, ow = orc.csr_build_weighted(n, src, dst, w)
    return orc.cheapest_path_length(n, v, e, ow, ps, pd, sv, dv)


def device_csr(ctx, n, src, dst, w, chunk=997):
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    return build_chunked(ctx, n, src, dst, np.arange(len(src), dtype=np.int64), np.asarray(w), chunk=chunk)


def dijkstra_rows(n, src, dst, w, ps, pd):
    """scipy Dijkstra (weights >= 1; parallel edges reduced to their cheapest first, as scipy would sum them)."""
    o = np.lexsort((w, dst, src))
    s, d, ww = src[o], dst[o], w[o]
    first = np.ones(len(s), dtype=bool)
    first[1:] = (s[1:] != s[:-1]) | (d[1:] != d[:-1])
    A = csr_matrix((ww[first].astype(np.float64), (s[first], d[first])), shape=(n, n))
    cost, valid = np.zeros(len(ps), dtype=np.int64), np.zeros(len(ps), dtype=np.uint8)
    for s0 in np.unique(ps):
        rows = np.flatnonzero(ps == s0)
        dist = dijkstra(A, directed=True, indices=int(s0))[pd[rows]]
        valid[rows] = np.isfinite(dist)
        cost[rows] = np.where(np.isfinite(dist), dist, 0).astype(np.int64)
    return cost, valid


# ---- CPU: the exact references agree with the restatement ---------------------------------------------------------
@pytest.mark.parametrize("n,m,seed", DAGS)
@pytest.mark.parametrize("kind", ["i64", "dyadic"])
def test_exact_references_agree_with_the_oracle(n, m, seed, kind):
    """Pins the restatement's behaviour at negative weights on the CPU: the closed form of the reference's fixed point
    (BIGINT) and exact dyadic sums (DOUBLE)."""
    c = dag_case(n, m, seed, kind)
    for k in range(3):  # every kind of row is there
        assert (c["rkind"] == k).sum() >= 100
    if kind == "i64":  # rows reached only from unreached vertices are valid and huge
        assert c["exp_valid"][c["rkind"] == 1].all() and not c["exp_valid"][c["rkind"] == 2].any()
    assert_rows(oracle_rows(c["n"], c["src"], c["dst"], c["w"], c["ps"], c["pd"]), (c["exp_cost"], c["exp_valid"]),
                "oracle vs exact")


def test_oracle_relaxes_from_unreached_vertices_and_never_through_nan():
    """0 -> 1 (1), 1 -> 2 (-5), vertex 3 isolated: (3, 2) is max/2 - 5 alone and in a batch with (0, 2).
    A weight -1e300 behind an unreached vertex gives max/2 - 1e300; a NaN edge never relaxes, whatever its sign."""
    v, e, _, w = orc.csr_build_weighted(4, [0, 1], [1, 2], np.array([1, -5]))
    assert orc.cheapest_path_length(4, v, e, w, [3], [2])[0].tolist() == [INF_I64 - 5]
    cost, valid = orc.cheapest_path_length(4, v, e, w, [0, 3], [2, 2])
    assert cost.tolist() == [-4, INF_I64 - 5] and valid.tolist() == [1, 1]
    v, e, _, w = orc.csr_build_weighted(4, [0, 1], [1, 2], np.array([1.0, -1e300]))
    cost, valid = orc.cheapest_path_length(4, v, e, w, [3, 0], [2, 2])
    assert valid.tolist() == [1, 1] and cost[0] == INF_F64 - 1e300 and cost[1] == 1.0 - 1e300
    for nan in (np.nan, NEG_NAN):
        v, e, _, w = orc.csr_build_weighted(3, [0, 1], [1, 2], np.array([1.0, nan]))
        assert orc.cheapest_path_length(3, v, e, w, [0], [2])[1].tolist() == [0]


def test_dijkstra_agrees_with_the_oracle_on_a_cyclic_graph():
    rng = np.random.default_rng(21)
    n = 400
    src, dst = datagen.random_graph(n, 1600, seed=22)
    w = rng.integers(1, 1000, len(src))
    ps, pd = rng.integers(0, n, 300), rng.integers(0, n, 300)
    assert_rows(oracle_rows(n, src, dst, w, ps, pd), dijkstra_rows(n, src, dst, w, ps, pd), "oracle vs Dijkstra")


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,m,seed", DAGS)
def test_negative_bigint_dag(gpu_ctx, n, m, seed):
    """Negative BIGINT weights, parallel edges: the closed form of the reference's fixed point and the restatement."""
    c = dag_case(n, m, seed, "i64")
    csr = device_csr(gpu_ctx, c["n"], c["src"], c["dst"], c["w"])
    got = csr.cheapest_path_length(c["ps"], c["pd"])
    csr.free()
    for k, what in enumerate(("reachable from the source", "reached only from unreached vertices", "reached by nothing")):
        sel = c["rkind"] == k
        assert_rows((got[0][sel], got[1][sel]), (c["exp_cost"][sel], c["exp_valid"][sel]), f"device vs closed form, {what}")
    assert_rows(got, oracle_rows(c["n"], c["src"], c["dst"], c["w"], c["ps"], c["pd"]), "device vs oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("n,m,seed", DAGS)
def test_rows_do_not_depend_on_their_batch(gpu_ctx, n, m, seed):
    """A row's result is the same alone (p = 1), after the rows are shuffled, and amid unrelated rows."""
    c = dag_case(n, m, seed, "i64")
    ps, pd = c["ps"], c["pd"]
    csr = device_csr(gpu_ctx, c["n"], c["src"], c["dst"], c["w"])
    full = csr.cheapest_path_length(ps, pd)
    alone_c, alone_v = np.zeros_like(full[0]), np.zeros_like(full[1])
    for i in range(len(ps)):
        cst, vld, st = csr.cheapest_path_length(ps[i:i + 1], pd[i:i + 1])
        alone_c[i], alone_v[i] = cst[0], vld[0]
        assert st["lanes"] == 32 and st["batches"] == 1
    assert_rows((alone_c, alone_v), full, "one row alone vs the full call")
    rng = np.random.default_rng(seed)
    perm = rng.permutation(len(ps))
    sc, sv, _ = csr.cheapest_path_length(ps[perm], pd[perm])
    assert_rows((sc[np.argsort(perm)], sv[np.argsort(perm)]), full, "shuffled rows vs the full call")
    other = rng.integers(0, c["n"], 333)
    mc, mv, _ = csr.cheapest_path_length(np.concatenate([other, ps[:200], other[:100]]),
                                         np.concatenate([rng.integers(0, c["n"], 333), pd[:200], other[:100]]))
    assert_rows((mc[333:533], mv[333:533]), (full[0][:200], full[1][:200]), "rows amid unrelated rows vs the full call")
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("w,expect", [(-5, INF_I64 - 5), (-1e300, INF_F64 - 1e300)])
def test_row_reached_only_from_an_unreached_vertex(gpu_ctx, w, expect):
    """0 -> 1 (1), 1 -> 2 (w), vertex 3 isolated: (3, 2) ends at max/2 + w, alone or batched with (0, 2)."""
    csr = device_csr(gpu_ctx, 4, [0, 1], [1, 2], np.array([1, w]))
    for ps, pd in (([3], [2]), ([0, 3], [2, 2]), ([3, 0], [2, 2])):
        cost, valid, _ = csr.cheapest_path_length(ps, pd)
        assert valid.tolist() == [1, 1][:len(ps)]
        assert cost[ps.index(3)] == expect
        if len(ps) == 2:
            assert cost[ps.index(0)] == 1 + w
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("n,m,seed", DAGS)
def test_dyadic_negative_doubles_are_exact(gpu_ctx, n, m, seed):
    c = dag_case(n, m, seed, "dyadic")
    csr = device_csr(gpu_ctx, c["n"], c["src"], c["dst"], c["w"])
    got = csr.cheapest_path_length(c["ps"], c["pd"])
    csr.free()
    assert_rows(got, (c["exp_cost"], c["exp_valid"]), "device vs exact dyadic sums")
    assert_rows(got, oracle_rows(c["n"], c["src"], c["dst"], c["w"], c["ps"], c["pd"]), "device vs oracle")


@pytest.mark.gpu
def test_mixed_magnitude_doubles_with_cycles(gpu_ctx):
    """Weights 1e16, 1.0, 0.1, 3e-17, 0.0 on a cyclic multigraph with self-loops: sums depend on the order of
    addition, so only the reference's own fixed point matches bit for bit."""
    rng = np.random.default_rng(31)
    n = 500
    src, dst = datagen.random_graph(n, 2500, seed=32)
    w = rng.choice(np.array([1e16, 1.0, 0.1, 3e-17, 0.0]), len(src))
    ps, pd = rng.integers(0, n, 700), rng.integers(0, n, 700)
    csr = device_csr(gpu_ctx, n, src, dst, w)
    got = csr.cheapest_path_length(ps, pd)
    csr.free()
    assert got[1].sum() > 500
    assert_rows(got, oracle_rows(n, src, dst, w, ps, pd), "device vs oracle")


# 0 -(+0.0)-> 1 -(-0.0)-> 2 -(-NaN)-> 8 -(1)-> 11;  0 -(+inf)-> 3 -(1)-> 4;  0 -(-inf)-> 5 -(+inf)-> 6 <-(2)- 0;
# 1 -(+NaN)-> 7 <-(5)- 0;  9 -(-1e300)-> 10;  12 -(-inf)-> 13;  9 and 12 have no in-edges
SPECIAL_F64 = ([0, 1, 2, 8, 0, 3, 0, 5, 0, 1, 0, 9, 12], [1, 2, 8, 11, 3, 4, 5, 6, 6, 7, 7, 10, 13],
               [0.0, -0.0, NEG_NAN, 1.0, np.inf, 1.0, -np.inf, np.inf, 2.0, np.nan, 5.0, -1e300, -np.inf])
# 0 -(0)-> 1 -(0)-> 2;  0 -(max/2)-> 3;  0 -(max/2 - 1)-> 4;  0 -(2^61)-> 5 -(2^61)-> 6;  7 -(max/2)-> 8;  9 -(-3)-> 10
SPECIAL_I64 = ([0, 1, 0, 0, 0, 5, 7, 9], [1, 2, 3, 4, 5, 6, 8, 10],
               [0, 0, INF_I64, INF_I64 - 1, 1 << 61, 1 << 61, INF_I64, -3])


def special_case(case):
    src, dst, w = SPECIAL_F64 if case == "f64" else SPECIAL_I64
    n = max(max(src), max(dst)) + 1
    return n, np.array(src), np.array(dst), np.array(w, dtype=np.float64 if case == "f64" else np.int64)


def test_oracle_special_values():
    """What the reference's comparisons give from vertex 0 on the special-value graphs above."""
    n, src, dst, w = special_case("f64")
    cost, valid = oracle_rows(n, src, dst, w, np.zeros(n, dtype=np.int64), np.arange(n))
    assert valid.tolist() == [1, 1, 1, 0, 0, 1, 1, 1, 0, 0, 1, 0, 0, 1]
    assert bits(cost[:3]).tolist() == [0, 0, 0]                  # +0.0 + -0.0 = +0.0
    assert cost[5] == -np.inf and cost[6] == 2.0 and cost[7] == 5.0  # -inf + inf and +NaN never relax
    assert cost[10] == INF_F64 - 1e300 and cost[13] == -np.inf      # behind unreached vertices
    # +inf never improves on max/2 (3, 4); the -NaN edge never relaxes (8, 11); 9 and 12 are only sources
    n, src, dst, w = special_case("i64")
    cost, valid = oracle_rows(n, src, dst, w, np.zeros(n, dtype=np.int64), np.arange(n))
    assert valid.tolist() == [1, 1, 1, 0, 1, 1, 0, 0, 0, 0, 1]
    assert cost[valid == 1].tolist() == [0, 0, 0, INF_I64 - 1, 1 << 61, INF_I64 - 3]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["f64", "i64"])
def test_special_values(gpu_ctx, case):
    """Signed zeros, infinities, NaNs of either sign, -1e300 and -inf behind unreached vertices (DOUBLE); zero, the
    sentinel max/2 itself, max/2 - 1, and 2^61 + 2^61 >= max/2 (BIGINT): every pair, then every row from vertex 0
    alone, so that no other lane starts at an unreached vertex."""
    n, src, dst, w = special_case(case)
    csr = device_csr(gpu_ctx, n, src, dst, w, chunk=3)
    ps, pd = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    assert_rows(csr.cheapest_path_length(ps, pd), oracle_rows(n, src, dst, w, ps, pd), "every pair")
    for t in range(n):
        assert_rows(csr.cheapest_path_length([0], [t]), oracle_rows(n, src, dst, w, [0], [t]), f"row (0, {t}) alone")
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("p", [1, 31, 32, 33, 255, 256, 257, 700])
@pytest.mark.parametrize("kind", ["i64", "f64"])
def test_batch_shapes(gpu_ctx, p, kind):
    """L = min(256, ceil(p/32)*32) lanes per batch; duplicate sources, src == dst rows, NULL sources and targets with
    out-of-range values under them.  BIGINT: negative weights on a DAG; DOUBLE: a cyclic multigraph, weights >= 0."""
    rng = np.random.default_rng(p * 7 + (kind == "f64"))
    n = 300
    if kind == "i64":
        src, dst, _ = random_dag(rng, n, 800)
        w = rng.integers(-50, 51, len(src))
    else:
        src, dst = datagen.random_graph(n, 1200, seed=p)
        w = rng.random(len(src)) * 10.0
    ps = rng.choice(rng.integers(0, n, max(1, p // 4)), p)  # ~4 rows per source
    pd = rng.integers(0, n, p)
    same = rng.random(p) < 0.1
    pd[same] = ps[same]
    sv, dv = (rng.random(p) > 0.1).astype(np.uint8), (rng.random(p) > 0.1).astype(np.uint8)
    ps[sv == 0] = rng.choice([-7, n, n + 1000], int((sv == 0).sum()))
    pd[dv == 0] = rng.choice([-1, n, 1 << 40], int((dv == 0).sum()))
    csr = device_csr(gpu_ctx, n, src, dst, w)
    cost, valid, st = csr.cheapest_path_length(ps, pd, sv, dv)
    csr.free()
    lanes = min(256, -(-p // 32) * 32)
    assert st["lanes"] == lanes and st["batches"] == -(-p // lanes)
    assert_rows((cost, valid), oracle_rows(n, src, dst, w, ps, pd, sv, dv), "device vs oracle")
    assert not valid[(sv == 0) | (dv == 0)].any()
    assert valid[same & (sv == 1) & (dv == 1)].all() and not cost[same & (sv == 1) & (dv == 1)].any()


@pytest.mark.gpu
@pytest.mark.parametrize("n,lanes", [((1 << 20) + 1, 128), ((1 << 21) + 3, 64)])
def test_lane_count_shrinks_with_n(gpu_ctx, n, lanes):
    """The distance array is kept under 2 GB: more than 2^20 vertices -> 128 lanes, more than 2^21 -> 64.  Two random
    out-edges per vertex (small diameter, few sweeps), weights 1..1000, 200 rows from 16 sources -> several batches;
    against scipy's Dijkstra from those sources (the restatement would need gigabytes here)."""
    rng = np.random.default_rng(n)
    src = np.repeat(np.arange(n, dtype=np.int64), 2)
    dst = rng.integers(0, n, len(src))
    w = rng.integers(1, 1001, len(src))
    ps = rng.choice(rng.choice(n, 16, replace=False), 200)
    pd = rng.integers(0, n, 200)
    csr = device_csr(gpu_ctx, n, src, dst, w, chunk=1 << 20)
    cost, valid, st = csr.cheapest_path_length(ps, pd)
    csr.free()
    assert st["lanes"] == lanes and st["batches"] == -(-200 // lanes)
    exp = dijkstra_rows(n, src, dst, w, ps, pd)
    assert 0 < exp[1].sum() < 200
    assert_rows((cost, valid), exp, "device vs Dijkstra")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["i64", "f64"])
def test_in_hub_star(gpu_ctx, kind):
    """8 roots -> 50 000 spokes -> one hub: every spoke relaxes all 256 lanes into the hub's row at once."""
    rng = np.random.default_rng(41)
    spokes = 50_000
    hub, roots = 0, np.arange(1, 9)
    spoke = np.arange(9, 9 + spokes)
    n = 9 + spokes
    src = np.concatenate([np.repeat(roots, spokes), spoke])
    dst = np.concatenate([np.tile(spoke, len(roots)), np.full(spokes, hub)])
    w = rng.integers(0, 1 << 20, len(src)) if kind == "i64" else rng.random(len(src)) * 100.0
    ps = np.concatenate([rng.choice(roots, 200), rng.choice(spoke, 56)])
    pd = np.where(rng.random(256) < 0.8, hub, rng.integers(0, n, 256))
    csr = device_csr(gpu_ctx, n, src, dst, w, chunk=1 << 16)
    cost, valid, st = csr.cheapest_path_length(ps, pd)
    csr.free()
    assert st["lanes"] == 256 and st["batches"] == 1
    assert valid[pd == hub].all()
    assert_rows((cost, valid), oracle_rows(n, src, dst, w, ps, pd), "device vs oracle")


@pytest.mark.gpu
def test_long_chain_with_shortcuts(gpu_ctx):
    """A 3 000-vertex chain with a few shortcuts and back edges: thousands of dependent relaxations, so many sweeps."""
    rng = np.random.default_rng(51)
    n = 3000
    src = np.concatenate([np.arange(n - 1), rng.integers(0, n, 30)])
    dst = np.concatenate([np.arange(1, n), rng.integers(0, n, 30)])
    w = rng.integers(1, 10, len(src))
    ps = np.concatenate([rng.integers(0, 50, 200), rng.integers(0, n - 500, 56)])
    pd = rng.integers(n - 500, n, 256)
    csr = device_csr(gpu_ctx, n, src, dst, w)
    got = csr.cheapest_path_length(ps, pd)
    csr.free()
    assert got[1].all()
    assert_rows(got, oracle_rows(n, src, dst, w, ps, pd), "device vs oracle")
    assert_rows(got, dijkstra_rows(n, src, dst, w, ps, pd), "device vs Dijkstra")


@pytest.mark.gpu
def test_edgeless_and_isolated(gpu_ctx):
    """A CSR without edges has no weights: the reference's bind refuses it ("Need to initialize CSR before doing
    cheapest path"), and so does the device.  With one zero-weight self-loop among 500 isolated vertices, only
    src == dst rows are valid (cost 0)."""
    csr = device_csr(gpu_ctx, 50, [], [], np.zeros(0, dtype=np.int64))
    with pytest.raises(pgq.PgqError):
        csr.cheapest_path_length([0, 1], [0, 1])
    csr.free()
    rng = np.random.default_rng(61)
    n = 500
    ps, pd = rng.integers(0, n, 300), rng.integers(0, n, 300)
    pd[::3] = ps[::3]
    for w in (np.array([0]), np.array([0.0])):
        csr = device_csr(gpu_ctx, n, [7], [7], w)
        got = csr.cheapest_path_length(ps, pd)
        csr.free()
        assert got[1].tolist() == (ps == pd).astype(np.uint8).tolist()
        assert_rows(got, oracle_rows(n, [7], [7], w, ps, pd), "device vs oracle")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["i64", "f64"])
def test_zero_weight_cycles_and_self_loops(gpu_ctx, kind):
    """Cycles and self-loops of weight 0 (and -0.0 for DOUBLE) improve nothing, so the sweeps stop."""
    rng = np.random.default_rng(71)
    n = 400
    src, dst = datagen.random_graph(n, 1600, seed=72)
    ring = np.arange(0, 40)
    src = np.concatenate([src, ring, ring])
    dst = np.concatenate([dst, np.roll(ring, -1), ring])  # a 40-cycle and 40 self-loops
    if kind == "i64":
        w = np.where(rng.random(len(src)) < 0.5, 0, rng.integers(1, 20, len(src)))
        w[-80:] = 0
    else:
        w = np.where(rng.random(len(src)) < 0.5, rng.choice(np.array([0.0, -0.0]), len(src)), rng.random(len(src)))
        w[-80:] = rng.choice(np.array([0.0, -0.0]), 80)
    ps, pd = rng.integers(0, n, 500), rng.integers(0, n, 500)
    csr = device_csr(gpu_ctx, n, src, dst, w)
    got = csr.cheapest_path_length(ps, pd)
    csr.free()
    assert_rows(got, oracle_rows(n, src, dst, w, ps, pd), "device vs oracle")


@pytest.mark.gpu
def test_concurrent_callers(gpu_ctx):
    """Eight threads call cheapest_path_length at once, as DuckDB's workers do: on a BIGINT DAG with negative weights
    and on a DOUBLE graph with cycles, each thread its own rows; every result equals the restatement's."""
    c = dag_case(*DAGS[1], "i64")
    rng = np.random.default_rng(81)
    n2 = 1000
    src2, dst2 = datagen.random_graph(n2, 5000, seed=82)
    w2 = rng.random(len(src2)) * 5.0
    graphs = [(c["n"], c["src"], c["dst"], c["w"]), (n2, src2, dst2, w2)]
    csrs = [device_csr(gpu_ctx, *g) for g in graphs]
    jobs = []
    for t in range(8):
        n = graphs[t % 2][0]
        p = int(rng.integers(100, 700))
        jobs.append((t % 2, rng.integers(0, n, p), rng.integers(0, n, p)))
    expected = [oracle_rows(*graphs[g], ps, pd) for g, ps, pd in jobs]

    def run(job):
        g, ps, pd = job
        return [csrs[g].cheapest_path_length(ps, pd) for _ in range(3)]

    with ThreadPoolExecutor(max_workers=8) as pool:
        results = list(pool.map(run, jobs))
    for t, (res, exp) in enumerate(zip(results, expected)):
        for r in res:
            assert_rows(r, exp, f"thread {t}")
    for csr in csrs:
        csr.free()
