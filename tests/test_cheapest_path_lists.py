"""cheapest_path: the cheapest path itself as shortestpath's list [s, e1, v1, ..., ek, t], with shortestpath's tie-break
over the edges the final Bellman-Ford distances make tight (include/duckpgq_b200.h, pgq_cheapest_path).

The CPU tests pin the oracle (oracle/pgq_oracle_cheapest.c, orc_cheapest_path_*: a sequential BFS over the tight edges that keeps
the first parent written) against independent checks: the edges of every path exist in order, its weights sum left to
right to the cost of orc_cheapest_path_length bit for bit, and, for integer weights >= 0, its hop count and every step
of its tie-break agree with a restatement built on scipy's Dijkstra and, on graphs of at most 7 vertices, on all simple
paths.  They also prove that each case of the catalogue below reaches what it is named after.  The GPU tests require
the device's lists, validity and tight-search counters to equal the oracle's at the device's lane count.
"""
import itertools
import pathlib
import threading

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

from duckpgq_extension_b200 import datagen, pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_INVALID_ARG, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_RANGE
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_cheapest as orc_cp

PGQ_ERR_UNSUPPORTED = 8
INF_I64 = (2**63 - 1) // 2
MAX_LEVEL = 65534  # h is uint16 on the device, 0xFFFF meaning "not reached"


# ---- graphs and the independent checks ------------------------------------------------------------------------------
def weighted_csr(n, src, dst, w, eid=None):
    """-> (v, e, edge_ids, w) in the reference's CSR order (unique edge ids: the CSR position of the input edge)"""
    return orc.csr_build_weighted(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w), eid)


def lanes_for(n, p):
    """run_bf's lane count: as many as a 2 GB distance array allows, at most 256, rounded up to the rows' multiple of 32"""
    L = 256
    while L > 32 and L * max(n, 1) * 8 > (2 << 30):
        L >>= 1
    return min(L, -(-p // 32) * 32)


def wrap_sum(ws, is_f):
    """left-to-right sum from 0 in the weight type's arithmetic (int64 wraps, doubles round to nearest)"""
    if is_f:
        acc = 0.0
        for x in ws:
            acc = acc + float(x)
        return acc
    acc = 0
    for x in ws:
        acc = (acc + int(x) + 2**63) % 2**64 - 2**63
    return acc


def same_value(a, b, is_f):
    if is_f:
        return np.float64(a).tobytes() == np.float64(b).tobytes()
    return int(a) == int(b)


def path_weights(v, e, ids, w, path):
    """the weights along a path, checking that each (a, edge id, b) step is an edge a -> b of the CSR with that id"""
    pos_of = {int(i): k for k, i in enumerate(ids)}
    out = []
    for j in range(0, len(path) - 1, 2):
        a, eid, b = path[j], path[j + 1], path[j + 2]
        k = pos_of[eid]
        assert v[a] <= k < v[a + 1] and e[k] == b, f"step {a} -[{eid}]-> {b} is not an edge"
        out.append(w[k])
    return out


def check_paths(n, v, e, ids, w, src, dst, sv, dv, paths):
    """The independent checks every oracle result passes; -> the rows' costs and validity (orc_cheapest_path_length)."""
    is_f = w.dtype.kind == "f"
    cost, cvalid = orc.cheapest_path_length(n, v, e, w, src, dst, sv, dv)
    ok_s = np.ones(len(src), np.uint8) if sv is None else np.asarray(sv, np.uint8)
    dss, dsv = orc.cheapest_path_length(n, v, e, w, src, src, ok_s, None)  # d(s)
    for i, path in enumerate(paths):
        if path is None:
            continue
        assert cvalid[i], f"row {i}: a path where the cost is NULL"
        assert path[0] == src[i] and path[-1] == dst[i] and len(path) % 2 == 1
        ws = path_weights(v, e, ids, w, path)
        if dsv[i] and same_value(dss[i], 0, is_f) and not (is_f and np.signbit(dss[i])):
            assert same_value(wrap_sum(ws, is_f), cost[i], is_f), f"row {i}: {ws} does not sum to {cost[i]}"
    return cost, cvalid


def restated_paths(n, src, dst, w, ps, pd):
    """For integer weights >= 0: the path by the semantics, restated on scipy's Dijkstra -- d, the tight edges, BFS
    depths h over them, then the walk back choosing the smallest parent one level up and its first tight position."""
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    rows = np.repeat(np.arange(n), np.diff(v[: n + 1]))
    out = []
    cache = {}
    for s, t in zip(ps, pd):
        s, t = int(s), int(t)
        if s not in cache:
            best = {}
            for k in range(len(e)):  # parallel edges: the cheapest one carries the distance
                key = (rows[k], e[k])
                best[key] = min(best.get(key, np.inf), ww[k])
            if best:
                kk = np.array(list(best.keys()))
                mat = csr_matrix((np.array(list(best.values()), float) + 0.0, (kk[:, 0], kk[:, 1])), shape=(n, n))
                mat.data[mat.data == 0] = 1e-300  # keep zero-weight edges as edges (1e-300 vanishes in the integer sums)
                d = dijkstra(mat, indices=s)
            else:
                d = np.full(n, np.inf)
                d[s] = 0
            d = np.where(np.isinf(d), np.inf, np.round(d))
            tight = np.isfinite(d[rows]) & (d[rows] + ww == d[e])
            h = np.full(n, -1)
            h[s] = 0
            front, k = [s], 0
            while front:
                nxt = set()
                for x in front:
                    for pos in range(v[x], v[x + 1]):
                        if tight[pos] and h[e[pos]] == -1:
                            nxt.add(int(e[pos]))
                for y in nxt:
                    h[y] = k + 1
                front, k = sorted(nxt), k + 1
            cache[s] = (d, tight, h)
        d, tight, h = cache[s]
        if s == t:
            out.append([s])
            continue
        if h[t] < 0:
            out.append(None)
            continue
        path, u = [t], t
        while u != s:
            par = min(x for x in range(n) if h[x] == h[u] - 1 and any(tight[q] and e[q] == u for q in range(v[x], v[x + 1])))
            q = next(q for q in range(v[par], v[par + 1]) if tight[q] and e[q] == u)
            path += [int(ids[q]), par]
            u = par
        out.append(path[::-1])
    return out


def random_multigraph(rng, n, m, kind):
    """m random edges with parallel twins of other weights, self-loops and zero-weight cycles"""
    a, b = rng.integers(0, n, m), rng.integers(0, n, m)
    twin = rng.integers(0, m, m // 4)
    loops = rng.integers(0, n, max(1, n // 8))
    cyc = rng.choice(n, size=min(n, 3), replace=False)
    src = np.concatenate([a, a[twin], loops, cyc])
    dst = np.concatenate([b, b[twin], loops, np.roll(cyc, 1)])
    if kind == "i64":
        w = rng.integers(0, 20, len(src))
        w[-len(cyc):] = 0
    else:
        w = rng.integers(0, 64, len(src)) / 8.0
        w[-len(cyc):] = 0.0
    return src.astype(np.int64), dst.astype(np.int64), w


# ---- the catalogue --------------------------------------------------------------------------------------------------
def internal_order(n, src, dst):
    """the device's vertex numbering (DESIGN section 2): class (out and in, in only, out only, isolated), then
    descending out-degree (descending in-degree for in-only vertices), stable"""
    outd, ind = np.bincount(src, minlength=n), np.bincount(dst, minlength=n)
    cls = np.where(outd > 0, np.where(ind > 0, 0, 2), np.where(ind > 0, 1, 3))
    deg = np.where(cls == 1, ind, outd)
    return sorted(range(n), key=lambda x: (cls[x], -deg[x]))


def case_hub_ties():
    """0 -> parents 1..8 (1) -> hub 9 (1); parent i has i more edges into sinks, so the device numbers the parents in
    descending degree, opposite to their ids.  Every parent is tight: the smallest id, 1, must win."""
    src, dst = [], []
    for i in range(1, 9):
        src += [0, i]
        dst += [i, 9]
    w = [1] * len(src)
    sink = 10
    for i in range(1, 9):
        for _ in range(i):
            src.append(i)
            dst.append(sink)
            w.append(5)
            sink += 1
    return dict(n=sink, src=src, dst=dst, w=np.array(w), ps=[0, 0, 1], pd=[9, 9, 9])


def case_parallel_first_not_tight():
    """0 -> 1 three times, weights 5, 2, 2: the first position is not tight, the second is"""
    return dict(n=3, src=[0, 0, 0, 1], dst=[1, 1, 1, 2], w=np.array([5, 2, 2, 1]), ps=[0, 0], pd=[1, 2])


def case_valid_cost_null_path():
    """test_cheapest_path_edges' unreached-vertex case: 0 -> 1 (1), 1 -> 2 (-5), 3 isolated: (3, 2) has the valid cost
    max/2 - 5 but no path"""
    return dict(n=4, src=[0, 1], dst=[1, 2], w=np.array([1, -5]), ps=[3, 0, 3, 0], pd=[2, 2, 3, 3])


def case_specials_f64():
    """-inf, NaN and -0.0 against 0.0 (DOUBLE): 0 -> 1 NaN then 3.0 (the NaN edge is tight for nothing); 1 -> 2 -0.0
    then 0.0 (both tight by value, the first wins); 2 -> 3 -inf; 3 -> 4 1.0; and 6 -> 5 -inf with 6 unreached, so that
    d(5) = -inf from the start and (5, x) rows have d(s) != 0"""
    src = [0, 0, 1, 1, 2, 3, 6, 5]
    dst = [1, 1, 2, 2, 3, 4, 5, 4]
    w = np.array([np.nan, 3.0, -0.0, 0.0, -np.inf, 1.0, -np.inf, 2.0])
    return dict(n=7, src=src, dst=dst, w=w, ps=[0, 0, 0, 0, 5, 5, 2], pd=[1, 2, 3, 4, 4, 5, 4])


def case_chain(hops, shortcuts=True):
    """a chain 0 -> 1 -> ... of `hops` edges of weight 1, with heavier shortcuts every 7 vertices"""
    n = hops + 1
    src, dst, w = list(range(hops)), list(range(1, n)), [1] * hops
    if shortcuts:
        for a in range(0, hops - 7, 7):
            src.append(a)
            dst.append(a + 7)
            w.append(8)
    return dict(n=n, src=src, dst=dst, w=np.array(w), ps=[0, 0, 5], pd=[hops, hops // 2, hops])


def case_rows(p, seed=5):
    rng = np.random.default_rng(seed)
    n = 60
    src, dst, w = random_multigraph(rng, n, 240, "i64")
    ps, pd = rng.integers(0, n, p), rng.integers(0, n, p)
    sv = (rng.random(p) > 0.1).astype(np.uint8)
    dv = (rng.random(p) > 0.1).astype(np.uint8)
    return dict(n=n, src=src, dst=dst, w=w, ps=ps, pd=pd, sv=sv, dv=dv)


def case_edgeless():
    """5 vertices, no edges; and 6 vertices with only 0 -> 1, so 2..5 are isolated"""
    return dict(n=6, src=[0], dst=[1], w=np.array([4]), ps=[0, 0, 2, 3, 1, 4], pd=[1, 0, 2, 4, 0, 5])


def case_all_null(which):
    c = case_rows(40, seed=9)
    z = np.zeros(40, np.uint8)
    if which in ("src", "both"):
        c["sv"] = z
    if which in ("dst", "both"):
        c["dv"] = z
    return c


CATALOGUE = {
    "hub_ties": case_hub_ties,
    "parallel_first_not_tight": case_parallel_first_not_tight,
    "valid_cost_null_path": case_valid_cost_null_path,
    "specials_f64": case_specials_f64,
    "chain_300": lambda: case_chain(300),
    "edgeless_and_isolated": case_edgeless,
    "all_null_src": lambda: case_all_null("src"),
    "all_null_dst": lambda: case_all_null("dst"),
    "all_null_both": lambda: case_all_null("both"),
    **{f"rows_{p}": (lambda p=p: case_rows(p)) for p in (1, 31, 32, 33, 255, 256, 257, 513)},
}


def run_oracle(c, lanes=None):
    v, e, ids, w = weighted_csr(c["n"], c["src"], c["dst"], c["w"])
    p = len(c["ps"])
    lanes = lanes or lanes_for(c["n"], p)
    paths, st = orc_cp.cheapest_path(c["n"], v, e, ids, w, c["ps"], c["pd"], c.get("sv"), c.get("dv"), lanes)
    return (v, e, ids, w), paths, st


# ---- CPU: the oracle against the independent checks -----------------------------------------------------------------
@pytest.mark.parametrize("kind", ["i64", "f64"])
@pytest.mark.parametrize("seed", range(6))
def test_oracle_paths_are_cheapest_on_random_multigraphs(kind, seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(8, 40))
    src, dst, w = random_multigraph(rng, n, 4 * n, kind)
    p = 150
    ps, pd = rng.integers(0, n, p), rng.integers(0, n, p)
    sv = (rng.random(p) > 0.05).astype(np.uint8)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    paths, _ = orc_cp.cheapest_path(n, v, e, ids, ww, ps, pd, sv, None, 64)
    cost, cvalid = check_paths(n, v, e, ids, ww, ps, pd, sv, None, paths)
    assert [p_ is not None for p_ in paths] == [bool(x) for x in cvalid]  # weights >= 0: a valid cost has a path
    if kind == "i64":
        exp = restated_paths(n, src, dst, w, ps, pd)
        for i in range(p):
            assert paths[i] == (exp[i] if sv[i] else None), f"row {i}"


@pytest.mark.parametrize("seed", range(12))
def test_oracle_against_all_simple_paths(seed):
    """n <= 7: the least cost over all simple paths, the fewest edges among those, and the tie-break step by step"""
    rng = np.random.default_rng(200 + seed)
    n = int(rng.integers(2, 8))
    src, dst, w = random_multigraph(rng, n, 3 * n, "i64")
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    ps, pd = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    paths, _ = orc_cp.cheapest_path(n, v, e, ids, ww, ps, pd, None, None, 64)
    check_paths(n, v, e, ids, ww, ps, pd, None, None, paths)
    for s, t, path in zip(ps, pd, paths):
        best = None  # (cost, hops) over simple edge sequences
        for k in range(0, n):
            for mid in itertools.permutations([x for x in range(n) if x not in (s, t)], k):
                verts = [s, *mid, t] if s != t else [s]
                if s != t and len(set(verts)) < len(verts):
                    continue
                c = 0
                for a, b in zip(verts, verts[1:]):
                    ws_ = [ww[q] for q in range(v[a], v[a + 1]) if e[q] == b]
                    if not ws_:
                        c = None
                        break
                    c += min(ws_)
                if c is not None and (best is None or (c, len(verts) - 1) < best):
                    best = (c, len(verts) - 1)
            if s == t:
                break
        if best is None:
            assert path is None
            continue
        assert path is not None and sum(path_weights(v, e, ids, ww, path)) == best[0] and (len(path) - 1) // 2 == best[1]
    assert paths == restated_paths(n, src, dst, w, ps, pd)


GOLDEN = pathlib.Path(__file__).parent / "golden"
REFW = sorted(f.name for f in GOLDEN.glob("refw_*.npz"))


def golden_case(name):
    """a refw golden as a case: its edges fed in the reference binary's CSR order (edge id = CSR position), so that
    the CSR built from them is the reference's, adjacency order included"""
    z = np.load(GOLDEN / name)
    n = int(z["n"])
    cv = z["csr_v"].astype(np.int64)
    src = np.repeat(np.arange(n), np.diff(cv[: n + 1]))
    return z, dict(n=n, src=src, dst=z["csr_e"].astype(np.int64), w=z["csr_w"], ps=z["psrc"].astype(np.int64),
                   pd=z["pdst"].astype(np.int64), dv=z["pdst_valid"])


@pytest.mark.parametrize("name", REFW)
def test_oracle_paths_sum_to_the_reference_costs(name):
    """Every non-NULL path sums to the reference binary's cost; a NULL path only where the cost is NULL or t is not
    reached over tight edges (then the cost is the sentinel's)."""
    z, c = golden_case(name)
    n = c["n"]
    v, e, ids, ww = weighted_csr(n, c["src"], c["dst"], c["w"])
    assert np.array_equal(v[: len(z["csr_v"])], z["csr_v"]) and np.array_equal(ww, z["csr_w"])
    ps, pd, dv = c["ps"], c["pd"], c["dv"]
    paths, _ = orc_cp.cheapest_path(n, v, e, ids, ww, ps, pd, None, dv, 256)
    is_f = ww.dtype.kind == "f"
    dss, _ = orc.cheapest_path_length(n, v, e, ww, ps, ps)
    for i, path in enumerate(paths):
        if path is None:
            if z["cost_valid"][i]:  # (then t is not reached over tight edges and the cost is the sentinel's)
                big = abs(float(z["cost"][i])) > 1e18 if not is_f else abs(float(z["cost"][i])) > 1e290 or np.isinf(z["cost"][i])
                assert big, f"row {i}: NULL path at an ordinary cost {z['cost'][i]}"
            continue
        assert z["cost_valid"][i]
        if same_value(dss[i], 0, is_f):
            assert same_value(wrap_sum(path_weights(v, e, ids, ww, path), is_f), z["cost"][i], is_f), f"row {i}"


# ---- CPU: each catalogue case reaches what it is named after --------------------------------------------------------
def test_catalogue_hub_ties_disagree_with_the_internal_order():
    c = case_hub_ties()
    order = internal_order(c["n"], np.array(c["src"]), np.array(c["dst"]))
    parents = [x for x in order if 1 <= x <= 8]
    assert parents[0] == 8 and parents == sorted(parents, reverse=True)
    (_, e, ids, _), paths, _ = run_oracle(c)
    assert paths[0] == [0, 0, 1, 1, 9]  # edge ids: 0 -> 1 is input edge 0, 1 -> 9 input edge 1


def test_catalogue_parallel_edge_first_position_not_tight():
    c = case_parallel_first_not_tight()
    (v, e, ids, w), paths, _ = run_oracle(c)
    assert list(w[v[0]:v[1]]) == [5, 2, 2] and paths[0] == [0, int(ids[v[0] + 1]), 1]


def test_catalogue_valid_cost_null_path():
    c = case_valid_cost_null_path()
    (v, e, ids, w), paths, _ = run_oracle(c)
    cost, cvalid = orc.cheapest_path_length(c["n"], v, e, w, c["ps"], c["pd"])
    assert cvalid.tolist() == [1, 1, 1, 0] and cost[0] == INF_I64 - 5  # (3, 2): valid, huge, and no path
    assert paths == [None, [0, 0, 1, 1, 2], [3], None]


def test_catalogue_specials():
    c = case_specials_f64()
    (v, e, ids, w), paths, _ = run_oracle(c)
    assert np.isnan(w[0]) and np.signbit(w[2]) and not np.signbit(w[3]) and w[2] == w[3]
    assert paths[0] == [0, 1, 1]                     # the NaN edge (id 0) is not tight, the 3.0 edge is
    assert paths[1] == [0, 1, 1, 2, 2]                # -0.0 (id 2) and 0.0 (id 3) are both tight: the first wins
    assert paths[3] == [0, 1, 1, 2, 2, 4, 3, 5, 4]    # through -inf
    cost, cvalid = orc.cheapest_path_length(c["n"], v, e, w, c["ps"], c["pd"])
    assert cost[3] == -np.inf
    ds, _ = orc.cheapest_path_length(c["n"], v, e, w, [5], [5])
    assert ds[0] == -np.inf                           # d(s) != 0 for the rows from 5
    assert paths[5] == [5] and paths[4] is not None


def test_catalogue_long_chains():
    c = case_chain(300)
    _, paths, st = run_oracle(c)
    assert (len(paths[0]) - 1) // 2 == 300 > 256 and st.levels == 300
    c = case_chain(MAX_LEVEL + 1, shortcuts=False)
    c["ps"], c["pd"] = [0], [MAX_LEVEL + 1]
    with pytest.raises(orc.OracleError) as ex:
        run_oracle(c)
    assert ex.value.code == orc_cp.ERR_UNSUPPORTED
    c["pd"] = [MAX_LEVEL]
    _, paths, _ = run_oracle(c)
    assert (len(paths[0]) - 1) // 2 == MAX_LEVEL


@pytest.mark.parametrize("p", [1, 31, 32, 33, 255, 256, 257, 513])
def test_catalogue_row_counts(p):
    L = lanes_for(60, p)
    _, paths, st = run_oracle(case_rows(p))
    assert L == min(256, -(-p // 32) * 32) and st.batches == -(-p // L)
    assert sum(x is not None and len(x) > 1 for x in paths) > 0


def test_catalogue_lane_count_shrinks():
    assert lanes_for((1 << 20) + 1, 300) == 128 and lanes_for((1 << 21) + 3, 300) == 64 and lanes_for(1 << 20, 300) == 256


def test_catalogue_edgeless_and_all_null():
    _, paths, st = run_oracle(case_edgeless())
    assert paths == [[0, 0, 1], [0], [2], None, None, None] and st.edges_traversed == 1
    (v, e, ids, w), paths, _ = run_oracle(dict(n=5, src=[], dst=[], w=np.array([], np.int64), ps=[0, 1, 2], pd=[0, 2, 2]))
    assert paths == [[0], None, [2]]
    for which in ("src", "dst", "both"):
        _, paths, st = run_oracle(case_all_null(which))
        assert all(x is None for x in paths)
        assert st.levels == 0


# ---- GPU: the device against the oracle ---------------------------------------------------------------------------
def device_csr(ctx, n, src, dst, w, chunk=None):
    src, dst, w = np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w)
    m = len(src)
    csr = pgq.DeviceCSR.create(ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n) if m else np.zeros(n, np.int64))
    step = chunk or max(m, 1)
    for o in range(0, m, step):
        csr.add_edges(m, m, src[o:o + step], dst[o:o + step], np.arange(o, min(o + step, m)), w[o:o + step])
    csr.finalize()
    return csr


def compare_with_oracle(ctx, c, chunk=None):
    csr = device_csr(ctx, c["n"], c["src"], c["dst"], c["w"], chunk)
    paths, st = csr.cheapest_path(c["ps"], c["pd"], c.get("sv"), c.get("dv"))
    cost, cvalid, cst = csr.cheapest_path_length(c["ps"], c["pd"], c.get("sv"), c.get("dv"))
    csr.free()
    (v, e, ids, w), opaths, ost = run_oracle(c, st["lanes"])
    assert paths == opaths
    assert (st["push_levels"], st["frontier_vertices"], st["edges_traversed"]) == (ost.levels, ost.frontier_vertices,
                                                                                    ost.edges_traversed)
    assert (st["batches"], st["lanes"]) == (cst["batches"], cst["lanes"]) == (ost.batches, lanes_for(c["n"], len(c["ps"])))
    ocost, ocvalid = orc.cheapest_path_length(c["n"], v, e, w, c["ps"], c["pd"], c.get("sv"), c.get("dv"))
    assert np.array_equal(cvalid, ocvalid)
    assert all(cvalid[i] for i, x in enumerate(paths) if x is not None)  # the cost's validity covers the path's
    check_paths(c["n"], v, e, ids, w, np.asarray(c["ps"]), np.asarray(c["pd"]), c.get("sv"), c.get("dv"), paths)
    return paths, st


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    compare_with_oracle(gpu_ctx, CATALOGUE[name]())


@pytest.mark.gpu
@pytest.mark.parametrize("name", REFW)
def test_device_reference_graphs(gpu_ctx, name):
    _, c = golden_case(name)
    paths, _ = compare_with_oracle(gpu_ctx, c)
    assert any(x is not None and len(x) > 1 for x in paths)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [14, 16])
@pytest.mark.parametrize("kind", ["i64", "f64"])
def test_device_rmat(gpu_ctx, scale, kind):
    n, src, dst = datagen.rmat_edges(scale)
    rng = np.random.default_rng(scale)
    w = rng.integers(1, 100, len(src)) if kind == "i64" else rng.integers(1, 1 << 20, len(src)) / 1024.0
    ps, pd = datagen.hashed_pairs(64, n)
    paths, st = compare_with_oracle(gpu_ctx, dict(n=n, src=src, dst=dst, w=w, ps=ps, pd=pd), chunk=1 << 16)
    assert st["push_levels"] > 3 and sum(x is not None for x in paths) > 16


@pytest.mark.gpu
def test_device_depth_limit(gpu_ctx):
    c = case_chain(MAX_LEVEL + 1, shortcuts=False)
    csr = device_csr(gpu_ctx, c["n"], c["src"], c["dst"], c["w"])
    paths, st = csr.cheapest_path([0], [MAX_LEVEL])
    assert (len(paths[0]) - 1) // 2 == MAX_LEVEL and st["push_levels"] == MAX_LEVEL
    with pytest.raises(pgq.PgqError) as ex:
        csr.cheapest_path([0], [MAX_LEVEL + 1])
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("n,lanes", [((1 << 20) + 1, 128)])
def test_device_lane_count_shrinks_with_n(gpu_ctx, n, lanes):
    """More than 2^20 vertices -> 128 lanes; 200 rows from 8 sources -> two batches.  Against the restatement on
    scipy's Dijkstra (the oracle would need gigabytes here): every step tight, the edge its parent's first tight one."""
    rng = np.random.default_rng(n)
    src = np.repeat(np.arange(n, dtype=np.int64), 2)
    dst = rng.integers(0, n, len(src))
    w = rng.integers(0, 4, len(src))  # few distinct costs: many ties
    ps = rng.choice(rng.choice(n, 8, replace=False), 200)
    pd = rng.integers(0, n, 200)
    csr = device_csr(gpu_ctx, n, src, dst, w, chunk=1 << 20)
    paths, st = csr.cheapest_path(ps, pd)
    csr.free()
    assert st["lanes"] == lanes and st["batches"] == -(-200 // lanes)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    rows = np.repeat(np.arange(n), np.diff(v[: n + 1]))
    mat = csr_matrix((ww + 1e-300, (rows, e)), shape=(n, n))
    srcs = np.unique(ps)
    D = dijkstra(mat, indices=srcs)
    D = np.where(np.isinf(D), np.inf, np.round(D))
    reached = 0
    for k, s in enumerate(srcs):
        d = D[k]
        tight = np.isfinite(d[rows]) & (d[rows] + ww == d[e])
        for i in np.flatnonzero(ps == s):
            if not np.isfinite(d[pd[i]]):
                assert paths[i] is None
                continue
            reached += 1
            path = paths[i]
            assert sum(path_weights(v, e, ids, ww, path)) == d[pd[i]]
            for j in range(2, len(path), 2):
                a, eid, b = path[j - 2], path[j - 1], path[j]
                q = [x for x in range(v[a], v[a + 1]) if tight[x] and e[x] == b]
                assert q and ids[q[0]] == eid
    assert 0 < reached < 200


@pytest.mark.gpu
def test_device_errors(gpu_ctx):
    csr = device_csr(gpu_ctx, 4, [0, 1], [1, 2], np.array([1, 2]))
    for ps, pd, sv, dv in (([0, 4], [1, 1], None, None), ([0, 1], [1, -1], None, None)):
        with pytest.raises(pgq.PgqError) as ex:
            csr.cheapest_path(ps, pd, sv, dv)
        assert ex.value.status == PGQ_ERR_RANGE
    paths, _ = csr.cheapest_path([0, 9], [9, 1], [1, 0], [0, 1])  # outside ids under NULL are never read
    assert paths == [None, None]
    paths, st = csr.cheapest_path([], [])
    assert paths == [] and st["batches"] == 0
    csr.free()
    from duckpgq_extension_b200 import _native
    import ctypes as C
    lib = _native.load()
    un = pgq.DeviceCSR.build(gpu_ctx, 3, np.array([0]), np.array([1]))
    for call in (lambda: un.cheapest_path([0], [1]), lambda: un.cheapest_path_length([0], [1])):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == PGQ_ERR_NOT_INITIALIZED
        assert lib.pgq_last_error() == b"Need to initialize CSR before doing cheapest path"  # the ABI's text
    un.free()
    h = pgq.DeviceCSR.build(gpu_ctx, 3, np.array([0]), np.array([1]))
    assert lib.pgq_cheapest_path(h._h, -1, None, None, None, None, None, None, None, None, None, None) == PGQ_ERR_INVALID_ARG
    assert lib.pgq_cheapest_path(h._h, 1, None, None, None, None, None, None, None,
                                 C.byref(C.POINTER(C.c_int64)()), C.byref(C.c_int64()), None) == PGQ_ERR_INVALID_ARG
    h.free()


@pytest.mark.gpu
def test_udf_mirror(gpu_ctx):
    state = pgq.DuckPGQState(gpu_ctx)
    with pytest.raises(pgq.ConstraintException) as ex:
        pgq.cheapest_path(state, 3, 4, [0], [1])
    assert "CSR not found with ID 3" in str(ex.value)
    pgq.create_csr_vertex(state, 0, 4, np.arange(4), np.array([1, 1, 0, 0]))
    pgq.create_csr_edge(state, 0, 4, 2, 2, [0, 1], [1, 2], [10, 11], np.array([3, 4]))
    paths = pgq.cheapest_path(state, 0, 4, [0, 0, 3], [2, 0, 2])
    assert paths == [[0, 10, 1, 11, 2], [0], None] and 0 in state.csr_to_delete
    state.query_end()
    pgq.create_csr_vertex(state, 1, 3, np.arange(3), np.array([1, 0, 0]))
    pgq.create_csr_edge(state, 1, 3, 1, 1, [0], [1], [0])
    with pytest.raises(pgq.PgqError) as ex:
        pgq.cheapest_path(state, 1, 3, [0], [1])
    assert "Need to initialize CSR before doing cheapest path" in str(ex.value) and 1 in state.csr_to_delete
    state.query_end()


@pytest.mark.gpu
def test_one_workspace_in_turn(gpu_ctx):
    """iterativelength, shortestpath, cheapest_path_length and cheapest_path called in turn from one thread (so on the
    context's one pooled workspace), repeated, answer as each does alone: the search masks' known-zero rows stay
    intact."""
    n, src, dst = datagen.rmat_edges(12)
    rng = np.random.default_rng(3)
    w = rng.integers(1, 30, len(src))
    ps, pd = datagen.hashed_pairs(300, n)
    csr = device_csr(gpu_ctx, n, src, dst, w)
    alone = (csr.iterativelength(ps, pd)[:2], csr.shortestpath(ps, pd)[0], csr.cheapest_path_length(ps, pd)[:2],
             csr.cheapest_path(ps, pd)[0])
    for _ in range(2):
        il = csr.iterativelength(ps, pd)[:2]
        cp = csr.cheapest_path(ps, pd)[0]
        sp = csr.shortestpath(ps, pd)[0]
        cl = csr.cheapest_path_length(ps, pd)[:2]
        assert np.array_equal(il[0], alone[0][0]) and np.array_equal(il[1], alone[0][1])
        assert sp == alone[1] and cp == alone[3]
        assert np.array_equal(cl[0], alone[2][0]) and np.array_equal(cl[1], alone[2][1])
    csr.free()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    """Eight threads call cheapest_path on one CSR built from chunks sent by four threads
    (pgq_csr_add_edges_weighted).  Each thread sends the edges of its own range of source vertices, so the order
    inside every adjacency list is the input order whatever the threads' timing."""
    n, src, dst = datagen.rmat_edges(12)
    rng = np.random.default_rng(8)
    w = rng.integers(1, 50, len(src)).astype(np.float64) / 4
    m = len(src)
    csr = pgq.DeviceCSR.create(gpu_ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    by_src = np.argsort(src, kind="stable")
    parts = [by_src[(src[by_src] >= lo) & (src[by_src] < lo + n // 4)] for lo in range(0, n, n // 4)]
    ths = [threading.Thread(target=lambda ix=ix: csr.add_edges(m, m, src[ix], dst[ix], ix, w[ix])) for ix in parts]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.finalize()
    ps, pd = datagen.hashed_pairs(200, n)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    exp, _ = orc_cp.cheapest_path(n, v, e, ids, ww, ps, pd, None, None, 256)
    out = [None] * 8

    def work(k):
        out[k] = csr.cheapest_path(ps, pd)[0]

    ths = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(o == exp for o in out)
