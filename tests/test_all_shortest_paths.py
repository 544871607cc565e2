"""shortest_path_count and all_shortest_paths: every shortest path of a row, SQL/PGQ's ALL SHORTEST
(include/duckpgq_b200.h, pgq_shortest_path_count / pgq_all_shortest_paths).

The CPU tests pin the oracle (oracle/pgq_oracle_allshortest.c: one sequential BFS per distinct source, saturating
path counts, a depth-first enumeration in step order) against independent restatements: the count is (A^h)[s, t]
computed with Python integers over the adjacency matrix with edge multiplicities and clamped to INT64_MAX; on small
graphs the lists are the walks of length h that a brute-force search finds, sorted by their step key; path 0 is
orc.shortestpath's path; a saturated row's first lists come from a lazy product over its diamonds.  They also show that
each case of the catalogue reaches what it is named after.  The GPU tests require the device's counts, validity and
lists to equal the oracle's, and its BFS counters to equal pgq_shortestpath's.
"""
import itertools
import threading

import numpy as np
import pytest

from conftest import golden_names, load_golden
from duckpgq_extension_b200 import datagen, pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_INVALID_ARG, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_RANGE
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_keys as orc_keys

PGQ_ERR_UNSUPPORTED = 8
INT64_MAX = (1 << 63) - 1
DEPTH_MAX = 65533  # path mode's levels are uint16: 0xFFFF = not reached, and a level 0xFFFE may not find a vertex
BFS_COUNTERS = ("batches", "levels", "edges_traversed", "frontier_vertices", "push_levels", "pull_levels", "lanes",
                "searches", "pruned", "search_rows")


# ---- independent restatements ----------------------------------------------------------------------------------------
def ref_csr(n, src, dst, eid=None):
    return orc.csr_build(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), eid)


def depth(n, v, e, s):
    dist = [-1] * n
    dist[s] = 0
    q = [s]
    for u in q:
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            if dist[w] < 0:
                dist[w] = dist[u] + 1
                q.append(w)
    return dist


def matrix_count(n, v, e, s, t):
    """(A^h)[s, t] with Python integers, A with edge multiplicities, clamped to INT64_MAX; None when t is unreachable"""
    h = depth(n, v, e, s)[t]
    if h < 0:
        return None
    vec = [0] * n
    vec[s] = 1
    for _ in range(h):
        nxt = [0] * n
        for u in range(n):
            if vec[u]:
                for idx in range(v[u], v[u + 1]):
                    nxt[int(e[idx])] += vec[u]
        vec = nxt
    return min(vec[t], INT64_MAX)


def brute_lists(n, v, e, ids, s, t):
    """every walk of h(s, t) edges from s to t as [s, e1, v1, ..., t], sorted by its steps from t back to s, a step
    being (parent, the edge's position in the parent's adjacency)"""
    h = depth(n, v, e, s)[t]
    if h < 0:
        return None
    walks = []

    def walk(u, k, elems, steps):
        if k == h:
            if u == t:
                walks.append((list(reversed(steps)), elems))
            return
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            walk(w, k + 1, elems + [int(ids[idx]), w], steps + [(u, idx - int(v[u]))])

    walk(s, 0, [s], [])
    return [el for _, el in sorted(walks, key=lambda x: x[0])]


def random_multigraph(seed, n_lo=6, n_hi=30):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(n_lo, n_hi))
    m = int(rng.integers(n, 4 * n))
    src = rng.integers(0, n, m)
    dst = rng.integers(0, n, m)
    k = m // 5  # parallel edges and self-loops
    src = np.concatenate([src, src[:k], np.arange(3) % n])
    dst = np.concatenate([dst, dst[:k], np.arange(3) % n])
    perm = rng.permutation(len(src))
    return n, src[perm], dst[perm]


def diamonds(k):
    """k diamonds in a row: x_i -> a_i, x_i -> b_i, a_i -> x_i+1, b_i -> x_i+1; 2^k paths of 2k edges from x_0 to x_k.
    x_i = 3i, a_i = 3i + 1, b_i = 3i + 2."""
    src, dst = [], []
    for i in range(k):
        x, a, b, y = 3 * i, 3 * i + 1, 3 * i + 2, 3 * i + 3
        src += [x, x, a, b]
        dst += [a, b, y, y]
    return 3 * k + 1, np.array(src), np.array(dst)


def diamond_lists(k, ids_of, count):
    """the first `count` paths of diamonds(k) in step order, lazily: the step nearest t varies slowest, and at every
    diamond the parent a_i (smaller id) comes before b_i"""
    out = []
    for choice in itertools.product((0, 1), repeat=k):  # choice[0]: the diamond nearest t
        mids = {k - 1 - j: c for j, c in enumerate(choice)}
        path = [0]
        for i in range(k):
            mid = 3 * i + 1 + mids[i]
            path += [ids_of[(3 * i, mid)], mid, ids_of[(mid, 3 * i + 3)], 3 * i + 3]
        out.append(path)
        if len(out) == count:
            return out
    return out


def edge_id_map(v, e, ids):
    m = {}
    for u in range(len(v) - 2):
        for idx in range(v[u], v[u + 1]):
            m.setdefault((u, int(e[idx])), int(ids[idx]))
    return m


# ---- the catalogue ---------------------------------------------------------------------------------------------------
def case_hub_ties():
    """0 -> parents 1..8 -> 9, parent i with i more edges into sinks: the device numbers the parents by descending
    degree, opposite to their ids, and the paths must come in the order of the ORIGINAL ids 1..8"""
    src, dst = [], []
    for i in range(1, 9):
        src += [0, i]
        dst += [i, 9]
    sink = 10
    for i in range(1, 9):
        for _ in range(i):
            src.append(i)
            dst.append(sink)
            sink += 1
    return dict(n=sink, src=src, dst=dst, ps=[0, 0, 1], pd=[9, 10, 9])


def case_parallel():
    """three parallel edges 0 -> 1 and two 1 -> 2, a self-loop at 1: 6 paths 0 -> 2"""
    return dict(n=3, src=[0, 1, 0, 1, 0, 1], dst=[1, 2, 1, 1, 1, 2], ps=[0, 0, 1], pd=[2, 1, 2])


def case_specials():
    """src == dst, NULL source, NULL destination, an unreachable row"""
    return dict(n=5, src=[0, 1, 2, 3], dst=[1, 2, 0, 3], ps=[0, 0, 1, 4, 0, 2], pd=[0, 2, 3, 0, 1, 1],
                sv=[1, 0, 1, 1, 1, 1], dv=[1, 1, 0, 1, 1, 1])


def case_edgeless():
    return dict(n=4, src=[], dst=[], ps=[0, 1, 2, 3], pd=[0, 2, 2, 1])


def case_rows(p, seed=5):
    n, src, dst = random_multigraph(seed, 40, 41)
    rng = np.random.default_rng(p)
    return dict(n=n, src=src, dst=dst, ps=rng.integers(0, n, p), pd=rng.integers(0, n, p))


CATALOGUE = {
    "hub_ties": case_hub_ties,
    "parallel": case_parallel,
    "specials": case_specials,
    "edgeless": case_edgeless,
    "diamonds62": lambda: dict(zip(("n", "src", "dst"), diamonds(62)), ps=[0, 0, 3], pd=[186, 6, 186]),
    **{f"rows{p}": (lambda p=p: case_rows(p)) for p in (1, 31, 32, 33, 255, 256, 257, 513)},
}


def oracle_csr(c):
    return ref_csr(c["n"], c["src"], c["dst"])


def internal_order(n, src, dst):
    """the device's vertex numbering (DESIGN section 2): class (out and in, in only, out only, isolated), then
    descending out-degree (descending in-degree for in-only vertices), stable"""
    outd, ind = np.bincount(src, minlength=n), np.bincount(dst, minlength=n)
    cls = np.where(outd > 0, np.where(ind > 0, 0, 2), np.where(ind > 0, 1, 3))
    deg = np.where(cls == 1, ind, outd)
    return sorted(range(n), key=lambda x: (cls[x], -deg[x]))


# ---- CPU: the oracle against the restatements ------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_oracle_counts_are_matrix_powers(seed):
    n, src, dst = random_multigraph(seed)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    cnt, valid = oas.shortest_path_count(n, v, e, ids, ps, pd)
    for i in range(len(ps)):
        exp = matrix_count(n, v, e, int(ps[i]), int(pd[i]))
        assert (cnt[i] if valid[i] else None) == exp, (seed, ps[i], pd[i])


@pytest.mark.parametrize("seed", range(10))
def test_oracle_lists_are_the_brute_force_walks(seed):
    n, src, dst = random_multigraph(100 + seed, 4, 9)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    paths, cnt = oas.all_shortest_paths(n, v, e, ids, ps, pd, 0)
    for i in range(len(ps)):
        exp = brute_lists(n, v, e, ids, int(ps[i]), int(pd[i]))
        assert paths[i] == exp, (seed, ps[i], pd[i])
        assert exp is None or cnt[i] == len(exp)
    limited, _ = oas.all_shortest_paths(n, v, e, ids, ps, pd, 2)
    assert limited == [None if x is None else x[:2] for x in paths]


@pytest.mark.parametrize("seed", range(6))
def test_oracle_path0_is_shortestpath(seed):
    n, src, dst = random_multigraph(200 + seed, 20, 60)
    v, e, ids = ref_csr(n, src, dst)
    rng = np.random.default_rng(seed)
    ps, pd = rng.integers(0, n, 300), rng.integers(0, n, 300)
    paths, _ = oas.all_shortest_paths(n, v, e, ids, ps, pd, 1)
    sp, _ = orc.shortestpath(n, v, e, ids, ps, pd)
    assert [None if x is None else x[0] for x in paths] == sp


def test_catalogue_hub_ties_disagree_with_the_internal_order():
    c = case_hub_ties()
    order = internal_order(c["n"], np.array(c["src"]), np.array(c["dst"]))
    parents = [x for x in order if 1 <= x <= 8]
    assert parents == sorted(parents, reverse=True)
    v, e, ids = oracle_csr(c)
    paths, cnt = oas.all_shortest_paths(c["n"], v, e, ids, c["ps"], c["pd"])
    assert cnt.tolist() == [8, 1, 1] and [p[2] for p in paths[0]] == list(range(1, 9))


def test_catalogue_parallel_edges():
    c = case_parallel()
    v, e, ids = oracle_csr(c)
    paths, cnt = oas.all_shortest_paths(c["n"], v, e, ids, c["ps"], c["pd"])
    assert cnt.tolist() == [6, 3, 2] and len({tuple(p) for p in paths[0]}) == 6
    assert paths[0] == brute_lists(c["n"], v, e, ids, 0, 2)


def case_duplicated_key():
    """vertex key 7 on rows 1 and 2: the key build puts edges 0 (7 -> 9) and 2 (7 -> 5) into both their adjacencies,
    and the edge 5 -> 9 twice into row 0's"""
    return dict(vk=np.array([5, 7, 7, 9]), es=np.array([7, 5, 7, 5]), ed=np.array([9, 9, 5, 9]), ps=[1, 2, 1, 2, 0],
                pd=[3, 3, 0, 0, 3])


def test_catalogue_duplicated_source_key():
    c = case_duplicated_key()
    n = len(c["vk"])
    v, e, ids = orc_keys.csr_build_keys(c["vk"], c["es"], c["ed"])
    paths, cnt = oas.all_shortest_paths(n, v, e, ids, c["ps"], c["pd"])
    assert paths == [[[1, 0, 3]], [[2, 0, 3]], [[1, 2, 0]], [[2, 2, 0]], [[0, 1, 3], [0, 3, 3]]]
    assert cnt.tolist() == [1, 1, 1, 1, 2]


def test_catalogue_diamonds_exact_and_saturated():
    n, src, dst = diamonds(62)
    v, e, ids = ref_csr(n, src, dst)
    cnt, valid = oas.shortest_path_count(n, v, e, ids, [0, 0], [186, 6])
    assert cnt.tolist() == [1 << 62, 4] and cnt[0] == matrix_count(n, v, e, 0, 186)
    n, src, dst = diamonds(63)
    v, e, ids = ref_csr(n, src, dst)
    cnt, valid = oas.shortest_path_count(n, v, e, ids, [0], [189])
    assert cnt.tolist() == [INT64_MAX] and matrix_count(n, v, e, 0, 189) == INT64_MAX  # 2^63 saturates


def test_catalogue_saturated_row_first_lists():
    n, src, dst = diamonds(64)
    v, e, ids = ref_csr(n, src, dst)
    paths, cnt = oas.all_shortest_paths(n, v, e, ids, [0], [192], 5)
    assert cnt.tolist() == [INT64_MAX]
    assert paths[0] == diamond_lists(64, edge_id_map(v, e, ids), 5)
    with pytest.raises(orc.OracleError) as ex:
        oas.all_shortest_paths(n, v, e, ids, [0], [192], 0)
    assert ex.value.code == oas.ERR_UNSUPPORTED


def test_catalogue_specials_and_edgeless():
    c = case_specials()
    v, e, ids = oracle_csr(c)
    paths, cnt = oas.all_shortest_paths(c["n"], v, e, ids, c["ps"], c["pd"], 0, c["sv"], c["dv"])
    assert paths == [[[0]], None, None, None, [[0, 0, 1]], [[2, 2, 0, 0, 1]]] and cnt.tolist() == [1, 0, 0, 0, 1, 1]
    c = case_edgeless()
    v, e, ids = oracle_csr(c)
    paths, cnt = oas.all_shortest_paths(c["n"], v, e, ids, c["ps"], c["pd"])
    assert paths == [[[0]], None, [[2]], None]


@pytest.mark.parametrize("p", [1, 31, 32, 33, 255, 256, 257, 513])
def test_catalogue_row_counts(p):
    c = case_rows(p)
    v, e, ids = oracle_csr(c)
    cnt, valid = oas.shortest_path_count(c["n"], v, e, ids, c["ps"], c["pd"])
    assert len(cnt) == p and valid.sum() > 0
    for i in range(min(p, 40)):
        assert (cnt[i] if valid[i] else None) == matrix_count(c["n"], v, e, int(c["ps"][i]), int(c["pd"][i]))


def chain(n):
    return n, np.arange(n - 1), np.arange(1, n)


def test_catalogue_depth_limit():
    n, src, dst = chain(DEPTH_MAX + 2)
    v, e, ids = ref_csr(n, src, dst)
    paths, cnt = oas.all_shortest_paths(n, v, e, ids, [0], [DEPTH_MAX])
    assert cnt.tolist() == [1] and len(paths[0][0]) == 2 * DEPTH_MAX + 1
    with pytest.raises(orc.OracleError) as ex:
        oas.shortest_path_count(n, v, e, ids, [0], [DEPTH_MAX + 1])
    assert ex.value.code == oas.ERR_UNSUPPORTED


# ---- GPU: the device against the oracle --------------------------------------------------------------------------------
def compare(csr, n, v, e, ids, ps, pd, sv=None, dv=None, max_paths=(0,), options=None):
    cnt, valid, st = csr.shortest_path_count(ps, pd, sv, dv, options)
    ocnt, ovalid = oas.shortest_path_count(n, v, e, ids, ps, pd, sv, dv)
    assert np.array_equal(valid, ovalid) and np.array_equal(cnt, ocnt)
    out = {}
    for mp in max_paths:
        paths, dcnt, lst = csr.all_shortest_paths(ps, pd, mp, sv, dv, options)
        opaths, _ = oas.all_shortest_paths(n, v, e, ids, ps, pd, mp, sv, dv)
        assert np.array_equal(dcnt, ocnt)
        assert paths == opaths, f"max_paths={mp}"
        assert {k: lst[k] for k in BFS_COUNTERS} == {k: st[k] for k in BFS_COUNTERS}
        out[mp] = paths
    return cnt, out, st


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    c = CATALOGUE[name]()
    v, e, ids = oracle_csr(c)
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))
    mps = (1, 64) if name.startswith("diamonds") else (0, 1, 3)
    compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], c.get("sv"), c.get("dv"), mps)
    csr.free()


@pytest.mark.gpu
def test_device_duplicated_source_key(gpu_ctx):
    c = case_duplicated_key()
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, c["vk"], c["es"], c["ed"])
    v, e, ids = orc_keys.csr_build_keys(c["vk"], c["es"], c["ed"])
    compare(csr, len(c["vk"]), v, e, ids, c["ps"], c["pd"], max_paths=(0, 1))
    csr.free()


@pytest.mark.gpu
def test_device_saturation(gpu_ctx):
    n, src, dst = diamonds(64)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    paths, cnt, _ = csr.all_shortest_paths([0, 0], [192, 189], 5)
    assert cnt.tolist() == [INT64_MAX, INT64_MAX]
    assert paths[0] == diamond_lists(64, edge_id_map(v, e, ids), 5)
    with pytest.raises(pgq.PgqError) as ex:
        csr.all_shortest_paths([0], [192], 0)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    cnt, _, _ = csr.shortest_path_count([0, 0], [186, 6])
    assert cnt.tolist() == [1 << 62, 4]
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names())
def test_device_reference_graphs(gpu_ctx, name):
    g = load_golden(name)
    n = g["n"]
    v, e, ids = ref_csr(n, g["src"], g["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, n, g["src"], g["dst"])
    sv = g["psrc_valid"].astype(np.uint8)
    compare(csr, n, v, e, ids, g["psrc"], g["pdst"], sv, None, (1, 64))
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [12, 14, 16])
def test_device_rmat(gpu_ctx, scale):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(1024, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    cnt, paths, st = compare(csr, n, v, e, ids, ps, pd, max_paths=(1, 64))
    sp, sst = csr.shortestpath(ps, pd)
    assert [None if x is None else x[0] for x in paths[1]] == sp
    assert {k: st[k] for k in BFS_COUNTERS} == {k: sst[k] for k in BFS_COUNTERS}
    assert (cnt > 1).sum() > 0
    csr.free()


@pytest.mark.gpu
def test_device_options_do_not_change_results(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(700, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    base = compare(csr, n, v, e, ids, ps, pd, max_paths=(8,))[:2]
    variants = [pgq.Options(lanes) for lanes in (64, 128, 256, 512)]
    variants += [pgq.Options(256, direction=d) for d in (0, 1, 2)]
    variants += [pgq.Options(0, no_dedup=True), pgq.Options(0, no_prune=True)]
    for opt in variants:
        cnt, paths, st = compare(csr, n, v, e, ids, ps, pd, max_paths=(8,), options=opt)
        assert np.array_equal(cnt, base[0]) and paths == base[1]
        _, sst = csr.shortestpath(ps, pd, None, opt)
        assert {k: st[k] for k in BFS_COUNTERS} == {k: sst[k] for k in BFS_COUNTERS}
    csr.free()


@pytest.mark.gpu
def test_device_depth_limit(gpu_ctx):
    n, src, dst = chain(DEPTH_MAX + 2)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    paths, cnt, _ = csr.all_shortest_paths([0], [DEPTH_MAX])
    assert cnt.tolist() == [1] and paths[0][0] == [0] + [x for k in range(1, DEPTH_MAX + 1) for x in (k - 1, k)]
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_path_count([0], [DEPTH_MAX + 1])
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()


@pytest.mark.gpu
def test_device_construction_routes(gpu_ctx):
    n, src, dst = datagen.rmat_edges(10)
    ps, pd = datagen.hashed_pairs(400, n)
    v, e, ids = ref_csr(n, src, dst)
    m = len(src)
    chunked = pgq.DeviceCSR.create(gpu_ctx, n)
    chunked.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    for o in range(0, m, 1000):
        chunked.add_edges(m, m, src[o:o + 1000], dst[o:o + 1000], np.arange(o, min(o + 1000, m)))
    chunked.finalize()
    routes = [chunked, pgq.DeviceCSR.build(gpu_ctx, n, src, dst), pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)]
    for csr in routes:
        compare(csr, n, v, e, ids, ps, pd, max_paths=(4,))
        csr.free()
    up = pgq.DeviceCSR.upload(gpu_ctx, n, v, e)  # no ids: CSR positions
    compare(up, n, v, e, np.arange(len(e)), ps, pd, max_paths=(4,))
    up.free()
    rng = np.random.default_rng(4)
    vk = rng.permutation(n).astype(np.int64) * 3
    sources = np.flatnonzero((np.bincount(dst, minlength=n) == 0) & (np.bincount(src, minlength=n) > 0))
    dup = vk.copy()
    dup[sources[1]] = dup[sources[0]]  # a duplicated source key (no edge ends there, so every join stays unique)
    for keys, undirected in ((vk, False), (dup, False), (vk, True)):
        es, ed = keys[src], keys[dst]
        csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, es, ed, undirected=undirected)
        kv, ke, kids = csr.download()
        compare(csr, csr.n, kv, ke, kids, ps % csr.n, pd % csr.n, max_paths=(4,))
        csr.free()


@pytest.mark.gpu
def test_device_errors(gpu_ctx):
    import ctypes as C
    from duckpgq_extension_b200 import _native
    lib = _native.load()
    csr = pgq.DeviceCSR.build(gpu_ctx, 4, np.array([0, 1]), np.array([1, 2]))
    for call in (lambda: csr.shortest_path_count([0, 4], [1, 1]), lambda: csr.all_shortest_paths([0], [-1])):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == PGQ_ERR_RANGE
    paths, cnt, _ = csr.all_shortest_paths([0, 9], [9, 1], 0, [1, 0], [0, 1])  # ids under NULL are never read
    assert paths == [None, None] and cnt.tolist() == [0, 0]
    with pytest.raises(pgq.PgqError) as ex:
        csr.all_shortest_paths([0], [1], -1)
    assert ex.value.status == PGQ_ERR_INVALID_ARG
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_path_count([0], [1], options=pgq.Options(0, shard_index=0, shard_count=2))
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    p64 = C.POINTER(C.c_int64)
    assert lib.pgq_shortest_path_count(csr._h, 1, None, None, None, None, None, None, None, None) == PGQ_ERR_INVALID_ARG
    one = np.zeros(1, np.int64)
    assert lib.pgq_shortest_path_count(csr._h, 1, one.ctypes.data_as(p64), one.ctypes.data_as(p64), None, None, None,
                                       None, None, None) == PGQ_ERR_INVALID_ARG
    assert lib.pgq_all_shortest_paths(csr._h, 1, one.ctypes.data_as(p64), one.ctypes.data_as(p64), None, None, None, 0,
                                      None, None, None, None, None, None, None, None) == PGQ_ERR_INVALID_ARG
    paths, cnt, st = csr.all_shortest_paths([], [])
    assert paths == [] and st["batches"] == 0
    csr.free()
    un = pgq.DeviceCSR.create(gpu_ctx, 3)
    for call in (lambda: un.shortest_path_count([0], [1]), lambda: un.all_shortest_paths([0], [1])):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == PGQ_ERR_NOT_INITIALIZED
    un.free()


@pytest.mark.gpu
def test_udf_mirror(gpu_ctx):
    state = pgq.DuckPGQState(gpu_ctx)
    with pytest.raises(pgq.ConstraintException) as ex:
        pgq.all_shortest_paths(state, 3, 4, [0], [1])
    assert "Invalid ID" in str(ex.value)
    pgq.create_csr_vertex(state, 0, 4, np.arange(4), np.array([2, 1, 1, 0]))
    pgq.create_csr_edge(state, 0, 4, 4, 4, [0, 0, 1, 2], [1, 2, 3, 3], [10, 11, 12, 13])
    paths = pgq.all_shortest_paths(state, 0, 4, [0, 0, 3], [3, 0, 0], 0)
    assert paths == [[[0, 10, 1, 12, 3], [0, 11, 2, 13, 3]], [[0]], None] and 0 in state.csr_to_delete
    counts, valid = pgq.shortest_path_count(state, 0, 4, [0, 0, 3], [3, 0, 0])
    assert counts.tolist() == [2, 1, 0] and valid.tolist() == [1, 1, 0]
    assert pgq.shortestpath(state, 0, 4, [0], [3]) == [paths[0][0]]
    state.query_end()


@pytest.mark.gpu
def test_one_workspace_in_turn(gpu_ctx):
    """shortestpath, iterativelength, cheapest_path and both new functions in turn on the context's one pooled
    workspace answer as each does alone"""
    n, src, dst = datagen.rmat_edges(12)
    w = np.random.default_rng(3).integers(1, 30, len(src))
    ps, pd = datagen.hashed_pairs(300, n)
    csr = pgq.DeviceCSR.create(gpu_ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    csr.add_edges(len(src), len(src), src, dst, np.arange(len(src)), w)
    csr.finalize()
    alone = (csr.shortestpath(ps, pd)[0], csr.iterativelength(ps, pd)[:2], csr.cheapest_path(ps, pd)[0],
             csr.shortest_path_count(ps, pd)[0], csr.all_shortest_paths(ps, pd, 16)[0])
    for _ in range(2):
        ap = csr.all_shortest_paths(ps, pd, 16)[0]
        sp = csr.shortestpath(ps, pd)[0]
        cnt = csr.shortest_path_count(ps, pd)[0]
        il = csr.iterativelength(ps, pd)[:2]
        cp = csr.cheapest_path(ps, pd)[0]
        assert sp == alone[0] and cp == alone[2] and ap == alone[4]
        assert np.array_equal(il[0], alone[1][0]) and np.array_equal(il[1], alone[1][1])
        assert np.array_equal(cnt, alone[3])
    csr.free()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(200, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    exp, _ = oas.all_shortest_paths(n, v, e, ids, ps, pd, 8)
    out = [None] * 8

    def work(k):
        out[k] = csr.all_shortest_paths(ps, pd, 8)[0]

    ths = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(o == exp for o in out)
