"""cheapest_path_count and all_cheapest_paths: every cheapest path of a row, the walks of the edges its Bellman-Ford
distances make tight, in the order of all_shortest_paths within a length (include/duckpgq_b200.h).

The CPU tests pin the oracle (oracle/pgq_oracle_allcheapest.c) against independent restatements: a brute-force
enumeration of tight walks in Python on random small multigraphs (zero and negative weights without negative cycles,
NaN, self-loops, parallel edges), a separate search for a tight cycle on a tight s -> t route, the worked examples of
the header, and the existing oracles (unit weights: all_shortest_paths; zero weights: shortest_k_paths; path 0:
cheapest_path).  The GPU tests require the device's validity, counts, lists and counters to equal the oracle's, and
check the same identities with the device's own functions.
"""
import ctypes as C
import math

import numpy as np
import pytest

from duckpgq_extension_b200 import _native, datagen, pgq
from duckpgq_extension_b200.pgq import (PGQ_ERR_INVALID_ARG, PGQ_ERR_INVALID_ID, PGQ_ERR_NOT_INITIALIZED,
                                        PGQ_ERR_RANGE, PGQ_ERR_UNSUPPORTED)
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allcheapest as oac
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_cheapest as ocp
from oracle import pgq_oracle_kshortest as oks

INT64_MAX = (1 << 63) - 1
INF_I64 = INT64_MAX // 2
INF_F64 = 1.7976931348623157e308 / 2


# ---- graphs ---------------------------------------------------------------------------------------------------------
def weighted_csr(n, src, dst, w):
    return orc.csr_build_weighted(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w))


def example(which):
    a = [(0, 1, 1), (0, 2, 2), (1, 2, 1), (1, 3, 3), (2, 3, 2), (0, 3, 4)]
    edges = {"A": a, "B": a + [(2, 5, 1), (5, 5, 0)], "C": a + [(1, 4, 0), (4, 1, 0)],
             "D": [(0, 1, 0.1), (1, 2, 0.2), (0, 2, 0.3)]}[which]
    n = 3 if which == "D" else 6
    w = np.array([x[2] for x in edges], np.float64 if which == "D" else np.int64)
    return n, [x[0] for x in edges], [x[1] for x in edges], w


def has_negative_cycle(n, src, dst, w):
    d = np.full((n, n), np.inf)
    for a, b, x in zip(src, dst, w):
        if not math.isnan(float(x)):
            d[a, b] = min(d[a, b], float(x))
    for k in range(n):
        d = np.minimum(d, d[:, k:k + 1] + d[k:k + 1, :])
    return any(d[i, i] < 0 for i in range(n))


def random_multigraph(seed, is_f):
    """small multigraphs with self-loops, parallel edges, zero and negative weights (no negative cycle), NaN (DOUBLE)"""
    rng = np.random.default_rng(seed)
    while True:
        n = int(rng.integers(3, 8))
        m = int(rng.integers(n, 3 * n))
        src = rng.integers(0, n, m)
        dst = rng.integers(0, n, m)
        if is_f:
            w = rng.choice([0.0, 0.1, 0.2, 0.3, 0.5, 1.0, -0.1, np.nan], m, p=[.2, .15, .15, .15, .1, .1, .1, .05])
        else:
            w = rng.choice([0, 1, 2, 3, -1], m, p=[.3, .3, .2, .1, .1]).astype(np.int64)
        if not has_negative_cycle(n, src, dst, w):
            return n, src, dst, w


def all_rows(n):
    return np.repeat(np.arange(n), n), np.tile(np.arange(n), n)


# ---- the independent restatement ------------------------------------------------------------------------------------
def distances(n, v, e, w, s):
    """d(s, .) from orc_cheapest_path_length, the sentinel where the cost is NULL"""
    cost, valid = orc.cheapest_path_length(n, v, e, w, np.full(n, s), np.arange(n))
    inf = INF_F64 if w.dtype.kind == "f" else INF_I64
    return [cost[u] if valid[u] else inf for u in range(n)]


def tight_edges(n, v, e, w, d):
    """[(parent, position in the parent's adjacency, CSR index, child)] of the edges d makes tight"""
    out = []
    for a in range(n):
        for k in range(v[a], v[a + 1]):
            if w.dtype.kind == "f":
                ok = float(d[a]) + float(w[k]) == float(d[e[k]])
            else:
                ok = (int(d[a]) + int(w[k]) + 2**63) % 2**64 - 2**63 == int(d[e[k]])
            if ok:
                out.append((a, k - v[a], k, int(e[k])))
    return out


def brute_walks(tight, ids, s, t, max_len):
    """every tight walk s -> t of at most max_len edges, with its step key (walking back from t), in (length, key)
    order; the search enters only vertices with a tight walk to t"""
    out_edges, into = {}, {}
    for a, pos, k, b in tight:
        out_edges.setdefault(a, []).append((pos, k, b))
        into.setdefault(b, set()).add(a)
    live, stack = {t}, [t]
    while stack:
        for a in into.get(stack.pop(), ()):
            if a not in live:
                live.add(a)
                stack.append(a)
    res = []

    def go(u, elems, key):
        if u == t:
            res.append((len(key), tuple(reversed(key)), list(elems)))
        if len(key) == max_len:
            return
        for pos, k, b in out_edges.get(u, []):
            if b in live:
                go(b, elems + [int(ids[k]), b], key + [(u, pos)])

    if s in live:
        go(s, [s], [])
    res.sort(key=lambda x: (x[0], x[1]))
    return res


def tight_cycle_on_route(n, tight, s, t):
    """a separate search: a cycle of tight edges among the vertices that s reaches and that reach t"""
    fwd, bwd = {}, {}
    for a, _, _, b in tight:
        fwd.setdefault(a, set()).add(b)
        bwd.setdefault(b, set()).add(a)

    def closure(x, adj):
        seen, stack = {x}, [x]
        while stack:
            for y in adj.get(stack.pop(), ()):
                if y not in seen:
                    seen.add(y)
                    stack.append(y)
        return seen

    route = closure(s, fwd) & closure(t, bwd)
    for x in route:  # x reaches itself over >= 1 tight edge inside the route
        seen, stack = set(), [y for y in fwd.get(x, ()) if y in route]
        while stack:
            y = stack.pop()
            if y == x:
                return True
            if y not in seen:
                seen.add(y)
                stack.extend(z for z in fwd.get(y, ()) if z in route)
    return False


# ---- CPU: the oracle against the restatement ------------------------------------------------------------------------
@pytest.mark.parametrize("is_f", [False, True])
@pytest.mark.parametrize("seed", range(12))
def test_oracle_equals_brute_force(seed, is_f):
    n, src, dst, w = random_multigraph(seed, is_f)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    ps, pd = all_rows(n)
    cnt, valid, _ = oac.cheapest_path_count(n, v, e, ids, ww, ps, pd)
    K = 40
    paths, cnt2, _ = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, K)
    assert np.array_equal(cnt, cnt2)
    for s in range(n):
        d = distances(n, v, e, ww, s)
        tight = tight_edges(n, v, e, ww, d)
        for t in range(n):
            i = s * n + t
            inf = tight_cycle_on_route(n, tight, s, t)
            open_row = s == t or d[t] != (INF_F64 if is_f else INF_I64)
            if not inf:
                walks = brute_walks(tight, ids, s, t, n) if open_row else []
                assert cnt[i] == len(walks), (s, t)
                assert bool(valid[i]) == (len(walks) > 0)
                want = [x[2] for x in walks[:K]]
            else:
                assert cnt[i] == INT64_MAX and valid[i]
                last = (len(paths[i][-1]) - 1) // 2
                walks = brute_walks(tight, ids, s, t, last)
                assert len(walks) >= K
                want = [x[2] for x in walks[:K]]
            assert (paths[i] or []) == want, (s, t)


def test_worked_examples():
    n, s, d, w = example("A")
    v, e, ids, ww = weighted_csr(n, s, d, w)
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, [0, 0, 0, 3], [3, 2, 0, 0])
    assert cnt.tolist() == [4, 2, 1, 0]
    assert paths == [[[0, 5, 3], [0, 0, 1, 3, 3], [0, 1, 2, 4, 3], [0, 0, 1, 2, 2, 4, 3]],
                     [[0, 1, 2], [0, 0, 1, 2, 2]], [[0]], None]
    n, s, d, w = example("B")
    v, e, ids, ww = weighted_csr(n, s, d, w)
    assert oac.cheapest_path_count(n, v, e, ids, ww, [0], [3])[0].tolist() == [4]
    n, s, d, w = example("C")
    v, e, ids, ww = weighted_csr(n, s, d, w)
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, [0, 2], [3, 3], 6)
    assert cnt.tolist() == [INT64_MAX, 1]
    assert paths == [[[0, 5, 3], [0, 0, 1, 3, 3], [0, 1, 2, 4, 3], [0, 0, 1, 2, 2, 4, 3], [0, 0, 1, 6, 4, 7, 1, 3, 3],
                      [0, 0, 1, 6, 4, 7, 1, 2, 2, 4, 3]], [[2, 4, 3]]]
    with pytest.raises(orc.OracleError) as ei:
        oac.all_cheapest_paths(n, v, e, ids, ww, [0], [3], 0)
    assert ei.value.code == oac.ERR_UNSUPPORTED
    n, s, d, w = example("D")
    v, e, ids, ww = weighted_csr(n, s, d, w)
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, [0], [2])
    assert cnt.tolist() == [1] and paths == [[[0, 2, 2]]]


@pytest.mark.parametrize("seed", range(6))
def test_oracle_identities(seed):
    rng = np.random.default_rng(100 + seed)
    n = 40
    m = 160
    src, dst = rng.integers(0, n, m), rng.integers(0, n, m)
    ps, pd = rng.integers(0, n, 120), rng.integers(0, n, 120)
    # unit weights: all_shortest_paths, order included
    v, e, ids, ww = weighted_csr(n, src, dst, np.ones(m, np.int64))
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, 0)
    apaths, acnt = oas.all_shortest_paths(n, v, e, ids, ps, pd, 0)
    assert cnt.tolist() == acnt.tolist() and paths == apaths
    # path 0 is cheapest_path's, on weights 0..3
    w = rng.integers(0, 4, m).astype(np.int64)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, 3)
    cpaths, _ = ocp.cheapest_path(n, v, e, ids, ww, ps, pd)
    assert [x[0] if x else None for x in paths] == cpaths
    # zero weights: every walk is cheapest, so the first k are shortest_k_paths'
    v, e, ids, ww = weighted_csr(n, src, dst, np.zeros(m, np.int64))
    k = 7
    paths, _, _ = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, k)
    kpaths, _, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, k)
    assert paths == kpaths


def test_oracle_errors_and_nulls():
    n, s, d, w = example("A")
    v, e, ids, ww = weighted_csr(n, s, d, w)
    with pytest.raises(orc.OracleError):
        oac.all_cheapest_paths(n, v, e, ids, ww, [0], [3], -1)
    with pytest.raises(orc.OracleError):
        oac.all_cheapest_paths(n, v, e, ids, ww, [0], [9])
    paths, cnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, [0, 0, 4, 2], [3, 3, 4, 2], 0, [0, 1, 1, 1], [1, 0, 1, 1])
    assert paths == [None, None, [[4]], [[2]]] and cnt.tolist() == [0, 0, 1, 1]


# ---- GPU: the device against the oracle -----------------------------------------------------------------------------
def device_csr(ctx, n, src, dst, w):
    src, dst, w = np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w)
    m = len(src)
    csr = pgq.DeviceCSR.create(ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n) if m else np.zeros(n, np.int64))
    if m:
        csr.add_edges(m, m, src, dst, np.arange(m), w)
    csr.finalize()
    return csr


def compare(ctx, n, src, dst, w, ps, pd, max_paths, sv=None, dv=None):
    """the device's counts, validity, lists and counters equal the oracle's; -> (paths, counts, stats)"""
    csr = device_csr(ctx, n, src, dst, w)
    try:
        cnt, valid, cst = csr.cheapest_path_count(ps, pd, sv, dv)
        paths, cnt2, st = csr.all_cheapest_paths(ps, pd, max_paths, sv, dv)
        _, _, lst = csr.cheapest_path_length(ps, pd, sv, dv)
        cpaths, _ = csr.cheapest_path(ps, pd, sv, dv)
    finally:
        csr.free()
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    ocnt, ovalid, ost = oac.cheapest_path_count(n, v, e, ids, ww, ps, pd, sv, dv, st["lanes"])
    opaths, ocnt2, ost2 = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, max_paths, sv, dv, st["lanes"])
    assert cnt.tolist() == ocnt.tolist() and cnt2.tolist() == ocnt2.tolist() and valid.tolist() == ovalid.tolist()
    assert paths == opaths
    # (the number of sweeps varies from call to call with the order of the parallel relaxations; each sweep is one
    # launch, so launches - sweeps is fixed: three launches per batch for cheapest_path_length)
    assert lst["kernel_launches"] - lst["levels"] == 3 * lst["batches"]
    for s_ in (cst, st):
        assert (s_["batches"], s_["lanes"]) == (lst["batches"], lst["lanes"])
        assert (s_["batches"], s_["push_levels"]) == (ost["batches"], ost["push_levels"])
    assert cst["pull_levels"] == ost["pull_levels"] and st["pull_levels"] == ost2["pull_levels"]
    assert [x[0] if x else None for x in paths] == cpaths  # path 0 is cheapest_path's
    return paths, cnt, st


@pytest.fixture(scope="module")
def ctx():
    return pgq.default_context(0)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["A", "B", "C", "D"])
def test_device_worked_examples(ctx, which):
    n, s, d, w = example(which)
    ps, pd = all_rows(n)
    paths, cnt, _ = compare(ctx, n, s, d, w, ps, pd, 6)
    if which == "C":
        assert cnt[0 * n + 3] == INT64_MAX and len(paths[3]) == 6


@pytest.mark.gpu
@pytest.mark.parametrize("is_f", [False, True])
@pytest.mark.parametrize("seed", range(8))
def test_device_random_multigraphs(ctx, seed, is_f):
    n, src, dst, w = random_multigraph(seed, is_f)
    ps, pd = all_rows(n)
    compare(ctx, n, src, dst, w, ps, pd, 25)


def rmat_case(scale, kind, p, seed=0):
    n, src, dst = datagen.rmat_edges(scale)
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 4, len(src)).astype(np.int64) if kind == "i64" else rng.integers(1, 1025, len(src)) / 1024.0
    ps, pd = datagen.hashed_pairs(p, n)
    return n, src, dst, w, ps, pd


@pytest.mark.gpu
@pytest.mark.parametrize("scale,kind", [(9, "i64"), (9, "f64"), (10, "i64"), (10, "f64")])
def test_device_rmat(ctx, scale, kind):
    n, src, dst, w, ps, pd = rmat_case(scale, kind, 300)  # more rows than one sweep batch (256)
    ps[::11] = pd[::11]  # s == t
    sv = (np.arange(300) % 17 != 0).astype(np.uint8)
    dv = (np.arange(300) % 19 != 0).astype(np.uint8)
    paths, cnt, st = compare(ctx, n, src, dst, w, ps, pd, 16, sv, dv)
    assert st["batches"] == 2 and sum(x is not None for x in paths) > 100
    if kind == "i64":  # every listed path's weights sum to the cost
        v, e, ids, ww = weighted_csr(n, src, dst, w)
        cost, cvalid = orc.cheapest_path_length(n, v, e, ww, ps, pd, sv, dv)
        pos_of = {int(i): k for k, i in enumerate(ids)}
        for i, rows in enumerate(paths):
            for path in rows or []:
                assert sum(int(ww[pos_of[x]]) for x in path[1::2]) == cost[i]


@pytest.mark.gpu
def test_device_identities(ctx):
    n, src, dst = datagen.rmat_edges(9)
    ps, pd = datagen.hashed_pairs(300, n)
    m = len(src)
    csr = device_csr(ctx, n, src, dst, np.ones(m, np.int64))
    plain = pgq.DeviceCSR.build(ctx, n, src, dst)
    try:
        cnt, valid, _ = csr.cheapest_path_count(ps, pd)
        scnt, svalid, _ = plain.shortest_path_count(ps, pd)
        assert cnt.tolist() == scnt.tolist() and valid.tolist() == svalid.tolist()
        paths, _, _ = csr.all_cheapest_paths(ps, pd, 50)
        apaths, _, _ = plain.all_shortest_paths(ps, pd, 50)
        assert paths == apaths
    finally:
        csr.free()
    zcsr = device_csr(ctx, n, src, dst, np.zeros(m, np.int64))
    try:
        paths, _, _ = zcsr.all_cheapest_paths(ps, pd, 5)
        kpaths, _, _ = plain.shortest_k_paths(ps, pd, 5)
        assert paths == kpaths
    finally:
        zcsr.free()
        plain.free()


@pytest.mark.gpu
def test_device_c_abi_and_udf_mirror(ctx):
    n, s, d, w = example("C")
    csr = device_csr(ctx, n, s, d, w)
    lib = _native.load()
    src, dst = np.array([0, 2], np.int64), np.array([3, 3], np.int64)
    cnt, npaths, first = (np.zeros(2, np.int64) for _ in range(3))
    ov = np.zeros(2, np.uint8)
    offs, elems, total = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)(), C.c_int64(0)
    p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
    rc = lib.pgq_all_cheapest_paths(csr._h, 2, p64(src), p64(dst), None, None, 6, p64(cnt), p64(npaths), p64(first),
                                    ov.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(offs), C.byref(elems),
                                    C.byref(total), None)
    assert rc == 0 and total.value == 7 and npaths.tolist() == [6, 1] and cnt.tolist() == [INT64_MAX, 1]
    assert [offs[j] for j in range(8)] == [0, 3, 8, 13, 20, 29, 40, 43]
    lib.pgq_free(offs)
    lib.pgq_free(elems)
    assert lib.pgq_cheapest_path_count(None, 1, p64(src), p64(dst), None, None, p64(cnt),
                                       ov.ctypes.data_as(C.POINTER(C.c_uint8)), None) == PGQ_ERR_INVALID_ID
    state = pgq.DuckPGQState(ctx)
    state.csr_list[0] = csr
    counts, valid = pgq.cheapest_path_count(state, 0, n, src, dst)
    assert counts.tolist() == [INT64_MAX, 1] and valid.tolist() == [1, 1] and 0 in state.csr_to_delete
    assert pgq.all_cheapest_paths(state, 0, n, src, dst, 1) == [[[0, 5, 3]], [[2, 4, 3]]]
    with pytest.raises(pgq.ConstraintException):
        pgq.all_cheapest_paths(state, 7, n, src, dst, 1)
    plain = pgq.DeviceCSR.build(ctx, n, np.array(s), np.array(d))
    state.csr_list[1] = plain
    with pytest.raises(pgq.ConstraintException) as ei:
        pgq.cheapest_path_count(state, 1, n, src, dst)
    assert ei.value.status == PGQ_ERR_NOT_INITIALIZED
    csr.free()
    plain.free()


@pytest.mark.gpu
def test_device_errors(ctx, monkeypatch):
    n, s, d, w = example("C")
    csr = device_csr(ctx, n, s, d, w)
    try:
        with pytest.raises(pgq.PgqError) as ei:
            csr.all_cheapest_paths([0], [3], -1)
        assert ei.value.status == PGQ_ERR_INVALID_ARG
        with pytest.raises(pgq.PgqError) as ei:
            csr.all_cheapest_paths([0], [3], 0)  # infinitely many
        assert ei.value.status == PGQ_ERR_UNSUPPORTED
        with pytest.raises(pgq.PgqError) as ei:
            csr.cheapest_path_count([0], [17])
        assert ei.value.status == PGQ_ERR_RANGE
        # the layer budget: a row's layers (H + 1) x n_ab x 8 bytes must fit (row 1: H = 10, n_ab = 4); a budget below two
        # rows' layers stores the rows one group at a time, with the same paths
        paths, _, st = csr.all_cheapest_paths([0, 0, 2, 1], [3, 2, 3, 3], 6)
        monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", "400")
        paths2, _, st2 = csr.all_cheapest_paths([0, 0, 2, 1], [3, 2, 3, 3], 6)
        assert paths2 == paths and st2["kernel_launches"] > st["kernel_launches"]
        monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", "100")
        with pytest.raises(pgq.PgqError) as ei:
            csr.all_cheapest_paths([0], [3], 6)
        assert ei.value.status == PGQ_ERR_UNSUPPORTED
        assert csr.cheapest_path_count([0], [3])[0].tolist() == [INT64_MAX]  # (a count stores no layers)
    finally:
        csr.free()
    plain = pgq.DeviceCSR.build(ctx, n, np.array(s), np.array(d))
    try:
        with pytest.raises(pgq.PgqError) as ei:
            plain.cheapest_path_count([0], [3])
        assert ei.value.status == PGQ_ERR_NOT_INITIALIZED
    finally:
        plain.free()


@pytest.mark.gpu
def test_device_walk_limit(ctx):
    """a zero-cost cycle through all 70000 vertices: |B(t)| = 70000, so the row still counts after 65533 edges"""
    k = 70000
    src = np.arange(k)
    dst = (np.arange(k) + 1) % k
    csr = device_csr(ctx, k, src, dst, np.zeros(k, np.int64))
    try:
        # a list of one path still needs the count, which is what runs into the limit
        for max_paths in (None, 3, 1):
            with pytest.raises(pgq.PgqError) as ei:
                if max_paths is None:
                    csr.cheapest_path_count([0], [5])
                else:
                    csr.all_cheapest_paths([0], [5], max_paths)
            assert ei.value.status == PGQ_ERR_UNSUPPORTED
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_empty_and_null_rows(ctx):
    n, s, d, w = example("A")
    csr = device_csr(ctx, n, s, d, w)
    try:
        paths, cnt, st = csr.all_cheapest_paths([], [], 0)
        assert paths == [] and st["batches"] == 0
        paths, cnt, _ = csr.all_cheapest_paths([0, 0, 3], [3, 3, 3], 0, [0, 1, 1], [1, 0, 1])
        assert paths == [None, None, [[3]]] and cnt.tolist() == [0, 0, 1]
    finally:
        csr.free()
