"""cheapest_k_paths: the k cheapest paths of a row in the WALK, TRAIL, ACYCLIC and SIMPLE path modes over a weighted CSR
with weights >= 0, ordered by cost, then length, then step order (include/duckpgq_b200.h).

The CPU tests pin the oracle (oracle/pgq_oracle_cheapest_k.c) against independent restatements: a brute-force
enumeration in Python on random small multigraphs (self-loops, parallel edges, zero weights, NaN edges; BIGINT and dyadic
DOUBLE weights), the worked examples of the header, and the existing oracles (weights all 0 or all 1: shortest_k_paths
and its modes; k = 1: cheapest_path; WALK: all_cheapest_paths).  The GPU tests require the device's validity, lists,
costs and deterministic counters to equal the oracle's, and check the same identities with the device's own functions.
"""
import ctypes as C
import math
import threading

import numpy as np
import pytest

from duckpgq_extension_b200 import _native, datagen, pgq
from duckpgq_extension_b200.pgq import (PGQ_ERR_INVALID_ARG, PGQ_ERR_INVALID_ID, PGQ_ERR_NOT_INITIALIZED,
                                        PGQ_ERR_RANGE, PGQ_ERR_UNSUPPORTED)
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allcheapest as oac
from oracle import pgq_oracle_cheapest as ocp
from oracle import pgq_oracle_cheapest_k as ock
from oracle import pgq_oracle_kpaths_modes as okm
from oracle import pgq_oracle_kshortest as oks
from oracle.pgq_oracle import OracleError

MODES = ("WALK", "TRAIL", "ACYCLIC", "SIMPLE")
KS = (1, 2, 3, 5, 10)


# ---- graphs ---------------------------------------------------------------------------------------------------------
def weighted_csr(n, src, dst, w):
    return orc.csr_build_weighted(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w))


def all_rows(n):
    return np.repeat(np.arange(n), n), np.tile(np.arange(n), n)


def least_cycle(n, src, dst, w):
    """the least cost of a cycle (NaN edges left out), inf without one"""
    d = np.full((n, n), np.inf)
    for a, b, x in zip(src, dst, w):
        if not math.isnan(float(x)):
            d[a, b] = min(d[a, b], float(x))
    for k in range(n):
        d = np.minimum(d, d[:, k:k + 1] + d[k:k + 1, :])
    return min(d[i, i] for i in range(n))


def random_multigraph(seed, is_f):
    """small multigraphs with self-loops, parallel edges, zero weights and (DOUBLE) NaN edges; dyadic doubles, so every
    sum is exact"""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(3, 7))
    m = int(rng.integers(n, 2 * n + 1))
    src = rng.integers(0, n, m)
    dst = rng.integers(0, n, m)
    if is_f:
        w = rng.choice([0.0, 0.25, 0.5, 1.0, 1.5, np.nan], m, p=[.15, .25, .2, .2, .1, .1])
    else:
        w = rng.choice([0, 1, 2, 3], m, p=[.2, .4, .25, .15]).astype(np.int64)
    return n, src, dst, w


# ---- the independent restatement ------------------------------------------------------------------------------------
def brute_paths(n, v, e, ids, w, s, t, mode, max_cost=None, max_len=None):
    """every path of the mode from s to t (WALK: of cost below max_cost and at most max_len edges), with its cost, in
    (cost, h, steps from t back to s) order; a step is (parent, position in the parent's adjacency)"""
    is_f = w.dtype.kind == "f"
    res = []

    def go(u, elems, key, verts, used, cost):
        if u == t:
            res.append((cost, len(key), tuple(reversed(key)), list(elems)))
        if mode == "WALK" and len(key) == max_len:
            return
        for k in range(v[u], v[u + 1]):
            b = int(e[k])
            x = float(w[k]) if is_f else int(w[k])
            if is_f and math.isnan(x):
                continue
            c = cost + x
            if mode == "WALK" and c >= max_cost:
                continue
            if mode == "TRAIL" and k in used:
                continue
            if mode == "ACYCLIC" and b in verts:
                continue
            if mode == "SIMPLE" and (b in verts and not (b == s == t)):
                continue
            if mode == "SIMPLE" and u == t == s and key:  # a closed simple path ends at its first return
                continue
            go(b, elems + [int(ids[k]), b], key + [(u, k - v[u])], verts | {b}, used | {k}, c)

    go(s, [s], [], {s}, frozenset(), 0.0 if is_f else 0)
    res.sort(key=lambda x: (x[0], x[1], x[2]))
    return [(r[3], r[0]) for r in res]


def fold_cost(path, pos_of, ww):
    """the path's weights summed left to right from 0 in the weight type's arithmetic"""
    c = 0.0 if ww.dtype.kind == "f" else 0
    for eid in path[1::2]:
        c = c + ww[pos_of[eid]]
    return c


def check_against_brute(n, src, dst, w):
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    ps, pd = all_rows(n)
    cyc = least_cycle(n, src, dst, w)
    big_h = 3 * n
    bound = (big_h // n) * cyc  # a walk of more than big_h edges holds big_h // n cycles, and costs at least this
    for mode in MODES:
        brute = {}
        for s, t in zip(ps.tolist(), pd.tolist()):
            brute[s, t] = brute_paths(n, v, e, ids, ww, s, t, mode, bound, big_h)
        for k in KS:
            paths, costs, npaths, _ = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, k, mode)
            for i, (s, t) in enumerate(zip(ps.tolist(), pd.tolist())):
                got = list(zip(paths[i] or [], costs[i] or []))
                exp = brute[s, t]
                if mode != "WALK":
                    assert got == exp[:k], (mode, k, s, t)
                elif len(exp) >= k:  # the k-th walk costs less than the bound: the enumeration holds every cheaper walk
                    assert got == exp[:k], (mode, k, s, t)
                else:
                    assert got[:len(exp)] == exp and all(c >= bound for _, c in got[len(exp):]), (mode, k, s, t)
                assert npaths[i] == len(got) and (paths[i] is None) == (len(got) == 0)


@pytest.mark.parametrize("is_f", [False, True])
@pytest.mark.parametrize("seed", range(30))
def test_oracle_equals_brute_force(seed, is_f):
    n, src, dst, w = random_multigraph(seed, is_f)
    if least_cycle(n, src, dst, w) == 0:  # WALK's enumeration needs every cycle to cost something: zero -> one
        w = np.where(w == 0, w + 1, w)
    check_against_brute(n, src, dst, w)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_modes_with_zero_cost_cycles(seed):
    """the modes admit finitely many paths whatever the cycles cost: zero-cost cycles included"""
    rng = np.random.default_rng(seed)
    n = 5
    src = np.concatenate([rng.integers(0, n, 8), [1, 2]])
    dst = np.concatenate([rng.integers(0, n, 8), [2, 1]])
    w = np.concatenate([rng.integers(0, 3, 8), [0, 0]]).astype(np.int64)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    ps, pd = all_rows(n)
    for mode in ("TRAIL", "ACYCLIC", "SIMPLE"):
        paths, costs, _, _ = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, 10, mode)
        for i, (s, t) in enumerate(zip(ps.tolist(), pd.tolist())):
            assert list(zip(paths[i] or [], costs[i] or [])) == brute_paths(n, v, e, ids, ww, s, t, mode)[:10]


def test_worked_examples():
    # a zero-cost cycle 1 -> 2 -> 1 on the route 0 -> 1 -> 3: WALK fills up with it, the modes do not
    n, src, dst, w = 4, [0, 1, 2, 1], [1, 2, 1, 3], np.array([1, 0, 0, 1], np.int64)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    got = {m: ock.cheapest_k_paths(n, v, e, ids, ww, [0], [3], 4, m)[:2] for m in MODES}
    assert got["WALK"] == ([[[0, 0, 1, 3, 3], [0, 0, 1, 1, 2, 2, 1, 3, 3], [0, 0, 1, 1, 2, 2, 1, 1, 2, 2, 1, 3, 3],
                             [0, 0, 1, 1, 2, 2, 1, 1, 2, 2, 1, 1, 2, 2, 1, 3, 3]]], [[2, 2, 2, 2]])
    assert got["TRAIL"] == ([[[0, 0, 1, 3, 3], [0, 0, 1, 1, 2, 2, 1, 3, 3]]], [[2, 2]])
    assert got["ACYCLIC"] == got["SIMPLE"] == ([[[0, 0, 1, 3, 3]]], [[2]])
    # {0 -> 1: 0.1, 1 -> 2: 0.2, 0 -> 2: 0.3}: 0.3 first, then 0.1 + 0.2 = 0.30000000000000004
    n, src, dst, w = 3, [0, 1, 0], [1, 2, 2], np.array([0.1, 0.2, 0.3])
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    paths, costs, _, _ = ock.cheapest_k_paths(n, v, e, ids, ww, [0, 0], [2, 0], 3, "WALK")
    assert paths == [[[0, 2, 2], [0, 0, 1, 1, 2]], [[0]]]
    assert costs == [[0.3, 0.1 + 0.2], [0.0]] and costs[0][1] == 0.30000000000000004


@pytest.mark.parametrize("seed", range(4))
def test_oracle_identities(seed):
    n, src, dst = datagen.rmat_edges(6, seed=seed)
    m = len(src)
    ps, pd = datagen.hashed_pairs(80, n)
    ps[::9] = pd[::9]
    pv, pe, pids = orc.csr_build(n, src, dst)
    for unit in (0, 1):  # every weight 0 or every weight 1: the unweighted sequence, costs 0 or h
        v, e, ids, ww = weighted_csr(n, src, dst, np.full(m, unit, np.int64))
        for mode in MODES:
            paths, costs, _, _ = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, 4, mode)
            if mode == "WALK":
                exp = oks.shortest_k_paths(n, pv, pe, pids, ps, pd, 4)[0]
            else:
                exp = okm.shortest_k_paths_mode(n, pv, pe, pids, ps, pd, 4, mode)[0]
            assert paths == exp
            assert costs == [None if r is None else [unit * (len(q) // 2) for q in r] for r in paths]
    rng = np.random.default_rng(seed)
    for w in (rng.integers(0, 4, m).astype(np.int64), rng.integers(0, 9, m) / 8.0):
        v, e, ids, ww = weighted_csr(n, src, dst, w)
        pos_of = {int(x): k for k, x in enumerate(ids)}
        cost, cvalid = orc.cheapest_path_length(n, v, e, ww, ps, pd)
        cpaths, _ = ocp.cheapest_path(n, v, e, ids, ww, ps, pd)
        acyclic = None
        for mode in MODES:
            one, one_c, _, _ = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, 1, mode)
            assert [r[0] if r else None for r in one] == cpaths  # k = 1: cheapest_path, with its cost
            assert [r[0] if r else None for r in one_c] == [cost[i] if cvalid[i] else None for i in range(len(ps))]
            paths, costs, _, _ = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, 6, mode)
            for r, rc in zip(paths, costs):
                assert rc is None or (rc == sorted(rc) and rc == [fold_cost(q, pos_of, ww) for q in r])
            if mode == "WALK" and w.dtype.kind == "i":  # the cheapest walks lead WALK's sequence
                apaths, acnt, _ = oac.all_cheapest_paths(n, v, e, ids, ww, ps, pd, 6)
                assert [r if r is None else r[:min(6, c)] for r, c in zip(paths, acnt.tolist())] == apaths
            if mode == "ACYCLIC":
                acyclic = paths
            if mode == "SIMPLE":  # SIMPLE is ACYCLIC for s != t
                assert [p for p, s, t in zip(paths, ps, pd) if s != t] == \
                       [p for p, s, t in zip(acyclic, ps, pd) if s != t]


def test_oracle_errors_and_nulls():
    n, src, dst, w = 4, [0, 1, 2, 1], [1, 2, 1, 3], np.array([1, 0, 0, 1], np.int64)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    for bad in (dict(k=0), dict(mode="BOGUS"), dict(lanes=512), dict(lanes=48)):
        args = dict(k=2, mode="WALK", lanes=0) | bad
        with pytest.raises(OracleError) as ei:
            ock.cheapest_k_paths(n, v, e, ids, ww, [0], [3], args["k"], args["mode"], lanes=args["lanes"])
        assert ei.value.code == ock.ERR_ARG
    with pytest.raises(OracleError) as ei:
        ock.cheapest_k_paths(n, v, e, ids, ww, [0], [9], 2)
    assert ei.value.code == ock.ERR_RANGE
    nv, ne, nids, nw = weighted_csr(n, src, dst, np.array([1.0, -0.5, 0.0, 1.0]))
    with pytest.raises(OracleError) as ei:
        ock.cheapest_k_paths(n, nv, ne, nids, nw, [0], [3], 2)
    assert ei.value.code == ock.ERR_UNSUPPORTED
    zv, ze, zids, zw = weighted_csr(n, src, dst, np.array([1.0, -0.0, 0.0, 1.0]))  # -0.0 is not below zero
    assert ock.cheapest_k_paths(n, zv, ze, zids, zw, [0], [3], 1)[1] == [[2.0]]
    paths, costs, npaths, _ = ock.cheapest_k_paths(n, v, e, ids, ww, [0, 0, 3, 2, 3], [3, 3, 3, 2, 0], 3, "SIMPLE",
                                                   [0, 1, 1, 1, 1], [1, 0, 1, 1, 1])
    assert paths == [None, None, [[3]], [[2], [2, 2, 1, 1, 2]], None] and costs == [None, None, [0], [0, 0], None]


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


def same_costs(a, b):
    """per-row cost lists equal bit for bit (NaN never occurs)"""
    return [None if r is None else [np.float64(x).tobytes() if isinstance(x, float) else x for x in r] for r in a] == \
           [None if r is None else [np.float64(x).tobytes() if isinstance(x, float) else x for x in r] for r in b]


def compare(csr, n, src, dst, w, ps, pd, k, mode, sv=None, dv=None, lanes=0):
    """the device's validity, lists, costs and deterministic counters equal the oracle's; -> (paths, costs, stats)"""
    paths, costs, npaths, st = csr.cheapest_k_paths(ps, pd, k, sv, dv, pgq.Options(lanes), mode)
    v, e, ids, ww = weighted_csr(n, src, dst, w)
    opaths, ocosts, onp, ost = ock.cheapest_k_paths(n, v, e, ids, ww, ps, pd, k, mode, sv, dv, lanes)
    assert npaths.tolist() == onp.tolist()
    assert paths == opaths
    assert same_costs(costs, ocosts)
    for key in ("batches", "lanes", "searches", "push_levels"):
        assert st[key] == ost[key], key
    assert st["levels"] >= st["batches"]
    return paths, costs, st


@pytest.fixture(scope="module")
def ctx():
    return pgq.default_context(0)


@pytest.mark.gpu
@pytest.mark.parametrize("is_f", [False, True])
@pytest.mark.parametrize("seed", range(8))
def test_device_random_multigraphs(ctx, seed, is_f):
    n, src, dst, w = random_multigraph(seed, is_f)
    ps, pd = all_rows(n)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        for mode in MODES:
            for k in (1, 3, 8):
                compare(csr, n, src, dst, w, ps, pd, k, mode)
    finally:
        csr.free()


def rmat_case(scale, kind, p, seed=0):
    n, src, dst = datagen.rmat_edges(scale)
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 8, len(src)).astype(np.int64) if kind == "i64" else rng.integers(0, 1025, len(src)) / 1024.0
    ps, pd = datagen.hashed_pairs(p, n)
    ps[::11] = pd[::11]  # s == t
    sv = (np.arange(p) % 17 != 0).astype(np.uint8)
    dv = (np.arange(p) % 19 != 0).astype(np.uint8)
    return n, src, dst, w, ps, pd, sv, dv


@pytest.mark.gpu
@pytest.mark.parametrize("scale,kind", [(9, "i64"), (9, "f64"), (10, "i64"), (10, "f64")])
def test_device_rmat(ctx, scale, kind):
    n, src, dst, w, ps, pd, sv, dv = rmat_case(scale, kind, 48)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        for mode in MODES:
            for k in (1, 3, 8):
                paths, costs, st = compare(csr, n, src, dst, w, ps, pd, k, mode, sv, dv)
                if k == 8:  # 32 lanes: several batches a round, the same results
                    paths32, costs32, st32 = compare(csr, n, src, dst, w, ps, pd, k, mode, sv, dv, 32)
                    assert paths32 == paths and same_costs(costs32, costs) and st32["batches"] > st["batches"]
        assert any(p is None for p in paths) and sum(p is not None for p in paths) > 20
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_unreachable_rows(ctx):
    n, src, dst, w = 6, [0, 1, 2, 3, 3], [1, 2, 0, 4, 4], np.array([1, 2, 3, 1, 1], np.int64)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        for mode in MODES:
            paths, _, _ = compare(csr, n, src, dst, w, [0, 3, 5, 4, 0], [4, 4, 5, 3, 0], 3, mode)
            assert paths[0] is None and paths[3] is None and paths[2] == [[5]]
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_identities(ctx):
    n, src, dst = datagen.rmat_edges(9)
    m = len(src)
    ps, pd = datagen.hashed_pairs(64, n)
    plain = pgq.DeviceCSR.build(ctx, n, src, dst)
    try:
        for unit in (0, 1):
            csr = device_csr(ctx, n, src, dst, np.full(m, unit, np.int64))
            try:
                for mode in MODES:
                    paths, costs, _, _ = csr.cheapest_k_paths(ps, pd, 4, mode=mode)
                    assert paths == plain.shortest_k_paths(ps, pd, 4, mode=mode)[0]
                    assert costs == [None if r is None else [unit * (len(q) // 2) for q in r] for r in paths]
            finally:
                csr.free()
    finally:
        plain.free()
    rng = np.random.default_rng(1)
    for w in (rng.integers(0, 4, m).astype(np.int64), rng.integers(0, 9, m) / 8.0):
        csr = device_csr(ctx, n, src, dst, w)
        try:
            cost, cvalid, _ = csr.cheapest_path_length(ps, pd)
            cpaths, _ = csr.cheapest_path(ps, pd)
            for mode in MODES:
                one, one_c, _, _ = csr.cheapest_k_paths(ps, pd, 1, mode=mode)
                assert [r[0] if r else None for r in one] == cpaths
                assert [r[0] if r else None for r in one_c] == [cost[i] if cvalid[i] else None for i in range(len(ps))]
            if w.dtype.kind == "i":
                paths, _, _, _ = csr.cheapest_k_paths(ps, pd, 6, mode="WALK")
                apaths, acnt, _ = csr.all_cheapest_paths(ps, pd, 6)
                assert [r if r is None else r[:min(6, c)] for r, c in zip(paths, acnt.tolist())] == apaths
            acyc, _, _, _ = csr.cheapest_k_paths(ps, pd, 6, mode="ACYCLIC")
            simp, _, _, _ = csr.cheapest_k_paths(ps, pd, 6, mode="SIMPLE")
            assert [a for a, s, t in zip(acyc, ps, pd) if s != t] == [b for b, s, t in zip(simp, ps, pd) if s != t]
        finally:
            csr.free()


@pytest.mark.gpu
def test_device_errors(ctx):
    n, src, dst, w = 4, [0, 1, 2, 1], [1, 2, 1, 3], np.array([1, 0, 0, 1], np.int64)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        for kw, status in ((dict(k=0), PGQ_ERR_INVALID_ARG), (dict(options=pgq.Options(512)), PGQ_ERR_INVALID_ARG),
                           (dict(options=pgq.Options(96)), PGQ_ERR_INVALID_ARG), (dict(dst=[9]), PGQ_ERR_RANGE)):
            args = dict(src=[0], dst=[3], k=2) | kw
            with pytest.raises(pgq.PgqError) as ei:
                csr.cheapest_k_paths(**args)
            assert ei.value.status == status
        lib = _native.load()
        npaths, first = np.zeros(1, np.int64), np.zeros(1, np.int64)
        ov = np.zeros(1, np.uint8)
        offs, elems, costs, total = C.POINTER(C.c_int64)(), C.POINTER(C.c_int64)(), C.c_void_p(), C.c_int64(0)
        p64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
        s_, d_ = np.array([0], np.int64), np.array([3], np.int64)
        args = (p64(npaths), p64(first), ov.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(offs), C.byref(elems),
                C.byref(costs), C.byref(total), None)
        assert lib.pgq_cheapest_k_paths(csr._h, 1, p64(s_), p64(d_), None, None, None, 2, 7, *args) == PGQ_ERR_INVALID_ARG
        assert lib.pgq_cheapest_k_paths(None, 1, p64(s_), p64(d_), None, None, None, 2, 0, *args) == PGQ_ERR_INVALID_ID
        opts = pgq.Options(0).c()
        opts.shard_count = 2
        assert lib.pgq_cheapest_k_paths(csr._h, 1, p64(s_), p64(d_), None, None, C.byref(opts), 2, 0,
                                        *args) == PGQ_ERR_UNSUPPORTED
        # the C ABI without costs, then with them
        assert lib.pgq_cheapest_k_paths(csr._h, 1, p64(s_), p64(d_), None, None, None, 3, 1, p64(npaths), p64(first),
                                        ov.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(offs), C.byref(elems), None,
                                        C.byref(total), None) == 0
        assert total.value == 2 and [offs[j] for j in range(3)] == [0, 5, 14]
        lib.pgq_free(offs)
        lib.pgq_free(elems)
        assert lib.pgq_cheapest_k_paths(csr._h, 1, p64(s_), p64(d_), None, None, None, 3, 1, *args) == 0
        assert [C.cast(costs, C.POINTER(C.c_int64))[j] for j in range(2)] == [2, 2]
        for x in (offs, elems, costs):
            lib.pgq_free(x)
    finally:
        csr.free()
    neg = device_csr(ctx, n, src, dst, np.array([1.0, -0.5, 0.0, 1.0]))
    try:
        with pytest.raises(pgq.PgqError) as ei:
            neg.cheapest_k_paths([0], [3], 2)
        assert ei.value.status == PGQ_ERR_UNSUPPORTED
    finally:
        neg.free()
    negz = device_csr(ctx, n, src, dst, np.array([1.0, -0.0, 0.0, 1.0]))  # -0.0 is not below zero
    try:
        assert negz.cheapest_k_paths([0], [3], 1)[1] == [[2.0]]
    finally:
        negz.free()
    plain = pgq.DeviceCSR.build(ctx, n, np.array(src), np.array(dst))
    try:
        with pytest.raises(pgq.PgqError) as ei:
            plain.cheapest_k_paths([0], [3], 2)
        assert ei.value.status == PGQ_ERR_NOT_INITIALIZED
    finally:
        plain.free()
    unfinished = pgq.DeviceCSR.create(ctx, n)  # weighted edges added, never finalised
    try:
        unfinished.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
        unfinished.add_edges(len(src), len(src), np.array(src), np.array(dst), np.arange(len(src)), w)
        with pytest.raises(pgq.PgqError) as ei:
            unfinished.cheapest_k_paths([0], [3], 2)
        assert ei.value.status == PGQ_ERR_NOT_INITIALIZED
    finally:
        unfinished.free()


@pytest.mark.gpu
def test_device_empty_null_rows_and_udf_mirror(ctx):
    n, src, dst, w = 4, [0, 1, 2, 1], [1, 2, 1, 3], np.array([1, 0, 0, 1], np.int64)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        paths, costs, npaths, st = csr.cheapest_k_paths([], [], 3)
        assert paths == [] and costs == [] and st["batches"] == 0
        paths, costs, _, _ = csr.cheapest_k_paths([0, 0, 3], [3, 3, 3], 3, [0, 1, 1], [1, 0, 1], mode="trail")
        assert paths == [None, None, [[3]]] and costs == [None, None, [0]]
        state = pgq.DuckPGQState(ctx)
        state.csr_list[0] = csr
        paths, costs = pgq.cheapest_k_paths(state, 0, n, [0], [3], 2, mode="ACYCLIC")
        assert paths == [[[0, 0, 1, 3, 3]]] and costs == [[2]] and 0 in state.csr_to_delete
        with pytest.raises(pgq.InvalidInputException):
            pgq.cheapest_k_paths(state, 0, n, [0], [3], 2, mode="SHORTEST")
        with pytest.raises(pgq.ConstraintException):
            pgq.cheapest_k_paths(state, 7, n, [0], [3], 2)
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_two_threads(ctx):
    n, src, dst, w, ps, pd, sv, dv = rmat_case(9, "f64", 40, seed=3)
    csr = device_csr(ctx, n, src, dst, w)
    try:
        single = {m: csr.cheapest_k_paths(ps, pd, 4, sv, dv, mode=m)[:2] for m in ("WALK", "TRAIL")}
        out, errs = {}, []

        def run(m):
            try:
                out[m] = csr.cheapest_k_paths(ps, pd, 4, sv, dv, mode=m)[:2]
            except Exception as x:  # noqa: BLE001 (reported below)
                errs.append(x)

        threads = [threading.Thread(target=run, args=(m,)) for m in ("WALK", "TRAIL")]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errs and out == single
    finally:
        csr.free()
