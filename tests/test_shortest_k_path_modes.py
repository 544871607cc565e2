"""shortest_k_paths in SQL/PGQ's TRAIL, ACYCLIC and SIMPLE path modes (include/duckpgq_b200.h,
pgq_shortest_k_paths_mode).

The CPU tests pin the oracle (oracle/pgq_oracle_kpaths_modes.c: Yen's algorithm with Lawler's rule, a sequential BFS
per spur search) against independent restatements: a brute-force enumeration of each mode's paths sorted by (h, steps
from t back to s); the worked examples on the reference's top_k.test / path_modes.test graph; k = 1 against
orc.shortestpath; SIMPLE against ACYCLIC for s != t; each mode's list as a prefix of the WALK oracle's walks filtered
by the mode; all_shortest_paths(max_paths = k) where a row has at least k shortest paths.  They also show that each
case of the catalogue reaches what it is named after.  The GPU tests require the device's validity, counts, lists and
batch counters to equal the oracle's.
"""
import threading

import numpy as np
import pytest

from conftest import golden_names, load_golden
from duckpgq_extension_b200 import datagen, pgq
from duckpgq_extension_b200.pgq import (PGQ_ERR_INVALID_ARG, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_RANGE,
                                        PGQ_ERR_UNSUPPORTED, PGQ_PATH_ACYCLIC, PGQ_PATH_SIMPLE, PGQ_PATH_TRAIL,
                                        PGQ_PATH_WALK)
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_kpaths_modes as okm
from oracle import pgq_oracle_kshortest as oks

MODES = ("TRAIL", "ACYCLIC", "SIMPLE")
COUNTERS = ("batches", "lanes", "searches", "levels")
PATH_MAX = 65533
# the reference's top_k.test / path_modes.test graph, edges in rowid order
TOPK = {"n": 5, "src": [0, 0, 0, 3, 1, 1, 2, 4], "dst": [1, 2, 3, 0, 2, 3, 3, 3]}


def ref_csr(n, src, dst, eid=None):
    return orc.csr_build(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), eid)


def admits(mode, path):
    """whether the list [s, e1, v1, ..., t] (edge ids unique per adjacency entry) is a path of the mode"""
    verts, edges = path[0::2], path[1::2]
    if mode == "TRAIL":
        return len(set(edges)) == len(edges)
    if mode == "SIMPLE" and len(verts) > 1 and verts[0] == verts[-1]:
        return len(set(verts[:-1])) == len(verts) - 1
    return len(set(verts)) == len(verts)


def brute_paths(n, v, e, ids, s, t, mode):
    """every path s -> t of the mode, sorted by (h, steps from t back to s), a step being (parent, the edge's
    position in the parent's adjacency)"""
    out = []

    def walk(u, elems, steps, used, visited):
        if u == t:
            out.append(((len(steps), list(reversed(steps))), list(elems)))
            if mode != "TRAIL" and (len(steps) > 0 or mode == "ACYCLIC" or s != t):
                return
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            if mode == "TRAIL":
                if idx in used:
                    continue
            elif w in visited and not (mode == "SIMPLE" and w == s == t):
                continue
            walk(w, elems + [int(ids[idx]), w], steps + [(u, idx - int(v[u]))], used | {idx}, visited | {w})

    walk(s, [s], [], frozenset(), frozenset([s]))
    return [el for _, el in sorted(out, key=lambda x: x[0])]


def random_multigraph(seed, n_hi=8, m_hi=13):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, n_hi))
    m = int(rng.integers(0, m_hi))
    src, dst = rng.integers(0, n, m), rng.integers(0, n, m)
    if m > 2:  # a parallel edge and a self-loop
        src[1], dst[1] = src[0], dst[0]
        dst[2] = src[2]
    return n, src.astype(np.int64), dst.astype(np.int64)


def all_rows(n):
    ps, pd = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    return ps.ravel().astype(np.int64), pd.ravel().astype(np.int64)


# ---- the oracle against brute force and the worked examples ----------------------------------------------------------
@pytest.mark.parametrize("seed", range(60))
def test_oracle_is_the_brute_force_enumeration(seed):
    n, src, dst = random_multigraph(seed)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = all_rows(n)
    for mode in MODES:
        brute = [brute_paths(n, v, e, ids, int(s), int(t), mode) for s, t in zip(ps, pd)]
        for k in (1, 2, 3, 5, 10):
            paths, npaths, _ = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, k, mode)
            for i in range(len(ps)):
                exp = brute[i][:k]
                assert (paths[i] or []) == exp, (mode, k, int(ps[i]), int(pd[i]))
                assert npaths[i] == len(exp)


def test_worked_examples():
    v, e, ids = ref_csr(TOPK["n"], TOPK["src"], TOPK["dst"])
    four = [[0, 2, 3], [0, 0, 1, 5, 3], [0, 1, 2, 6, 3], [0, 0, 1, 4, 2, 6, 3]]
    cycles = [[0], [0, 2, 3, 3, 0], [0, 0, 1, 5, 3, 3, 0], [0, 1, 2, 6, 3, 3, 0], [0, 0, 1, 4, 2, 6, 3, 3, 0]]

    def run(s, t, mode, k=5):
        return okm.shortest_k_paths_mode(5, v, e, ids, [s], [t], k, mode)[0][0]

    assert run(0, 3, "ACYCLIC") == four and run(0, 3, "SIMPLE") == four
    assert run(0, 3, "TRAIL") == four + [[0, 0, 1, 5, 3, 3, 0, 2, 3]]
    assert len(run(0, 3, "TRAIL", 100)) == 12
    assert run(0, 0, "ACYCLIC") == [[0]]
    assert run(0, 0, "SIMPLE") == cycles and run(0, 0, "TRAIL") == cycles
    assert run(4, 3, "ACYCLIC") == [[4, 7, 3]]
    assert run(4, 3, "TRAIL") == [[4, 7, 3], [4, 7, 3, 3, 0, 2, 3], [4, 7, 3, 3, 0, 0, 1, 5, 3],
                                  [4, 7, 3, 3, 0, 1, 2, 6, 3], [4, 7, 3, 3, 0, 0, 1, 4, 2, 6, 3]]
    # WALK fills up with cycles where the modes do not
    walks = oks.shortest_k_paths(5, v, e, ids, [0], [3], 5)[0][0]
    assert walks[3] == [0, 2, 3, 3, 0, 2, 3]


# ---- restatements ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(20))
def test_restatements(seed):
    n, src, dst = random_multigraph(1000 + seed, n_hi=7, m_hi=11)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = all_rows(n)
    sp, _ = orc.shortestpath(n, v, e, ids, ps, pd)
    walks, _, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, 300)
    res = {}
    for mode in MODES:
        one, _, _ = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, 1, mode)
        assert [None if p is None else p[0] for p in one] == sp  # k = 1 is shortestpath's path
        res[mode], _, _ = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, 8, mode)
        for i in range(len(ps)):  # a prefix of the walks filtered by the mode
            got = res[mode][i] or []
            filt = [w for w in (walks[i] or []) if admits(mode, w)]
            r = min(len(got), len(filt))
            assert got[:r] == filt[:r]
    cnt = oas.shortest_path_count(n, v, e, ids, ps, pd)[0]
    ap = oas.all_shortest_paths(n, v, e, ids, ps, pd, 8)[0]
    for i in range(len(ps)):
        if ps[i] != pd[i]:
            assert res["SIMPLE"][i] == res["ACYCLIC"][i]
        else:
            assert res["ACYCLIC"][i] == [[int(ps[i])]]
        for mode in MODES:
            if cnt[i] >= 8 and not (ps[i] == pd[i] and mode != "ACYCLIC"):
                assert res[mode][i] == ap[i]


def test_all_shortest_prefix_on_a_diamond_chain():
    # 4 diamonds in a row: 16 shortest paths, so every mode's first 16 are all_shortest_paths'
    src, dst = [], []
    for d in range(4):
        a = 3 * d
        src += [a, a, a + 1, a + 2]
        dst += [a + 1, a + 2, a + 3, a + 3]
    src += [12]
    dst += [0]  # a cycle back, so WALK has more
    n = 13
    v, e, ids = ref_csr(n, src, dst)
    ap = oas.all_shortest_paths(n, v, e, ids, [0], [12], 16)[0][0]
    assert len(ap) == 16
    for mode in MODES:
        assert okm.shortest_k_paths_mode(n, v, e, ids, [0], [12], 16, mode)[0][0] == ap


# ---- the catalogue ---------------------------------------------------------------------------------------------------
def case_cycle_behind_chain():  # 0 -> 1 -> 2 -> 3, with the cycle 1 -> 4 -> 1 behind the chain's head
    return {"n": 5, "src": [0, 1, 2, 1, 4], "dst": [1, 2, 3, 4, 1], "ps": [0, 1], "pd": [3, 3], "ks": [3, 6]}


def case_trail_through_t():  # 0 -> 1 -> 2 -> 3 -> 1: a trail reaches t = 1 and comes back
    return {"n": 4, "src": [0, 1, 2, 3], "dst": [1, 2, 3, 1], "ps": [0, 1], "pd": [1, 1], "ks": [3]}


def case_parallel_twice():  # two 0 -> 1 and two 1 -> 0
    return {"n": 2, "src": [0, 0, 1, 1], "dst": [1, 1, 0, 0], "ps": [0, 0, 1], "pd": [1, 0, 1], "ks": [4, 10]}


def case_self_loops():  # self-loops at s = 0, the spur node 1 and t = 2
    return {"n": 3, "src": [0, 0, 1, 1, 2, 1], "dst": [0, 1, 1, 2, 2, 0], "ps": [0, 0, 1], "pd": [2, 0, 1],
            "ks": [3, 8]}


def case_duplicated_source():  # the same source in several rows, which take a lane each
    rng = np.random.default_rng(5)
    n = 30
    src, dst = rng.integers(0, n, 90), rng.integers(0, n, 90)
    return {"n": n, "src": src.tolist(), "dst": dst.tolist(), "ps": [3] * 12, "pd": list(range(12)), "ks": [4]}


def case_wide_spur():  # 0 -> 1 .. 40 -> 41: the spur node 0 has out-degree 40
    src = [0] * 40 + list(range(1, 41))
    dst = list(range(1, 41)) + [41] * 40
    return {"n": 42, "src": src, "dst": dst, "ps": [0], "pd": [41], "ks": [5, 36, 45]}


def case_null_unreachable():  # rows with a NULL id, an unreachable target, an isolated vertex
    return {"n": 5, "src": [0, 1, 2], "dst": [1, 2, 0], "ps": [0, 9, 0, 4, 4, 3], "pd": [2, 1, 9, 0, 4, 3],
            "sv": [1, 0, 1, 1, 1, 1], "dv": [1, 1, 0, 1, 1, 1], "ks": [2]}


def case_exhausted():  # k above every row's total
    return {"n": 4, "src": [0, 0, 1, 2, 2], "dst": [1, 2, 3, 3, 1], "ps": [0, 0, 2], "pd": [3, 1, 3], "ks": [50]}


def case_rows(p, seed=3):  # p rows with s != t and a source with out-edges: round 0 has p searches
    rng = np.random.default_rng(seed)
    n = 200
    src, dst = rng.integers(0, n, 1200), rng.integers(0, n, 1200)
    srcs = np.unique(src)
    ps = rng.choice(srcs, p)
    pd = (ps + 1 + rng.integers(0, n - 1, p)) % n
    return {"n": n, "src": src.tolist(), "dst": dst.tolist(), "ps": ps.tolist(), "pd": pd.tolist(), "ks": [1, 3]}


CATALOGUE = {
    "cycle_behind_chain": case_cycle_behind_chain,
    "trail_through_t": case_trail_through_t,
    "parallel_twice": case_parallel_twice,
    "self_loops": case_self_loops,
    "duplicated_source": case_duplicated_source,
    "wide_spur": case_wide_spur,
    "null_unreachable": case_null_unreachable,
    "exhausted": case_exhausted,
    **{f"rows{p}": (lambda p=p: case_rows(p)) for p in (63, 64, 65, 511, 512, 513)},
}


def run_oracle(c, k, mode, lanes=0):
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    return okm.shortest_k_paths_mode(c["n"], v, e, ids, c["ps"], c["pd"], k, mode, c.get("sv"), c.get("dv"), lanes)


def test_catalogue_cycle_behind_chain():
    c = case_cycle_behind_chain()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    walks = oks.shortest_k_paths(5, v, e, ids, [0], [3], 3)[0][0]
    assert any(4 in w[0::2] for w in walks)
    for mode in ("ACYCLIC", "SIMPLE"):
        assert run_oracle(c, 6, mode)[0][0] == [[0, 0, 1, 1, 2, 2, 3]]
    assert run_oracle(c, 6, "TRAIL")[0][0] == [[0, 0, 1, 1, 2, 2, 3], [0, 0, 1, 3, 4, 4, 1, 1, 2, 2, 3]]


def test_catalogue_trail_through_t():
    paths = run_oracle(case_trail_through_t(), 3, "TRAIL")[0]
    assert paths[0] == [[0, 0, 1], [0, 0, 1, 1, 2, 2, 3, 3, 1]]
    assert paths[1] == [[1], [1, 1, 2, 2, 3, 3, 1]]
    assert run_oracle(case_trail_through_t(), 3, "ACYCLIC")[0][0] == [[0, 0, 1]]


def test_catalogue_parallel_edges_twice():
    paths = run_oracle(case_parallel_twice(), 10, "TRAIL")[0]
    # 0 -a-> 1 -c-> 0 -b-> 1: both parallel 0 -> 1 edges in one trail
    assert [0, 0, 1, 2, 0, 1, 1] in paths[0]
    assert all(len(set(p[1::2])) == len(p[1::2]) for p in paths[0])
    assert len(run_oracle(case_parallel_twice(), 10, "ACYCLIC")[0][0]) == 2


def test_catalogue_self_loops():
    c = case_self_loops()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    trail = run_oracle(c, 8, "TRAIL")[0]
    loops = {int(ids[v[u]]) for u in range(3) if int(e[v[u]]) == u}  # each vertex's self-loop
    assert len(loops) == 3
    for lp in loops:
        assert any(lp in p[1::2] for p in trail[0])
    assert [0, int(ids[v[0]]), 0] in run_oracle(c, 8, "SIMPLE")[0][1]  # a self-loop on s is a simple cycle
    assert run_oracle(c, 8, "ACYCLIC")[0][1] == [[0]]


def test_catalogue_undirected_trail_goes_back():
    # an undirected CSR: both directions of an edge, one rowid, two adjacency entries
    v, e, ids = ref_csr(2, [0, 1], [1, 0], np.array([7, 7]))
    paths = okm.shortest_k_paths_mode(2, v, e, ids, [0], [0], 5, "TRAIL")[0][0]
    assert paths == [[0], [0, 7, 1, 7, 0]]


def test_catalogue_duplicated_source_and_wide_spur():
    c = case_duplicated_source()
    paths, _, st = run_oracle(c, 4, "ACYCLIC")
    assert st["searches"] > len(c["ps"]) - 1
    one, _, _ = run_oracle({**c, "ps": [3], "pd": [5]}, 4, "ACYCLIC")
    assert paths[5] == one[0]
    c = case_wide_spur()
    paths, _, _ = run_oracle(c, 45, "ACYCLIC")
    assert len(paths[0]) == 40 and paths[0][39] == [0, 39, 40, 79, 41]


def test_catalogue_nulls_and_exhausted():
    paths, npaths, _ = run_oracle(case_null_unreachable(), 2, "TRAIL")
    assert paths[:4] == [[[0, 0, 1, 1, 2]], None, None, None] and paths[4] == [[4]] and npaths[1] == 0
    for mode in MODES:
        paths, npaths, _ = run_oracle(case_exhausted(), 50, mode)
        assert npaths.tolist() == [3, 2, 2] and paths[1] == [[0, 0, 1], [0, 1, 2, 4, 1]]


@pytest.mark.parametrize("p", [63, 64, 65, 511, 512, 513])
def test_catalogue_round_sizes(p):
    c = case_rows(p)
    _, npaths, st = run_oracle(c, 1, "ACYCLIC")
    assert st["searches"] == p and (npaths == 1).all()  # round 0: one search per row
    w = 512 if p > 256 else (256 if p > 128 else (128 if p > 64 else 64))
    assert st["lanes"] == w and st["batches"] == -(-p // w)
    _, _, st = run_oracle(c, 1, "TRAIL", lanes=64)
    assert st["batches"] == -(-p // 64)


def test_catalogue_path_limit():
    n = PATH_MAX + 2
    src, dst = np.arange(n - 1), np.arange(1, n)
    v, e, ids = ref_csr(n, src, dst)
    paths, _, _ = okm.shortest_k_paths_mode(n, v, e, ids, [0], [PATH_MAX], 3, "ACYCLIC")
    assert len(paths[0]) == 1 and (len(paths[0][0]) - 1) // 2 == PATH_MAX
    with pytest.raises(orc.OracleError) as ex:
        okm.shortest_k_paths_mode(n, v, e, ids, [0], [PATH_MAX + 1], 1, "TRAIL")
    assert ex.value.code == okm.ERR_UNSUPPORTED


def test_oracle_errors():
    v, e, ids = ref_csr(3, [0, 1], [1, 2])
    for args, code in ((([0], [1], 0, "TRAIL"), okm.ERR_ARG), (([0], [1], 1, "WALK"), okm.ERR_ARG),
                       (([0], [3], 1, "TRAIL"), okm.ERR_RANGE)):
        with pytest.raises(orc.OracleError) as ex:
            okm.shortest_k_paths_mode(3, v, e, ids, *args)
        assert ex.value.code == code


# ---- GPU: the device against the oracle ------------------------------------------------------------------------------
def compare(csr, n, v, e, ids, ps, pd, k, mode, sv=None, dv=None, options=None):
    paths, npaths, st = csr.shortest_k_paths(ps, pd, k, sv, dv, options, mode=mode)
    lanes = options.lanes if options else 0
    opaths, onp, ost = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, k, mode, sv, dv, lanes)
    assert np.array_equal(npaths, onp)
    assert paths == opaths
    assert {x: st[x] for x in COUNTERS} == {x: ost[x] for x in COUNTERS}
    return paths, st


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    c = CATALOGUE[name]()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))
    for mode in MODES:
        for k in sorted(set(c["ks"])) + [1]:
            compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], k, mode, c.get("sv"), c.get("dv"))
    csr.free()


@pytest.mark.gpu
def test_device_worked_examples_and_undirected(gpu_ctx):
    csr = pgq.DeviceCSR.build(gpu_ctx, 5, np.array(TOPK["src"]), np.array(TOPK["dst"]))
    paths, _, _ = csr.shortest_k_paths([0, 0, 4], [3, 0, 3], 5, mode="trail")
    assert paths[0][4] == [0, 0, 1, 5, 3, 3, 0, 2, 3] and paths[1][1] == [0, 2, 3, 3, 0]
    assert paths[2][1] == [4, 7, 3, 3, 0, 2, 3]
    csr.free()
    vk = np.array([10, 20, 30], np.int64)
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, vk, np.array([10, 20]), np.array([20, 30]), undirected=True)
    kv, ke, kids = csr.download()
    paths, _ = compare(csr, 3, kv, ke, kids, [0, 1], [0, 1], 6, "TRAIL")
    assert any(p[0::2][:3] == [0, 1, 0] for p in paths[0])  # u -> v -> u over one undirected edge
    csr.free()


@pytest.mark.gpu
def test_device_path_limit(gpu_ctx):
    n = PATH_MAX + 2
    src, dst = np.arange(n - 1), np.arange(1, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    paths, _ = compare(csr, n, v, e, ids, [0], [PATH_MAX], 3, "ACYCLIC")
    assert (len(paths[0][0]) - 1) // 2 == PATH_MAX
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_paths([0], [PATH_MAX + 1], 1, mode="TRAIL")
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names())
def test_device_reference_graphs(gpu_ctx, name):
    g = load_golden(name)
    n = g["n"]
    v, e, ids = ref_csr(n, g["src"], g["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, n, g["src"], g["dst"])
    sv = g["psrc_valid"].astype(np.uint8)
    for mode in MODES:
        for k in (1, 5):
            compare(csr, n, v, e, ids, g["psrc"][:300], g["pdst"][:300], k, mode, sv[:300])
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [12, 14])
def test_device_rmat(gpu_ctx, scale):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(512 if scale == 12 else 256, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    sp, _ = csr.shortestpath(ps, pd)
    for mode in MODES:
        for k in (1, 4, 16):
            paths, _ = compare(csr, n, v, e, ids, ps, pd, k, mode)
            if k == 1:
                assert [None if x is None else x[0] for x in paths] == sp
    csr.free()


@pytest.mark.gpu
def test_device_rmat16_all_shortest_prefix(gpu_ctx):
    n, src, dst = datagen.rmat_edges(16)
    ps, pd = datagen.hashed_pairs(512, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    k = 6
    ap, cnt, _ = csr.all_shortest_paths(ps, pd, k)
    for mode in ("TRAIL", "ACYCLIC"):
        paths, _, _ = csr.shortest_k_paths(ps, pd, k, mode=mode)
        hits = [i for i in range(len(ps)) if cnt[i] >= k and ps[i] != pd[i]]
        assert len(hits) > 20
        assert all(paths[i] == ap[i] for i in hits)
        pick = np.arange(0, len(ps), 37)
        opaths, _, _ = okm.shortest_k_paths_mode(n, v, e, ids, ps[pick], pd[pick], k, mode)
        assert [paths[i] for i in pick] == opaths
    csr.free()


@pytest.mark.gpu
def test_device_lane_widths_and_row_order(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(700, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    for mode in ("TRAIL", "ACYCLIC"):
        base, _ = compare(csr, n, v, e, ids, ps, pd, 5, mode)
        for lanes in range(64, 513, 64):
            paths, st = compare(csr, n, v, e, ids, ps, pd, 5, mode, options=pgq.Options(lanes))
            assert paths == base and st["lanes"] == lanes
        perm = np.random.default_rng(1).permutation(len(ps))
        paths, _, _ = csr.shortest_k_paths(ps[perm], pd[perm], 5, mode=mode)
        assert paths == [base[i] for i in perm]
    csr.free()


@pytest.mark.gpu
def test_device_construction_routes(gpu_ctx):
    import torch
    n, src, dst = datagen.rmat_edges(10)
    ps, pd = datagen.hashed_pairs(300, n)
    v, e, ids = ref_csr(n, src, dst)
    for csr in (pgq.DeviceCSR.build(gpu_ctx, n, src, dst), pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)):
        for mode in MODES:
            compare(csr, n, v, e, ids, ps, pd, 4, mode)
        csr.free()
    vk = np.random.default_rng(4).permutation(n).astype(np.int64) * 3
    cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (vk, vk[src], vk[dst])]
    routes = [pgq.DeviceCSR.build_from_keys(gpu_ctx, vk, vk[src], vk[dst], undirected=u) for u in (False, True)]
    routes.append(pgq.DeviceCSR.build_from_keys_device(gpu_ctx, n, len(src), *(c.data_ptr() for c in cols)))
    for csr in routes:
        kv, ke, kids = csr.download()
        for mode in MODES:
            compare(csr, csr.n, kv, ke, kids, ps % csr.n, pd % csr.n, 4, mode)
        csr.free()


@pytest.mark.gpu
def test_device_walk_mode_is_shortest_k_paths(gpu_ctx):
    import ctypes as C
    from duckpgq_extension_b200 import _native
    lib = _native.load()
    n, src, dst = datagen.rmat_edges(11)
    ps, pd = datagen.hashed_pairs(300, n)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    out = []
    for fn, extra in ((lib.pgq_shortest_k_paths, ()), (lib.pgq_shortest_k_paths_mode, (PGQ_PATH_WALK,))):
        npw, first, valid = np.zeros(len(ps), np.int64), np.zeros(len(ps), np.int64), np.zeros(len(ps), np.uint8)
        offs, elems, total = p64(), p64(), C.c_int64(0)
        st = _native.PgqStats()
        assert fn(csr._h, len(ps), ps.ctypes.data_as(p64), pd.ctypes.data_as(p64), None, None, None, 9, *extra,
                  npw.ctypes.data_as(p64), first.ctypes.data_as(p64), valid.ctypes.data_as(pu8), C.byref(offs),
                  C.byref(elems), C.byref(total), C.byref(st)) == 0
        o = [offs[j] for j in range(total.value + 1)]
        flat = [elems[j] for j in range(o[-1])]
        lib.pgq_free(offs)
        lib.pgq_free(elems)
        d = st.as_dict()
        out.append((npw.tolist(), first.tolist(), valid.tolist(), o, flat,
                    {x: d[x] for x in ("batches", "lanes", "searches", "levels", "push_levels", "kernel_launches")}))
    assert out[0] == out[1]
    v, e, ids = ref_csr(n, src, dst)
    assert csr.shortest_k_paths(ps, pd, 9, mode="walk")[0] == oks.shortest_k_paths(n, v, e, ids, ps, pd, 9)[0]
    csr.free()


@pytest.mark.gpu
def test_device_errors(gpu_ctx):
    import ctypes as C
    from duckpgq_extension_b200 import _native
    lib = _native.load()
    csr = pgq.DeviceCSR.build(gpu_ctx, 4, np.array([0, 1, 2]), np.array([1, 2, 0]))
    p64 = C.POINTER(C.c_int64)
    src, dst = np.array([0], np.int64), np.array([1], np.int64)
    npw, first, valid = np.zeros(1, np.int64), np.zeros(1, np.int64), np.zeros(1, np.uint8)
    offs, elems, total = p64(), p64(), C.c_int64(0)
    for bad in (4, -1):
        assert lib.pgq_shortest_k_paths_mode(csr._h, 1, src.ctypes.data_as(p64), dst.ctypes.data_as(p64), None, None,
                                             None, 2, bad, npw.ctypes.data_as(p64), first.ctypes.data_as(p64),
                                             valid.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(offs),
                                             C.byref(elems), C.byref(total), None) == PGQ_ERR_INVALID_ARG
    with pytest.raises(pgq.InvalidInputException):
        csr.shortest_k_paths([0], [1], 2, mode="cheapest")
    for mode in MODES:
        for call, status in ((lambda: csr.shortest_k_paths([0, 4], [1, 1], 2, mode=mode), PGQ_ERR_RANGE),
                             (lambda: csr.shortest_k_paths([0], [1], 0, mode=mode), PGQ_ERR_INVALID_ARG),
                             (lambda: csr.shortest_k_paths([0], [1], 2, options=pgq.Options(96), mode=mode),
                              PGQ_ERR_INVALID_ARG),
                             (lambda: csr.shortest_k_paths([0], [1], 2, options=pgq.Options(
                                 0, shard_index=0, shard_count=2), mode=mode), PGQ_ERR_UNSUPPORTED)):
            with pytest.raises(pgq.PgqError) as ex:
                call()
            assert ex.value.status == status
        paths, npaths, _ = csr.shortest_k_paths([0, 9], [9, 1], 3, [1, 0], [0, 1], mode=mode)
        assert paths == [None, None] and npaths.tolist() == [0, 0]
        paths, _, st = csr.shortest_k_paths([], [], 3, mode=mode)
        assert paths == [] and st["batches"] == 0
    csr.free()
    un = pgq.DeviceCSR.create(gpu_ctx, 3)
    with pytest.raises(pgq.PgqError) as ex:
        un.shortest_k_paths([0], [1], 2, mode="ACYCLIC")
    assert ex.value.status == PGQ_ERR_NOT_INITIALIZED
    un.free()


@pytest.mark.gpu
def test_udf_mirror(gpu_ctx):
    state = pgq.DuckPGQState(gpu_ctx)
    pgq.create_csr_vertex(state, 0, 4, np.arange(4), np.array([2, 1, 1, 1]))
    pgq.create_csr_edge(state, 0, 4, 5, 5, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], [10, 11, 12, 13, 14])
    paths = pgq.shortest_k_paths(state, 0, 4, [0, 0], [3, 0], 5, mode="acyclic")
    assert paths == [[[0, 10, 1, 12, 3], [0, 11, 2, 13, 3]], [[0]]]
    v, e, ids = ref_csr(4, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], np.arange(10, 15))
    assert pgq.shortest_k_paths(state, 0, 4, [0, 0], [3, 0], 5, mode="TRAIL") == \
        okm.shortest_k_paths_mode(4, v, e, ids, [0, 0], [3, 0], 5, "TRAIL")[0]
    with pytest.raises(pgq.InvalidInputException):
        pgq.shortest_k_paths(state, 0, 4, [0], [3], 5, mode="ANY")
    state.query_end()


@pytest.mark.gpu
def test_one_workspace_in_turn(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(300, n)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    alone = (csr.shortest_k_paths(ps, pd, 8, mode="TRAIL")[0], csr.shortest_k_paths(ps, pd, 8)[0],
             csr.all_shortest_paths(ps, pd, 8)[0])
    for _ in range(2):
        km = csr.shortest_k_paths(ps, pd, 8, mode="TRAIL")[0]
        ks = csr.shortest_k_paths(ps, pd, 8)[0]
        ap = csr.all_shortest_paths(ps, pd, 8)[0]
        assert km == alone[0] and ks == alone[1] and ap == alone[2]
    csr.free()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(200, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    exp = {m: okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, 6, m)[0] for m in MODES}
    out = [None] * 8

    def work(i):
        out[i] = csr.shortest_k_paths(ps, pd, 6, mode=MODES[i % 3])[0]

    ths = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(out[i] == exp[MODES[i % 3]] for i in range(8))


def test_path_mode_ids():
    assert (PGQ_PATH_WALK, PGQ_PATH_TRAIL, PGQ_PATH_ACYCLIC, PGQ_PATH_SIMPLE) == (0, 1, 2, 3)
    assert pgq.path_mode_id("Simple") == PGQ_PATH_SIMPLE
    with pytest.raises(pgq.InvalidInputException):
        pgq.path_mode_id("shortest")
