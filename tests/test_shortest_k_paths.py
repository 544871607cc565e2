"""shortest_k_paths: the k shortest walks of a row, SQL/PGQ's SHORTEST k (include/duckpgq_b200.h, pgq_shortest_k_paths).

The CPU tests pin the oracle (oracle/pgq_oracle_kshortest.c: one row at a time, backward reach, layered saturating
counts, a depth-first enumeration in step order) against independent restatements: the per-length counts are
(A^h)[s, t] in Python integers; on small graphs the lists are the walks a brute-force search finds, sorted by (h, step
key); the issue's worked examples; prefixes equal oracle/pgq_oracle_allshortest.c's paths for k <= count; walk 0 is
orc.shortestpath's path.  They also show that each case of the catalogue reaches what it is named after.  The GPU
tests require the device's validity, counts, lists and batch counters to equal the oracle's.
"""
import threading

import numpy as np
import pytest

from conftest import golden_names, load_golden
from duckpgq_extension_b200 import datagen, pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_INVALID_ARG, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_RANGE
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_kshortest as oks

PGQ_ERR_UNSUPPORTED = 8
INT64_MAX = (1 << 63) - 1
WALK_MAX = 65533
COUNTERS = ("batches", "lanes", "searches", "levels", "push_levels")


# ---- independent restatements ----------------------------------------------------------------------------------------
def ref_csr(n, src, dst, eid=None):
    return orc.csr_build(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), eid)


def length_counts(n, v, e, s, t, hmax):
    """[(A^h)[s, t] for h = 0 .. hmax] with Python integers"""
    vec = [0] * n
    vec[s] = 1
    out = [vec[t]]
    for _ in range(hmax):
        nxt = [0] * n
        for u in range(n):
            if vec[u]:
                for idx in range(v[u], v[u + 1]):
                    nxt[int(e[idx])] += vec[u]
        vec = nxt
        out.append(vec[t])
    return out


def reaches(n, v, e, s, t):
    seen, q = {s}, [s]
    for u in q:
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            if w not in seen:
                seen.add(w)
                q.append(w)
    return t in seen


def brute_walks(n, v, e, ids, s, t, hmax):
    """every walk s -> t of at most hmax edges, sorted by (h, steps from t back to s), a step being (parent, the
    edge's position in the parent's adjacency)"""
    walks = []

    def walk(u, k, elems, steps):
        if u == t:
            walks.append(((k, list(reversed(steps))), list(elems)))
        if k == hmax:
            return
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            walk(w, k + 1, elems + [int(ids[idx]), w], steps + [(u, idx - int(v[u]))])

    walk(s, 0, [s], [])
    return [el for _, el in sorted(walks, key=lambda x: x[0])]


def random_multigraph(seed, n_lo=4, n_hi=8):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(n_lo, n_hi))
    m = int(rng.integers(n, 2 * n + 2))
    src = rng.integers(0, n, m)
    dst = rng.integers(0, n, m)
    k = m // 5
    src = np.concatenate([src, src[:k]])
    dst = np.concatenate([dst, dst[:k]])
    return n, src, dst


def diamonds(k):
    """k diamonds in a row: 2^k paths of 2k edges from x_0 = 0 to x_k = 3k"""
    src, dst = [], []
    for i in range(k):
        x, a, b, y = 3 * i, 3 * i + 1, 3 * i + 2, 3 * i + 3
        src += [x, x, a, b]
        dst += [a, b, y, y]
    return 3 * k + 1, np.array(src), np.array(dst)


def cycle_with_tail(c, d):
    """a cycle 0 -> 1 -> ... -> c - 1 -> 0: the walks 0 -> d have lengths d, d + c, d + 2c, ..."""
    return c, np.arange(c), (np.arange(c) + 1) % c


TOPK = dict(n=5, src=[0, 0, 0, 3, 1, 1, 2, 4], dst=[1, 2, 3, 0, 2, 3, 3, 3])  # the reference's top_k.test graph


# ---- the catalogue ---------------------------------------------------------------------------------------------------
def case_crossing():
    """0 -> 1 -> 3, 0 -> 2 -> 3, 3 -> 0: two walks of 2 edges, then 3 -> 0 -> x -> 3 adds walks of 5 edges"""
    return dict(n=4, src=[0, 0, 1, 2, 3], dst=[1, 2, 3, 3, 0], ps=[0, 0, 0], pd=[3, 3, 3], ks=[1, 2, 3])


def case_bipartite():
    """a 4-cycle with a chord both ways: a bipartite graph, walks only of even lengths between its sides' vertices"""
    return dict(n=4, src=[0, 1, 2, 3, 0, 2], dst=[1, 2, 3, 0, 3, 1], ps=[0, 0], pd=[2, 0], ks=[7, 7])


def case_dag():
    """a DAG with 3 walks 0 -> 4, asked for 10"""
    return dict(n=5, src=[0, 0, 1, 2, 0, 3], dst=[1, 2, 4, 4, 3, 4], ps=[0], pd=[4], ks=[10])


def case_trap():
    """0 -> 1, 1 -> 1 (a self-loop that does not reach 2), 0 -> 2: one walk, and the count at 1 never dies out"""
    return dict(n=3, src=[0, 1, 0], dst=[1, 1, 2], ps=[0], pd=[2], ks=[5])


def case_long_chain_cycle():
    """a chain 0 -> 1 -> ... -> 40, then a 3-cycle 40 -> 41 -> 42 -> 40, and 40 -> 43: walks of 41, 44, 47, ..."""
    src = list(range(40)) + [40, 41, 42, 40]
    dst = list(range(1, 41)) + [41, 42, 40, 43]
    return dict(n=44, src=src, dst=dst, ps=[0, 0], pd=[43, 40], ks=[4, 3])


def case_parallel_loops():
    """two parallel edges 0 -> 1, self-loops at the source 0 and the target 1 (twice at 1)"""
    return dict(n=2, src=[0, 0, 0, 1, 1], dst=[1, 1, 0, 1, 1], ps=[0, 0], pd=[1, 0], ks=[9, 3])


def case_same_vertex():
    """s == t with a cycle through s (0 <-> 1) and without one (2 -> 0)"""
    return dict(n=3, src=[0, 1, 2], dst=[1, 0, 0], ps=[0, 2, 2], pd=[0, 2, 2], ks=[4, 1, 4])


def case_hub_ties():
    """0 -> parents 1..8 -> 9 -> 0, parent i with i more edges into sinks: the device numbers the parents by
    descending degree, opposite to their ids, and the walks must come in the order of the ORIGINAL ids"""
    src, dst = [9], [0]
    for i in range(1, 9):
        src += [0, i]
        dst += [i, 9]
    sink = 10
    for i in range(1, 9):
        for _ in range(i):
            src.append(i)
            dst.append(sink)
            sink += 1
    return dict(n=sink, src=src, dst=dst, ps=[0, 0], pd=[9, 0], ks=[12, 10])


def case_specials():
    """NULL source, NULL destination, an unreachable row, a valid one"""
    return dict(n=5, src=[0, 1, 2, 3], dst=[1, 2, 0, 3], ps=[0, 1, 4, 0, 2], pd=[2, 2, 0, 1, 1],
                sv=[1, 0, 1, 1, 1], dv=[1, 1, 1, 0, 1], ks=[3] * 5)


def case_edgeless():
    return dict(n=4, src=[], dst=[], ps=[0, 1, 2], pd=[0, 2, 2], ks=[3, 3, 1])


def case_rows(p, seed=5):
    rng = np.random.default_rng(seed)
    n = 40
    src, dst = rng.integers(0, n, 90), rng.integers(0, n, 90)
    r = np.random.default_rng(p)
    return dict(n=n, src=src, dst=dst, ps=r.integers(0, n, p), pd=r.integers(0, n, p), ks=[7] * p)


CATALOGUE = {
    "crossing": case_crossing,
    "bipartite": case_bipartite,
    "dag": case_dag,
    "trap": case_trap,
    "long_chain_cycle": case_long_chain_cycle,
    "parallel_loops": case_parallel_loops,
    "same_vertex": case_same_vertex,
    "hub_ties": case_hub_ties,
    "specials": case_specials,
    "edgeless": case_edgeless,
    **{f"rows{p}": (lambda p=p: case_rows(p)) for p in (1, 63, 64, 65, 513)},
}


def run_oracle(c, k, lanes=64, ps=None, pd=None):
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    return oks.shortest_k_paths(c["n"], v, e, ids, c["ps"] if ps is None else ps, c["pd"] if pd is None else pd, k,
                                c.get("sv"), c.get("dv"), lanes)


def per_row(c, fn):
    """the case's rows one by one with their own k (a call has one k)"""
    return [fn(i, k) for i, k in enumerate(c["ks"])]


# ---- CPU: the oracle against the restatements ------------------------------------------------------------------------
def test_worked_examples():
    v, e, ids = ref_csr(TOPK["n"], TOPK["src"], TOPK["dst"])
    paths, npaths, _ = oks.shortest_k_paths(5, v, e, ids, [0], [3], 5)
    assert paths[0] == [[0, 2, 3], [0, 0, 1, 5, 3], [0, 1, 2, 6, 3], [0, 2, 3, 3, 0, 2, 3], [0, 0, 1, 4, 2, 6, 3]]
    paths, _, _ = oks.shortest_k_paths(5, v, e, ids, [4], [0], 3)
    assert paths[0] == [[4, 7, 3, 3, 0], [4, 7, 3, 3, 0, 2, 3, 3, 0], [4, 7, 3, 3, 0, 0, 1, 5, 3, 3, 0]]
    paths, npaths, _ = oks.shortest_k_paths(5, v, e, ids, [0], [4], 4)
    assert paths == [None] and npaths.tolist() == [0]


@pytest.mark.parametrize("seed", range(12))
def test_oracle_lists_are_the_brute_force_walks(seed):
    n, src, dst = random_multigraph(300 + seed)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = np.repeat(np.arange(n), n), np.tile(np.arange(n), n)
    for k in (1, 3, 8):
        paths, npaths, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, k)
        for i in range(len(ps)):
            s, t = int(ps[i]), int(pd[i])
            if not reaches(n, v, e, s, t):
                assert paths[i] is None
                continue
            # k walks need at most k * n edges when a cycle lies on an s -> t walk; all of them are shorter otherwise
            exp = brute_walks(n, v, e, ids, s, t, min(k * n, 9))[:k]
            got = [w for w in paths[i] if (len(w) - 1) // 2 <= 9]
            assert got == exp[:len(got)] and len(got) == min(len(exp), len(got)), (seed, s, t, k)
            assert npaths[i] == len(paths[i]) <= k


@pytest.mark.parametrize("seed", range(8))
def test_oracle_length_counts_are_matrix_powers(seed):
    n, src, dst = random_multigraph(400 + seed, 6, 14)
    v, e, ids = ref_csr(n, src, dst)
    rng = np.random.default_rng(seed)
    ps, pd = rng.integers(0, n, 40), rng.integers(0, n, 40)
    k = 50
    paths, npaths, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, k)
    for i in range(len(ps)):
        if paths[i] is None:
            continue
        lens = [(len(w) - 1) // 2 for w in paths[i]]
        counts = length_counts(n, v, e, int(ps[i]), int(pd[i]), max(lens))
        # every length below the last is listed whole, the last up to k
        for h in range(max(lens)):
            assert lens.count(h) == counts[h]
        assert 1 <= lens.count(max(lens)) <= counts[max(lens)]
        assert len(lens) == k or sum(counts) == len(lens)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_prefix_is_all_shortest_paths(seed):
    n, src, dst = random_multigraph(500 + seed, 20, 60)
    v, e, ids = ref_csr(n, src, dst)
    rng = np.random.default_rng(seed)
    ps, pd = rng.integers(0, n, 200), rng.integers(0, n, 200)
    cnt, valid = oas.shortest_path_count(n, v, e, ids, ps, pd)
    for k in (1, 2, 5):
        paths, _, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, k)
        ap, _ = oas.all_shortest_paths(n, v, e, ids, ps, pd, k)
        for i in range(len(ps)):
            if valid[i] and k <= cnt[i]:
                assert paths[i] == ap[i]
            elif not valid[i]:
                assert paths[i] is None
    sp, _ = orc.shortestpath(n, v, e, ids, ps, pd)
    paths, _, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, 1)
    assert [None if x is None else x[0] for x in paths] == sp


def test_catalogue_crossing_into_the_next_length():
    c = case_crossing()
    out = per_row(c, lambda i, k: run_oracle(c, k, ps=[0], pd=[3])[0][0])
    assert [len(x) for x in out] == [1, 2, 3]
    assert [(len(w) - 1) // 2 for w in out[2]] == [2, 2, 5]


def test_catalogue_parity_gaps():
    c = case_bipartite()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    paths, _, _ = run_oracle(c, 7)
    for w in paths[0] + paths[1]:
        assert ((len(w) - 1) // 2) % 2 == 0
    assert length_counts(c["n"], v, e, 0, 2, 9)[1::2] == [0] * 5


def test_catalogue_fewer_than_k():
    for c in (case_dag(), case_trap()):
        paths, npaths, st = run_oracle(c, c["ks"][0])
        assert npaths[0] < c["ks"][0] and npaths[0] == len(brute_walks(c["n"], *ref_csr(c["n"], c["src"], c["dst"]),
                                                                      c["ps"][0], c["pd"][0], 12))
    c = case_trap()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    assert length_counts(c["n"], v, e, 0, 1, 20)[-1] == 1  # the self-loop keeps a walk to 1 alive forever
    _, _, st = run_oracle(c, 5)
    assert st["levels"] == 2  # ... yet the row stops: layer 2 is zero on B(2)


def test_catalogue_cycle_behind_a_long_chain():
    c = case_long_chain_cycle()
    paths, _, st = run_oracle(c, 4, ps=[0], pd=[43])
    assert [(len(w) - 1) // 2 for w in paths[0]] == [41, 44, 47, 50]
    assert st["levels"] == 50


def test_catalogue_parallel_edges_and_self_loops():
    c = case_parallel_loops()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    paths, _, _ = run_oracle(c, 9, ps=[0], pd=[1])
    assert paths[0] == brute_walks(2, v, e, ids, 0, 1, 4)[:9]
    assert len({tuple(w) for w in paths[0]}) == 9 and [(len(w) - 1) // 2 for w in paths[0][:2]] == [1, 1]


def test_catalogue_same_vertex():
    c = case_same_vertex()
    paths, _, _ = run_oracle(c, 4, ps=[0], pd=[0])
    assert paths[0] == [[0], [0, 0, 1, 1, 0], [0, 0, 1, 1, 0, 0, 1, 1, 0], [0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 1, 1, 0]]
    paths, _, st = run_oracle(c, 4, ps=[2], pd=[2])
    assert paths[0] == [[2]] and st["levels"] == 1
    _, _, st = run_oracle(c, 1, ps=[2], pd=[2])
    assert st["levels"] == 0


def internal_order(n, src, dst):
    """the device's vertex numbering (DESIGN section 2)"""
    outd, ind = np.bincount(src, minlength=n), np.bincount(dst, minlength=n)
    cls = np.where(outd > 0, np.where(ind > 0, 0, 2), np.where(ind > 0, 1, 3))
    deg = np.where(cls == 1, ind, outd)
    return sorted(range(n), key=lambda x: (cls[x], -deg[x]))


def test_catalogue_hub_ties_disagree_with_the_internal_order():
    c = case_hub_ties()
    order = internal_order(c["n"], np.array(c["src"]), np.array(c["dst"]))
    parents = [x for x in order if 1 <= x <= 8]
    assert parents == sorted(parents, reverse=True)
    paths, _, _ = run_oracle(c, 12, ps=[0], pd=[9])
    assert [w[2] for w in paths[0][:8]] == list(range(1, 9)) and (len(paths[0][8]) - 1) // 2 == 5


def test_catalogue_saturated_row():
    n, src, dst = diamonds(64)
    v, e, ids = ref_csr(n, src, dst)
    paths, npaths, _ = oks.shortest_k_paths(n, v, e, ids, [0], [192], 5)
    ap, cnt = oas.all_shortest_paths(n, v, e, ids, [0], [192], 5)
    assert cnt[0] == INT64_MAX and length_counts(n, v, e, 0, 192, 128)[128] == 1 << 64
    assert paths == ap and npaths.tolist() == [5]


def test_catalogue_specials_and_edgeless():
    c = case_specials()
    paths, npaths, _ = run_oracle(c, 3)
    assert paths[0][0] == [0, 0, 1, 1, 2] and paths[1:4] == [None, None, None] and paths[4][0] == [2, 2, 0, 0, 1]
    assert npaths.tolist() == [3, 0, 0, 0, 3]  # (the cycle 0 -> 1 -> 2 -> 0 gives every reachable row k walks)
    c = case_edgeless()
    paths, _, st = run_oracle(c, 3)
    assert paths == [[[0]], None, [[2]]] and st["levels"] == 1 and st["push_levels"] == 1


@pytest.mark.parametrize("p", [1, 63, 64, 65, 513])
def test_catalogue_row_counts(p):
    c = case_rows(p)
    paths, npaths, st = run_oracle(c, 7)
    assert st["batches"] == (p + 63) // 64 and st["searches"] == p
    assert sum(x is not None for x in paths) > 0


def test_catalogue_walk_limit():
    """a 256-cycle: the walks 0 -> 253 have lengths 253 + 256 j, the 256th exactly 65533 edges"""
    n, src, dst = cycle_with_tail(256, 253)
    v, e, ids = ref_csr(n, src, dst)
    paths, _, _ = oks.shortest_k_paths(n, v, e, ids, [0], [253], 256)
    assert (len(paths[0][-1]) - 1) // 2 == WALK_MAX
    with pytest.raises(orc.OracleError) as ex:
        oks.shortest_k_paths(n, v, e, ids, [0], [253], 257)
    assert ex.value.code == oks.ERR_UNSUPPORTED


def test_catalogue_layer_budget():
    """the hub_ties row (0, 0) with k = 10 ends with a walk of 6 edges: its layers need (6 + 1) x n_ab x 8 bytes"""
    c = case_hub_ties()
    paths, _, _ = run_oracle(c, 10, ps=[0], pd=[0])
    assert (len(paths[0][-1]) - 1) // 2 == 6
    assert budget_bytes(c, 6, 1) == 7 * 46 * 8  # n_ab: 0 .. 9 and the 36 sinks have in-edges


def budget_bytes(c, h, rows):
    n_ab = len(set(np.asarray(c["dst"]).tolist()))
    return (h + 1) * n_ab * rows * 8


def test_oracle_errors():
    v, e, ids = ref_csr(3, [0], [1])
    for call, code in ((lambda: oks.shortest_k_paths(3, v, e, ids, [0], [1], 0), oks.ERR_ARG),
                       (lambda: oks.shortest_k_paths(3, v, e, ids, [0], [3], 1), oks.ERR_RANGE)):
        with pytest.raises(orc.OracleError) as ex:
            call()
        assert ex.value.code == code
    paths, _, _ = oks.shortest_k_paths(3, v, e, ids, [0, 9], [9, 1], 1, [1, 0], [0, 1])
    assert paths == [None, None]


# ---- GPU: the device against the oracle ------------------------------------------------------------------------------
def compare(csr, n, v, e, ids, ps, pd, k, sv=None, dv=None, options=None):
    paths, npaths, st = csr.shortest_k_paths(ps, pd, k, sv, dv, options)
    opaths, onp, ost = oks.shortest_k_paths(n, v, e, ids, ps, pd, k, sv, dv, st["lanes"])
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
    for k in sorted(set(c["ks"])) + [1]:
        compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], k, c.get("sv"), c.get("dv"))
    csr.free()


@pytest.mark.gpu
def test_device_worked_examples_and_saturation(gpu_ctx):
    csr = pgq.DeviceCSR.build(gpu_ctx, 5, np.array(TOPK["src"]), np.array(TOPK["dst"]))
    paths, _, _ = csr.shortest_k_paths([0, 4, 0], [3, 0, 4], 5)
    assert paths[0] == [[0, 2, 3], [0, 0, 1, 5, 3], [0, 1, 2, 6, 3], [0, 2, 3, 3, 0, 2, 3], [0, 0, 1, 4, 2, 6, 3]]
    assert paths[1][:3] == [[4, 7, 3, 3, 0], [4, 7, 3, 3, 0, 2, 3, 3, 0], [4, 7, 3, 3, 0, 0, 1, 5, 3, 3, 0]]
    assert paths[2] is None
    csr.free()
    n, src, dst = diamonds(64)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    compare(csr, n, v, e, ids, [0, 0, 3], [192, 189, 3], 5)
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names())
def test_device_reference_graphs(gpu_ctx, name):
    g = load_golden(name)
    n = g["n"]
    v, e, ids = ref_csr(n, g["src"], g["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, n, g["src"], g["dst"])
    sv = g["psrc_valid"].astype(np.uint8)
    for k in (1, 7):
        compare(csr, n, v, e, ids, g["psrc"][:600], g["pdst"][:600], k, sv[:600])
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [12, 14, 16])
def test_device_rmat(gpu_ctx, scale):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(1024 if scale < 16 else 160, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    for k in (1, 2, 7, 64):
        paths, _ = compare(csr, n, v, e, ids, ps, pd, k)
        if k == 1:
            sp, _ = csr.shortestpath(ps, pd)
            assert [None if x is None else x[0] for x in paths] == sp
    ap, cnt, _ = csr.all_shortest_paths(ps, pd, 7)
    for i in range(len(ps)):
        if ap[i] is not None and cnt[i] >= 7:
            assert paths[i][:7] == ap[i]
    csr.free()


@pytest.mark.gpu
def test_device_lane_widths_and_row_order(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(700, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    base, _ = compare(csr, n, v, e, ids, ps, pd, 9)
    for lanes in range(64, 513, 64):
        paths, st = compare(csr, n, v, e, ids, ps, pd, 9, options=pgq.Options(lanes))
        assert paths == base and st["lanes"] == lanes
    perm = np.random.default_rng(1).permutation(len(ps))
    paths, _, _ = csr.shortest_k_paths(ps[perm], pd[perm], 9)
    assert paths == [base[i] for i in perm]
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
    for csr in (chunked, pgq.DeviceCSR.build(gpu_ctx, n, src, dst), pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)):
        compare(csr, n, v, e, ids, ps, pd, 6)
        csr.free()
    up = pgq.DeviceCSR.upload(gpu_ctx, n, v, e)  # no ids: CSR positions
    compare(up, n, v, e, np.arange(len(e)), ps, pd, 6)
    up.free()
    vk = np.random.default_rng(4).permutation(n).astype(np.int64) * 3
    for undirected in (False, True):
        csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, vk, vk[src], vk[dst], undirected=undirected)
        kv, ke, kids = csr.download()
        compare(csr, csr.n, kv, ke, kids, ps % csr.n, pd % csr.n, 6)
        csr.free()


@pytest.mark.gpu
def test_device_walk_limit(gpu_ctx):
    n, src, dst = cycle_with_tail(256, 253)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    paths, _ = compare(csr, n, v, e, ids, [0], [253], 256)
    assert (len(paths[0][-1]) - 1) // 2 == WALK_MAX
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_paths([0], [253], 257)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()


@pytest.mark.gpu
def test_device_layer_budget(gpu_ctx, monkeypatch):
    c = case_rows(130, seed=9)
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))
    base, _ = compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], 7)
    hmax = max((len(w) - 1) // 2 for p in base if p for w in p)
    one_row = budget_bytes(c, hmax, 1)
    for rows in (1, 2, 5):  # groups of at most `rows` rows of the longest walk
        monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(one_row * rows))
        paths, _ = compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], 7)
        assert paths == base
    monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(one_row - 1))
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_paths(c["ps"], c["pd"], 7)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", "x")
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_paths(c["ps"], c["pd"], 7)
    assert ex.value.status == PGQ_ERR_INVALID_ARG
    csr.free()


@pytest.mark.gpu
def test_device_errors_and_raw_abi(gpu_ctx):
    import ctypes as C
    from duckpgq_extension_b200 import _native
    lib = _native.load()
    csr = pgq.DeviceCSR.build(gpu_ctx, 4, np.array([0, 1, 2]), np.array([1, 2, 0]))
    for call in (lambda: csr.shortest_k_paths([0, 4], [1, 1], 2), lambda: csr.shortest_k_paths([0], [-1], 2)):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == PGQ_ERR_RANGE
    for call, status in ((lambda: csr.shortest_k_paths([0], [1], 0), PGQ_ERR_INVALID_ARG),
                         (lambda: csr.shortest_k_paths([0], [1], 2, options=pgq.Options(96)), PGQ_ERR_INVALID_ARG),
                         (lambda: csr.shortest_k_paths([0], [1], 2, options=pgq.Options(0, shard_index=0,
                                                                                         shard_count=2)),
                          PGQ_ERR_UNSUPPORTED)):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == status
    paths, npaths, _ = csr.shortest_k_paths([0, 9], [9, 1], 3, [1, 0], [0, 1])  # all NULL: ids under NULL unread
    assert paths == [None, None] and npaths.tolist() == [0, 0]
    paths, _, st = csr.shortest_k_paths([], [], 3)
    assert paths == [] and st["batches"] == 0
    # the raw lists: offsets into one element array, rows' first walks
    p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    src, dst = np.array([0, 3, 1], np.int64), np.array([2, 3, 1], np.int64)
    npw, first, valid = np.zeros(3, np.int64), np.zeros(3, np.int64), np.zeros(3, np.uint8)
    offs, elems, total = p64(), p64(), C.c_int64(0)
    assert lib.pgq_shortest_k_paths(csr._h, 3, src.ctypes.data_as(p64), dst.ctypes.data_as(p64), None, None, None, 2,
                                    npw.ctypes.data_as(p64), first.ctypes.data_as(p64), valid.ctypes.data_as(pu8),
                                    C.byref(offs), C.byref(elems), C.byref(total), None) == 0
    o = [offs[j] for j in range(total.value + 1)]
    flat = [elems[j] for j in range(o[-1])]
    lib.pgq_free(offs)
    lib.pgq_free(elems)
    assert npw.tolist() == [2, 1, 2] and first.tolist() == [0, 2, 3] and valid.tolist() == [1, 1, 1]
    assert [flat[o[j]:o[j + 1]] for j in range(5)] == [[0, 0, 1, 1, 2], [0, 0, 1, 1, 2, 2, 0, 0, 1, 1, 2], [3],
                                                       [1], [1, 1, 2, 2, 0, 0, 1]]
    assert lib.pgq_shortest_k_paths(csr._h, 1, None, None, None, None, None, 1, None, None, None, C.byref(offs),
                                    C.byref(elems), C.byref(total), None) == PGQ_ERR_INVALID_ARG
    assert lib.pgq_shortest_k_paths(csr._h, 0, None, None, None, None, None, 1, None, None, None, C.byref(offs),
                                    C.byref(elems), C.byref(total), None) == 0
    assert total.value == 0 and offs[0] == 0
    lib.pgq_free(offs)
    lib.pgq_free(elems)
    csr.free()
    un = pgq.DeviceCSR.create(gpu_ctx, 3)
    with pytest.raises(pgq.PgqError) as ex:
        un.shortest_k_paths([0], [1], 2)
    assert ex.value.status == PGQ_ERR_NOT_INITIALIZED
    un.free()


@pytest.mark.gpu
def test_udf_mirror(gpu_ctx):
    state = pgq.DuckPGQState(gpu_ctx)
    with pytest.raises(pgq.ConstraintException) as ex:
        pgq.shortest_k_paths(state, 3, 4, [0], [1], 2)
    assert "Invalid ID" in str(ex.value)
    pgq.create_csr_vertex(state, 0, 4, np.arange(4), np.array([2, 1, 1, 1]))
    pgq.create_csr_edge(state, 0, 4, 5, 5, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], [10, 11, 12, 13, 14])
    paths = pgq.shortest_k_paths(state, 0, 4, [0, 0, 3], [3, 0, 0], 3)
    assert paths[0][:2] == [[0, 10, 1, 12, 3], [0, 11, 2, 13, 3]] and paths[1][0] == [0] and paths[2][0] == [3, 14, 0]
    v, e, ids = ref_csr(4, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], np.arange(10, 15))
    assert paths == oks.shortest_k_paths(4, v, e, ids, [0, 0, 3], [3, 0, 0], 3)[0] and 0 in state.csr_to_delete
    state.query_end()


@pytest.mark.gpu
def test_one_workspace_in_turn(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(300, n)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    alone = (csr.iterativelength(ps, pd)[:2], csr.shortestpath(ps, pd)[0], csr.all_shortest_paths(ps, pd, 16)[0],
             csr.shortest_k_paths(ps, pd, 16)[0])
    for _ in range(2):
        ks = csr.shortest_k_paths(ps, pd, 16)[0]
        il = csr.iterativelength(ps, pd)[:2]
        sp = csr.shortestpath(ps, pd)[0]
        ap = csr.all_shortest_paths(ps, pd, 16)[0]
        assert ks == alone[3] and sp == alone[1] and ap == alone[2]
        assert np.array_equal(il[0], alone[0][0]) and np.array_equal(il[1], alone[0][1])
    csr.free()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(200, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    exp, _, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, 8)
    out = [None] * 8

    def work(k):
        out[k] = csr.shortest_k_paths(ps, pd, 8)[0]

    ths = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(o == exp for o in out)
