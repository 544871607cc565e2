"""local_clustering_coefficient, pagerank and weakly_connected_component on the device CSR, compared bit for bit with
the reference binary's outputs (tests/golden/refn4_*.npz) and with the CPU restatement (oracle/pgq_oracle.c):
float32 / float64 as bit patterns, component ids and PageRank iteration counts exactly.  Ids n and n + 1 are the
reference's two entries behind the vertices (vsize = n + 2).

The CPU-only test checks the argument the device WCC rests on: the reference's labels follow from replaying Link over
the merge edges alone, which are the minimum spanning forest under "weight = CSR position"."""
import glob
import importlib.util
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc

_spec = importlib.util.spec_from_file_location("make_golden_next4", os.path.join(GOLDEN, "make_golden_next4.py"))
make_golden_next4 = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden_next4)
undirected = make_golden_next4.undirected

GOLDENS = sorted(os.path.basename(p)[len("refn4_"):-len(".npz")] for p in glob.glob(os.path.join(GOLDEN, "refn4_*.npz")))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64 if a.dtype == np.float64 else a.dtype)


@pytest.fixture(scope="module")
def ctx():
    return pgq.default_context(0)


def build_csr(ctx, how, n, src, dst):
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    if how == "build":
        return pgq.DeviceCSR.build(ctx, n, src, dst)
    if how == "upload":
        v, e, ids = orc.csr_build(n, src, dst)
        return pgq.DeviceCSR.upload(ctx, n, v, e, ids)
    csr = pgq.DeviceCSR.create(ctx, n)  # chunked, as create_csr_vertex / create_csr_edge feed it
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    m = len(src)
    for o in range(0, m, 97):
        csr.add_edges(m, m, src[o:o + 97], dst[o:o + 97], np.arange(o, min(o + 97, m)))
    csr.finalize()
    return csr


def check_against_oracle(csr, n, src, dst, lcc_ids=None, golden=None):
    """Every id in [-2, n + 4) for PageRank and WCC, every vertex (or lcc_ids) for LCC."""
    v, e, _ = orc.csr_build(n, src, dst)
    ids = np.arange(-2, n + 4, dtype=np.int64)
    pr, prv, it, _ = csr.pagerank(ids)
    opr, oprv, oit = orc.pagerank(n, v, e, ids)
    assert it == oit
    assert np.array_equal(prv, oprv) and np.array_equal(bits(pr[prv == 1]), bits(opr[oprv == 1]))
    assert prv.tolist() == [0, 0] + [1] * (n + 2) + [0, 0]
    wcc, wv, _ = csr.weakly_connected_component(ids)
    owcc, owv = orc.weakly_connected_component(n, v, e, ids)
    assert np.array_equal(wv, owv) and np.array_equal(wcc[wv == 1], owcc[owv == 1])
    q = np.arange(n, dtype=np.int64) if lcc_ids is None else np.asarray(lcc_ids, dtype=np.int64)
    lcc, lv, _ = csr.local_clustering_coefficient(q)
    olcc, olv = orc.local_clustering_coefficient(n, v, e, q)
    assert np.array_equal(lv, olv) and np.array_equal(bits(lcc), bits(olcc))
    if golden is not None:
        assert np.array_equal(bits(lcc), bits(golden["lcc"].astype(np.float32)))
        assert np.array_equal(wcc[2:2 + n], golden["wcc"].astype(np.int64))
        assert np.array_equal(bits(pr[2:2 + n]), bits(golden["pagerank"]))


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["build", "upload", "chunked"])
@pytest.mark.parametrize("name", GOLDENS)
def test_goldens(ctx, name, how):
    g = np.load(os.path.join(GOLDEN, f"refn4_{name}.npz"))
    n = int(g["n"])
    csr = build_csr(ctx, how, n, g["src"], g["dst"])
    try:
        check_against_oracle(csr, n, g["src"].astype(np.int64), g["dst"].astype(np.int64), golden=g)
    finally:
        csr.free()


def star(leaves):
    c = leaves  # the centre has the highest id
    s = np.concatenate([np.full(leaves, c), np.arange(leaves), np.arange(0, leaves - 1, 7)])
    d = np.concatenate([np.arange(leaves), np.full(leaves, c), np.arange(1, leaves, 7)])
    return leaves + 1, s, d


def path(n):
    return n, np.arange(n - 1), np.arange(1, n)


def odd_shapes(seed=5):
    rng = np.random.default_rng(seed)
    n = 2000  # ids >= 1900 isolated; many small components; self-loops and parallel edges
    s = rng.integers(0, 1900, 3000)
    d = np.clip(s + rng.integers(-4, 5, 3000), 0, 1899)
    s = np.concatenate([s, np.arange(0, 1900, 11), s[:300]])
    d = np.concatenate([d, np.arange(0, 1900, 11), d[:300]])
    return n, s, d


def generated(name):
    if name.startswith("rmat"):
        scale = int(name[4:6])
        n, s, d = datagen.rmat_edges(scale)
        s, d = s.astype(np.int64), d.astype(np.int64)
        if name.endswith("u"):
            s, d = undirected(n, s, d)
        return n, s, d
    if name == "snb":
        n, s, d, _ = datagen.snb_shaped_edges(20000, 20.0, seed=3)
        return n, s, d
    if name == "star":
        return star(50000)
    if name == "path":
        return path(3000)
    return odd_shapes()


def lcc_sample(n, src):
    deg = np.bincount(src, minlength=n)
    top = np.argsort(-deg, kind="stable")[:64]  # the hubs: the bitmap path for out-degrees above 4096
    rest = np.random.default_rng(1).choice(n, size=min(n, 3000), replace=False)
    return np.concatenate([top, rest])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rmat12d", "rmat12u", "rmat14d", "rmat14u", "rmat16d", "rmat16u", "snb", "star",
                                  "path", "odd"])
def test_generated_graphs(ctx, name):
    n, s, d = generated(name)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        check_against_oracle(csr, n, s, d, lcc_ids=lcc_sample(n, np.asarray(s)) if n > 5000 else None)
    finally:
        csr.free()


@pytest.mark.gpu
def test_star_hub_paths(ctx):
    """The centre's out-list (50 000) takes the bitmap path of LCC, its in-list is one 50 000-long PageRank fold, and
    the leaves merge into it one by one."""
    n, s, d = star(50000)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    v, e, _ = orc.csr_build(n, s, d)
    try:
        ids = np.array([n - 1, 0, n - 1], dtype=np.int64)
        lcc, lv, _ = csr.local_clustering_coefficient(ids)
        olcc, _ = orc.local_clustering_coefficient(n, v, e, ids)
        assert lcc[0] > 0 and np.array_equal(bits(lcc), bits(olcc))
        wcc, _, _ = csr.weakly_connected_component(np.arange(n + 2))
        owcc, _ = orc.weakly_connected_component(n, v, e, np.arange(n + 2))
        assert np.array_equal(wcc, owcc)
    finally:
        csr.free()


@pytest.mark.gpu
def test_query_edge_cases(ctx):
    n, s, d = datagen.rmat_edges(10)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    v, e, _ = orc.csr_build(n, s, d)
    try:
        ids = np.array([3, 3, -1, n, n + 1, n + 2, 1 << 40, 0, 7, 7, -(1 << 40)], dtype=np.int64)
        valid = np.array([1, 0, 1, 1, 1, 1, 1, 1, 0, 1, 1], dtype=np.uint8)
        pr, prv, _, _ = csr.pagerank(ids, valid)
        opr, oprv, _ = orc.pagerank(n, v, e, ids, valid)
        assert prv.tolist() == [1, 0, 0, 1, 1, 0, 0, 1, 0, 1, 0] and np.array_equal(prv, oprv)
        assert np.array_equal(bits(pr[prv == 1]), bits(opr[oprv == 1]))
        wcc, wv, _ = csr.weakly_connected_component(ids, valid)
        assert wv.tolist() == [1, 0, 0, 1, 1, 0, 0, 1, 0, 1, 0]
        owcc, _ = orc.weakly_connected_component(n, v, e, ids)
        assert np.array_equal(wcc[wv == 1], owcc[wv == 1])
        assert wcc[4] == owcc[4] and wcc[4] == wcc[7]  # n + 1 carries vertex 0's label (forest[n + 1] = 0)
        lids = np.array([3, 3, 5, 0, 7], dtype=np.int64)
        lv_in = np.array([1, 1, 0, 1, 1], dtype=np.uint8)
        lcc, lv, _ = csr.local_clustering_coefficient(lids, lv_in)
        olcc, olv = orc.local_clustering_coefficient(n, v, e, lids, lv_in)
        assert lv.tolist() == [1, 1, 0, 1, 1] and np.array_equal(bits(lcc), bits(olcc))
        for empty in (csr.pagerank([]), csr.weakly_connected_component([]), csr.local_clustering_coefficient([])):
            assert len(empty[0]) == 0
        for bad in (-1, n, n + 1):
            with pytest.raises(pgq.InvalidInputException) as ex:
                csr.local_clustering_coefficient(np.array([0, bad]))
            assert ex.value.status == pgq.PGQ_ERR_RANGE
            again, _, _ = csr.local_clustering_coefficient(lids, lv_in)
            assert np.array_equal(bits(again), bits(lcc))
        nulled, nv, _ = csr.local_clustering_coefficient(np.array([-5, 2]), np.array([0, 1], dtype=np.uint8))
        assert nv.tolist() == [0, 1]  # a NULL row is not range-checked
    finally:
        csr.free()


@pytest.mark.gpu
def test_chunks_equal_one_call(ctx):
    n, s, d = datagen.rmat_edges(12)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        ids = np.random.default_rng(4).integers(0, n + 2, 10000)
        lids = ids[ids < n]
        one_pr = csr.pagerank(ids)[0]
        one_w = csr.weakly_connected_component(ids)[0]
        one_l = csr.local_clustering_coefficient(lids)[0]
        parts = range(0, len(ids), 2048)
        first = csr.pagerank(ids[:2048])
        assert first[3]["levels"] == 0  # answered from the cached vector
        assert np.array_equal(bits(np.concatenate([csr.pagerank(ids[o:o + 2048])[0] for o in parts])), bits(one_pr))
        assert np.array_equal(np.concatenate([csr.weakly_connected_component(ids[o:o + 2048])[0] for o in parts]), one_w)
        lparts = range(0, len(lids), 333)
        assert np.array_equal(bits(np.concatenate([csr.local_clustering_coefficient(lids[o:o + 333])[0] for o in lparts])),
                              bits(one_l))
    finally:
        csr.free()


@pytest.mark.gpu
def test_concurrent_first_calls(ctx):
    n, s, d = datagen.rmat_edges(14)
    ids = np.arange(-1, n + 3)
    results = {}
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        barrier = threading.Barrier(8)

        def work(t):
            barrier.wait()
            if t % 2:
                r = csr.pagerank(ids)
                results[t] = (bits(r[0]).tobytes(), r[1].tobytes(), r[2])
            else:
                r = csr.weakly_connected_component(ids)
                results[t] = (r[0].tobytes(), r[1].tobytes())
            csr.local_clustering_coefficient(np.arange(0, n, 17))

        threads = [threading.Thread(target=work, args=(t,)) for t in range(8)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert len(results) == 8
        assert len({results[t] for t in range(1, 8, 2)}) == 1
        assert len({results[t] for t in range(0, 8, 2)}) == 1
        v, e, _ = orc.csr_build(n, s, d)
        opr, _, oit = orc.pagerank(n, v, e, ids)
        assert results[1][0] == bits(opr).tobytes() and results[1][2] == oit
    finally:
        csr.free()


@pytest.mark.gpu
def test_module_functions_lookup_and_delete_marking(ctx):
    state = pgq.DuckPGQState(ctx)
    n, s, d = path(50)
    fns = (pgq.local_clustering_coefficient, pgq.pagerank, pgq.weakly_connected_component)
    for f in fns:
        with pytest.raises(pgq.ConstraintException, match="CSR not found. Is the graph populated?"):
            f(state, 0, np.array([0]))
    # vertices counted, no create_csr_edge yet: the binds' "Need to initialize CSR before ..." texts
    half = pgq.DeviceCSR.create(ctx, n)
    half.add_vertex_counts(np.arange(n), np.bincount(s, minlength=n))
    state.csr_list[1] = half
    for f, text in zip(fns, ("Need to initialize CSR before doing local clustering coefficient.",
                             "Need to initialize CSR before running PageRank.",
                             "Need to initialize CSR before doing weakly connected components.")):
        with pytest.raises(pgq.ConstraintException) as ex:
            f(state, 1, np.array([0]))
        assert str(ex.value) == text
    half.free()
    del state.csr_list[1]
    state.csr_list[0] = pgq.DeviceCSR.build(ctx, n, s, d)
    v, e, _ = orc.csr_build(n, s, d)
    ids = np.array([0, 49, 50, 51, 52])
    pr, prv = pgq.pagerank(state, 0, ids)
    opr, oprv, _ = orc.pagerank(n, v, e, ids)
    assert np.array_equal(prv, oprv) and np.array_equal(bits(pr[prv == 1]), bits(opr[oprv == 1]))
    lcc, lv = pgq.local_clustering_coefficient(state, 0, np.array([0, 1, 48]))
    assert lv.tolist() == [1, 1, 1] and lcc.tolist() == [0.0, 0.0, 0.0]
    assert pgq.weakly_connected_component(state, 0, np.array([49]))[0].tolist() == [49]
    assert 0 in state.csr_to_delete
    state.query_end()
    assert 0 not in state.csr_list


@pytest.mark.gpu
def test_path_functions_unchanged_after_analytics_on_one_workspace():
    """The analytics use workspace scratch slots only, never the BFS lane-mask arrays whose zero rows a workspace
    remembers between calls.  A fresh context has one workspace, so the searches before and after the analytics
    share it; lane width 64 (one mask word) and NO_PRUNE give destinations without in-edges a lane, whose rows the
    search reads but never writes."""
    own = pgq.Context(0)
    n, s, d = datagen.rmat_edges(11)
    s, d = np.asarray(s, dtype=np.int64), np.asarray(d, dtype=np.int64)
    n2 = n + 600  # 600 isolated vertices, and every R-MAT vertex without in-edges: rows past the reachable ones
    csr = pgq.DeviceCSR.build(own, n2, s, d)
    v, e, ids = orc.csr_build(n2, s, d)
    try:
        rng = np.random.default_rng(9)
        no_in = np.setdiff1d(np.arange(n2), d)
        ps = rng.integers(0, n, 400)
        pd = np.concatenate([rng.choice(no_in, 200), rng.integers(0, n2, 200)])
        opts = pgq.Options(lanes=64, no_prune=True)
        exp, expv, _ = orc.iterativelength(n2, v, e, ps, pd, None, 64)
        paths_exp, _ = orc.shortestpath(n2, v, e, ids, ps[:100], pd[:100])

        def check():
            out, valid, _ = csr.iterativelength(ps, pd, None, opts)
            assert np.array_equal(valid, expv) and np.array_equal(out, exp)
            paths, _ = csr.shortestpath(ps[:100], pd[:100], None, opts)
            assert paths == paths_exp

        check()
        csr.pagerank(np.arange(n2))
        check()
        csr.weakly_connected_component(np.arange(n2))
        check()
        csr.local_clustering_coefficient(np.arange(n2))
        check()
    finally:
        csr.free()
        own.close()


# ---- CPU only: the WCC argument ------------------------------------------------------------------------------------
def merge_edges_by_position(n, v, e):
    """Kruskal with weight = CSR position: the edges that join two different trees, in position order."""
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    out = []
    rows = np.repeat(np.arange(n), np.diff(v[:n + 1]))
    for a, b in zip(rows.tolist(), e.tolist()):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
            out.append((a, b))
    return out


def link_replay(n, merges):
    """Link (weakly_connected_component.cpp:26-35) over the merge edges only; forest[n + 1] = 0."""
    forest = np.arange(n + 2, dtype=np.int64)
    forest[n + 1] = 0

    def find(x):
        while forest[x] != x:
            forest[x] = forest[forest[x]]
            x = forest[x]
        return x

    for a, b in merges:
        ra, rb = find(a), find(b)
        if ra != rb:
            forest[ra] = rb
    return np.array([find(x) for x in range(n + 2)], dtype=np.int64)


@pytest.mark.parametrize("directed", [True, False])
def test_wcc_merge_edge_replay_equals_reference_cpu(directed):
    for seed in range(100):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(1, 60))
        m = int(rng.integers(0, 3 * n + 1))
        s = rng.integers(0, n, m)
        d = rng.integers(0, n, m)
        if rng.random() < 0.3:  # parallel edges
            s, d = np.concatenate([s, s[: m // 3]]), np.concatenate([d, d[: m // 3]])
        if not directed:
            s, d = undirected(n, s, d)
            if len(s) and rng.random() < 0.5:  # the reference's undirected CSR, but in a shuffled arrival order
                p = rng.permutation(len(s))
                s, d = s[p], d[p]
        v, e, _ = orc.csr_build(n, s, d)
        ids = np.arange(n + 2)
        expect, _ = orc.weakly_connected_component(n, v, e, ids)
        got = link_replay(n, merge_edges_by_position(n, v, e))
        assert np.array_equal(got, expect), (seed, n, m)
