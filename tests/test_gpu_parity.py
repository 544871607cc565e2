"""Parity of the CUDA path (through the C ABI, libduckpgq_b200.so) with the reference:
golden vectors produced by the reference binary, and differential tests against the CPU
restatement (oracle/) on seeded inputs.  Bit-exact: hop counts, NULL masks, path lists, CSR arrays,
and the work counters (levels, edges traversed W)."""
import numpy as np
import pytest

from conftest import golden_names, load_golden
from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc

pytestmark = pytest.mark.gpu

LANES = [64, 128, 256, 512]
PATH_GOLDEN = [n for n in golden_names() if load_golden(n)["has_paths"]]


def upload(ctx, g, with_ids=True):
    ids = None
    if with_ids:
        _, _, ids = orc.csr_build(g["n"], g["src"], g["dst"])
    return pgq.DeviceCSR.upload(ctx, g["n"], g["csr_v"], g["csr_e"], ids)


@pytest.mark.parametrize("name", golden_names())
def test_device_csr_build_equals_reference_csr(gpu_ctx, name):
    """create_csr_vertex + create_csr_edge on the device == get_csr_v / get_csr_e of the reference."""
    g = load_golden(name)
    csr = pgq.DeviceCSR.build(gpu_ctx, g["n"], g["src"], g["dst"])
    v, e, ids = csr.download()
    assert v.tolist() == g["csr_v"].tolist()
    assert e.tolist() == g["csr_e"].tolist()
    _, _, oids = orc.csr_build(g["n"], g["src"], g["dst"])
    assert ids.tolist() == oids.tolist()
    csr.free()


@pytest.mark.parametrize("name", golden_names())
@pytest.mark.parametrize("lanes", LANES)
@pytest.mark.parametrize("direction", [0, 1, 2])
def test_iterativelength_golden(gpu_ctx, name, lanes, direction):
    g = load_golden(name)
    csr = upload(gpu_ctx, g, with_ids=False)
    # reference batching: every non-NULL, src != dst row takes a lane exactly as in the reference
    out, valid, st = csr.iterativelength(g["psrc"], g["pdst"], g["psrc_valid"],
                                         pgq.Options(lanes, direction, reference_batching=True))
    assert valid.tolist() == g["length_valid"].tolist()
    assert out.tolist() == g["length"].tolist()
    # work counters are defined by the frontier sets -> identical to the restatement at the same lane width
    _, _, ost = orc.iterativelength(g["n"], g["csr_v"], g["csr_e"], g["psrc"], g["pdst"], g["psrc_valid"], lanes)
    assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
        ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices)
    assert st["pruned"] == 0
    # default: rows decided by the degrees alone take no lane -- same answers, fewer searches
    out2, valid2, st2 = csr.iterativelength(g["psrc"], g["pdst"], g["psrc_valid"], pgq.Options(lanes, direction))
    assert valid2.tolist() == g["length_valid"].tolist() and out2.tolist() == g["length"].tolist()
    assert st2["search_rows"] + st2["pruned"] == st["searches"] and st2["searches"] <= st2["search_rows"]
    csr.free()


@pytest.mark.parametrize("name", PATH_GOLDEN)
@pytest.mark.parametrize("lanes", [64, 512])
@pytest.mark.parametrize("direction", [0, 1, 2])
def test_shortestpath_golden(gpu_ctx, name, lanes, direction):
    g = load_golden(name)
    csr = upload(gpu_ctx, g)
    for ref_batching in (True, False):
        paths, st = csr.shortestpath(g["psrc"], g["pdst"], g["psrc_valid"],
                                     pgq.Options(lanes, direction, reference_batching=ref_batching))
        assert paths == g["paths"]
    csr.free()


@pytest.mark.parametrize("pairs", [1, 63, 64, 65, 511, 512, 513, 2048, 2049, 5000])
def test_pair_count_edges(gpu_ctx, pairs):
    """Nothing in the reference's tests exercises > 512 pairs / several lane batches (SURVEY section 4)."""
    n, src, dst = datagen.rmat_edges(11)
    v, e, ids = orc.csr_build(n, src, dst)
    ps, pd = datagen.hashed_pairs(pairs, n)
    csr = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    exp, expv, _ = orc.iterativelength(n, v, e, ps, pd, None, 512)
    for lanes in (64, 256, 512):
        out, valid, _ = csr.iterativelength(ps, pd, None, pgq.Options(lanes))
        assert valid.tolist() == expv.tolist() and out.tolist() == exp.tolist()
    csr.free()


@pytest.mark.parametrize("scale,pairs", [(14, 700), (16, 1024)])
def test_rmat_differential(gpu_ctx, scale, pairs):
    n, src, dst = datagen.rmat_edges(scale)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    v, e, ids = csr.download()
    ov, oe, oids = orc.csr_build(n, src, dst)
    assert np.array_equal(v, ov) and np.array_equal(e, oe) and np.array_equal(ids, oids)
    ps, pd = datagen.hashed_pairs(pairs, n)
    for lanes in (64, 256):
        exp, expv, ost = orc.iterativelength(n, v, e, ps, pd, None, lanes)
        for direction in (0, 1, 2):
            out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes, direction, reference_batching=True))
            assert np.array_equal(valid, expv) and np.array_equal(out, exp)
            assert st["edges_traversed"] == ost.edges_traversed and st["levels"] == ost.levels
            out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes, direction))
            assert np.array_equal(valid, expv) and np.array_equal(out, exp)
    csr.free()


def test_rmat_paths_differential(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    v, e, ids = orc.csr_build(n, src, dst, np.arange(len(src), dtype=np.int64) * 3 + 7)  # sparse edge rowids
    ps, pd = datagen.hashed_pairs(600, n)
    csr = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    exp, _ = orc.shortestpath(n, v, e, ids, ps, pd, None, 512)
    for lanes in (64, 128):
        got, _ = csr.shortestpath(ps, pd, None, pgq.Options(lanes))
        assert got == exp
    csr.free()


def test_undirected_snb_shaped_paths(gpu_ctx):
    """Config C4 at test size: SNB-shaped undirected knows graph, ANY SHORTEST with reconstruction."""
    n, src, dst, eid = datagen.snb_shaped_edges(3000, 20.0, seed=10)
    v, e, ids = orc.csr_build(n, src, dst, eid)
    rng = np.random.default_rng(5)
    ps, pd = rng.integers(0, n, 300), rng.integers(0, n, 300)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst, eid)
    exp, _ = orc.shortestpath(n, v, e, ids, ps, pd, None, 512)
    got, _ = csr.shortestpath(ps, pd)
    assert got == exp
    lens, valid, _ = csr.iterativelength(ps, pd)
    for path, ln, ok in zip(got, lens, valid):
        assert (path is None) == (not ok)
        if path is not None:
            assert len(path) // 2 == ln  # path_length(p) = len(path) // 2, match.cpp:745-757
    csr.free()


def test_reference_style_udf_calls(gpu_ctx):
    """The raw-SQL form of test/sql/path_finding/shortest_path.test:96-128, UDF by UDF."""
    st = pgq.DuckPGQState(gpu_ctx)
    src = np.array([0, 0, 0, 3, 1, 1, 2, 4]); dst = np.array([1, 2, 3, 0, 2, 3, 3, 3])
    cnt = np.bincount(src, minlength=5)
    total = int(pgq.create_csr_vertex(st, 0, 5, np.arange(5), cnt).sum())
    ones = pgq.create_csr_edge(st, 0, 5, total, len(src), src, dst, np.arange(8))
    assert ones.tolist() == [1] * 8
    a = np.zeros(5, dtype=np.int64); b = np.arange(5)
    lens, valid = pgq.iterativelength(st, 0, 5, a, b)
    assert lens.tolist() == [0, 1, 1, 1, -1] and valid.tolist() == [1, 1, 1, 1, 0]
    paths = pgq.shortestpath(st, 0, 5, a, b)
    assert paths == [[0], [0, 0, 1], [0, 1, 2], [0, 2, 3], None]
    assert 0 in st.csr_to_delete
    st.query_end()                       # duckpgq_state.cpp:162-170
    assert 0 not in st.csr_list
    with pytest.raises(pgq.ConstraintException, match="Invalid ID"):
        pgq.iterativelength(st, 0, 5, a, b)
    assert pgq.delete_csr(st, 0) is False


def test_constraint_exception_text(gpu_ctx):
    st = pgq.DuckPGQState(gpu_ctx)
    pgq.create_csr_vertex(st, 3, 3, [0, 1, 2], [1, 1, 0])
    with pytest.raises(pgq.ConstraintException, match="Non-existent/non-unique vertices detected"):
        pgq.create_csr_edge(st, 3, 3, 2, 3, [0, 1, 1], [1, 2, 0], [0, 1, 2])
    assert 3 in st.csr_to_delete
    st.query_end()


def test_out_of_range_ids_are_errors(gpu_ctx):
    csr = pgq.DeviceCSR.build(gpu_ctx, 4, [0, 1], [1, 2])
    with pytest.raises(pgq.InvalidInputException):
        csr.iterativelength([0], [4])
    with pytest.raises(pgq.InvalidInputException):
        pgq.DeviceCSR.build(gpu_ctx, 4, [0, 5], [1, 2])
    out, valid, _ = csr.iterativelength([9], [0], [0])  # NULL source rows are never looked at
    assert valid.tolist() == [0]
    csr.free()


def test_pruned_batching_work_counter(gpu_ctx):
    """With the degree shortcut on, W is the reference's W for the searches that still take a lane; with one
    lane per distinct source on top of it (the default), W is the restatement's for that lane assignment."""
    n, src, dst = datagen.rmat_edges(13)
    v, e, ids = orc.csr_build(n, src, dst)
    ps, pd = datagen.hashed_pairs(1500, n)
    csr = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    outdeg = np.diff(v[: n + 1])
    indeg = np.bincount(e, minlength=n)
    keep = (ps == pd) | ((outdeg[ps] > 0) & (indeg[pd] > 0))
    for lanes in (64, 256):
        out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes, no_dedup=True))
        exp, expv, ost = orc.iterativelength(n, v, e, ps[keep], pd[keep], None, lanes)
        assert np.array_equal(out[keep], exp) and np.array_equal(valid[keep], expv)
        assert not valid[~keep].any()
        assert (st["batches"], st["levels"], st["edges_traversed"]) == (ost.batches, ost.levels, ost.edges_traversed)
        assert st["pruned"] == int((~keep).sum())
        out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes))
        exp, expv, ost, used = orc.iterativelength_ex(n, v, e, ps, pd, None, lanes, prune=True, dedup=True)
        assert np.array_equal(out, exp) and np.array_equal(valid, expv)
        assert (st["searches"], st["batches"], st["levels"], st["edges_traversed"]) == (
            used, ost.batches, ost.levels, ost.edges_traversed)
    csr.free()


def test_one_lane_per_distinct_source(gpu_ctx):
    """The MATCH rewriter's cross product (match.cpp:476-487): 300 sources x 300 destinations = 90 000 rows.
    The reference burns 90 000 lanes (176 batches); one lane per distinct source needs 300 -- same rows."""
    rng = np.random.default_rng(77)
    n = 4000
    src, dst = rng.integers(0, n, 20000), rng.integers(0, n, 20000)
    v, e, ids = orc.csr_build(n, src, dst)
    csr = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    a, b = rng.choice(n, 300, replace=False), rng.choice(n, 300, replace=False)
    ps, pd = np.repeat(a, 300), np.tile(b, 300)
    perm = rng.permutation(len(ps))  # join output order: sources interleaved
    ps, pd = ps[perm], pd[perm]
    sv = (rng.random(len(ps)) > 0.01).astype(np.uint8)
    exp, expv, ost, used = orc.iterativelength_ex(n, v, e, ps, pd, sv, 256, dedup=True, omp=True)
    ref, refv, _, _ = orc.iterativelength_ex(n, v, e, ps[:5000], pd[:5000], sv[:5000], 512)  # the reference's own composition
    assert np.array_equal(exp[:5000], ref) and np.array_equal(expv[:5000], refv)
    out, valid, st = csr.iterativelength(ps, pd, sv, pgq.Options(256, no_prune=True))
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    assert st["searches"] == used == 300 and st["batches"] == 2
    assert (st["levels"], st["edges_traversed"]) == (ost.levels, ost.edges_traversed)
    out, valid, st = csr.iterativelength(ps, pd, sv)  # defaults
    assert np.array_equal(out, exp) and np.array_equal(valid, expv) and st["searches"] <= 300
    # paths: every row walks back through its source's lane
    sel = slice(0, 3000)
    epaths, _ = orc.shortestpath(n, v, e, ids, ps[sel], pd[sel], sv[sel], 512)
    paths, pst = csr.shortestpath(ps[sel], pd[sel], sv[sel])
    assert paths == epaths and pst["searches"] <= 300
    csr.free()


def test_empty_inputs(gpu_ctx):
    csr = pgq.DeviceCSR.build(gpu_ctx, 3, [], [])
    out, valid, st = csr.iterativelength([], [])
    assert out.shape == (0,)
    out, valid, _ = csr.iterativelength([0, 1], [0, 2])
    assert out.tolist() == [0, -1] and valid.tolist() == [1, 0]
    paths, _ = csr.shortestpath([0, 1], [0, 2])
    assert paths == [[0], None]
    csr.free()


@pytest.mark.parametrize("env", [{"PGQ_B200_NO_TAIL": "1"}, {"PGQ_B200_PULL_SKIP": "0"}, {"PGQ_B200_BATCH_STREAMS": "1"}])
def test_kernel_variants_agree(gpu_ctx, monkeypatch, env):
    """No k_tail, no skipping of finished rows in the bottom-up level, one stream: identical answers and identical
    work counters (the frontier sets do not depend on the kernels)."""
    cases = []
    for name in ("chain200", "rmat12", "snb0003_allpairs"):
        g = load_golden(name)
        cases.append((g, upload(gpu_ctx, g, with_ids=False)))
    n, src, dst, eid = datagen.snb_shaped_edges(2000, 24.0, seed=3)  # undirected: searches saturate
    v, e, ids = orc.csr_build(n, src, dst, eid)
    rng = np.random.default_rng(9)
    und = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    ups, upd = rng.integers(0, n, 400), rng.integers(0, n, 400)
    base = [csr.iterativelength(g["psrc"], g["pdst"], g["psrc_valid"], pgq.Options(64, d)) for g, csr in cases
            for d in (0, 2)]
    ubase = und.iterativelength(ups, upd, None, pgq.Options(128, 2))
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    got = [csr.iterativelength(g["psrc"], g["pdst"], g["psrc_valid"], pgq.Options(64, d)) for g, csr in cases
           for d in (0, 2)]
    ugot = und.iterativelength(ups, upd, None, pgq.Options(128, 2))
    for (o1, v1, s1), (o2, v2, s2) in zip(base + [ubase], got + [ugot]):
        assert np.array_equal(o1, o2) and np.array_equal(v1, v2)
        assert (s1["levels"], s1["edges_traversed"], s1["frontier_vertices"]) == (
            s2["levels"], s2["edges_traversed"], s2["frontier_vertices"])
    exp, expv, _ = orc.iterativelength(n, v, e, ups, upd, None, 128)
    assert np.array_equal(ugot[0], exp) and np.array_equal(ugot[1], expv)
    for _, csr in cases:
        csr.free()
    und.free()


def test_csr_build_from_device_columns(gpu_ctx):
    import torch
    n, src, dst = datagen.rmat_edges(12)
    d_src = torch.from_numpy(src.astype(np.int32)).cuda()
    d_dst = torch.from_numpy(dst.astype(np.int32)).cuda()
    csr = pgq.DeviceCSR.build_device(gpu_ctx, n, len(src), d_src.data_ptr(), d_dst.data_ptr())
    v, e, ids = csr.download()
    ov, oe, oids = orc.csr_build(n, src, dst)
    assert np.array_equal(v, ov) and np.array_equal(e, oe) and np.array_equal(ids, oids)
    csr.free()


def test_search_sharding_options(gpu_ctx):
    """pgq_options.shard_index / shard_count (the multi-GPU partition): the element-wise MAX of the
    shards' columns is the full answer, and the searches are dealt out evenly."""
    n, src, dst = datagen.rmat_edges(13)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    ps, pd = datagen.hashed_pairs(3000, n)
    sv = (np.arange(3000) % 17 != 0).astype(np.uint8)
    full, fvalid, fst = csr.iterativelength(ps, pd, sv)
    for count in (2, 3, 8):
        acc = np.full(3000, -1, dtype=np.int64)
        accv = np.zeros(3000, dtype=np.uint8)
        searches = []
        for idx in range(count):
            o, v, st = csr.iterativelength(ps, pd, sv, pgq.Options(shard_index=idx, shard_count=count))
            acc = np.maximum(acc, o)
            accv = np.maximum(accv, v)
            searches.append(st["searches"])
        assert np.array_equal(acc, full) and np.array_equal(accv, fvalid)
        assert sum(searches) == fst["searches"] and max(searches) - min(searches) <= 1
    with pytest.raises(pgq.InvalidInputException):
        csr.iterativelength(ps, pd, sv, pgq.Options(shard_index=3, shard_count=3))
    csr.free()


def test_concurrent_calls_share_one_csr(gpu_ctx):
    """DuckDB invokes the callbacks from several worker threads at once (one per 122 880-row row group);
    every call takes its own workspace + stream from the context's pool."""
    from concurrent.futures import ThreadPoolExecutor
    n, src, dst = datagen.rmat_edges(13)
    v, e, ids = orc.csr_build(n, src, dst)
    csr = pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)
    jobs = []
    for t in range(8):
        ps, pd = datagen.hashed_pairs(300 + 37 * t, n, first=1000 * t)
        jobs.append((ps, pd))

    def work(job):
        ps, pd = job
        out, valid, _ = csr.iterativelength(ps, pd, None, pgq.Options(64 if len(ps) % 2 else 256))
        paths, _ = csr.shortestpath(ps[:50], pd[:50])
        return out, valid, paths

    with ThreadPoolExecutor(max_workers=8) as pool:
        results = list(pool.map(work, jobs * 2))
    for (ps, pd), (out, valid, paths) in zip(jobs * 2, results):
        exp, expv, _ = orc.iterativelength(n, v, e, ps, pd, None, 512)
        assert np.array_equal(out, exp) and np.array_equal(valid, expv)
        epaths, _ = orc.shortestpath(n, v, e, ids, ps[:50], pd[:50], None, 64)
        assert paths == epaths
    csr.free()
