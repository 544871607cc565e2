"""reachability on the device CSR (pgq_reachability).

Default mode: the rows of pgq_iterativelength (a NULL destination counting as a NULL source), so answers and the
counters must be iterativelength's.  Reference batching: the reference's 512-lane batches, checked against the
oracle's loop-for-loop restatement (oracle/pgq_oracle_reach.c, defined batch start): answers, batches, levels and
edges_traversed exactly.  The goldens (tests/golden/refr_*.npz) hold the reference binary's rows."""
import glob
import os

import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb
from oracle import pgq_oracle_reach as orr

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "refr_*.npz")))
REF = pgq.Options(reference_batching=True)


@pytest.fixture(scope="module")
def ctx():
    return pgq.default_context(0)


def _both(sv, dv, p):
    ok = np.ones(p, np.uint8)
    if sv is not None:
        ok &= np.asarray(sv, np.uint8)
    if dv is not None:
        ok &= np.asarray(dv, np.uint8)
    return ok


def _check_ref(csr, n, src, dst, sv=None, dv=None, options=REF):
    v, e, _ = csr.download()
    out, valid, st = csr.reachability(src, dst, sv, dv, options)
    eo, ew, ost = orr.reachability(n, v, e, src, dst, sv, dv)
    assert np.array_equal(valid, ew), np.nonzero(valid != ew)[0][:10]
    assert np.array_equal(out, eo), np.nonzero(out != eo)[0][:10]
    assert (st["batches"], st["levels"], st["edges_traversed"]) == (ost.batches, ost.levels, ost.edges_traversed)
    assert st["lanes"] == 512
    return out, valid, st


def _check_default(csr, src, dst, sv=None, dv=None, options=None):
    p = len(src)
    out, valid, st = csr.reachability(src, dst, sv, dv, options)
    ok = _both(sv, dv, p)
    lo, lv, lst = csr.iterativelength(src, dst, ok if (sv is not None or dv is not None) else None, options)
    assert np.array_equal(valid, ok)
    assert np.array_equal(out, lv & ok)
    for k in ("batches", "levels", "edges_traversed", "searches", "pruned", "search_rows", "lanes"):
        assert st[k] == lst[k], k
    return out, valid, st


def _pairs(n, p, seed, nulls=True):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, max(n, 1), p)
    dst = rng.integers(0, max(n, 1), p)
    if p > 4:
        dst[::7] = src[::7]
        src[3::11] = src[0]
    sv = dv = None
    if nulls:
        sv = (rng.random(p) > 0.05).astype(np.uint8)
        dv = (rng.random(p) > 0.05).astype(np.uint8)
    return src, dst, sv, dv


def _graph(name):
    scale = int(name[4:6])
    n, s, d = datagen.rmat_edges(scale, seed=scale)
    if name.endswith("u"):
        s, d = np.concatenate([s, d]), np.concatenate([d, s])
    return n, s, d


# ---- the reference binary's rows ----------------------------------------------------------------------------------

def _routes(ctx, route, n, src, dst):
    if route == "build":
        return pgq.DeviceCSR.build(ctx, n, src, dst)
    if route == "upload":
        v, e, ids = orc.csr_build(n, src, dst)
        return pgq.DeviceCSR.upload(ctx, n, v, e, ids)
    return pgq.DeviceCSR.build_from_keys(ctx, np.arange(n, dtype=np.int64) * 3 + 7, src * 3 + 7, dst * 3 + 7)


def test_goldens_present():
    assert len(GOLDEN) >= 12


@pytest.mark.parametrize("route", ["build", "upload", "keys"])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[5:-4] for p in GOLDEN])
def test_golden(ctx, path, route):
    z = np.load(path)
    n = int(z["n"])
    src, dst = z["src"].astype(np.int64), z["dst"].astype(np.int64)
    es, ed = z["eff_src"].astype(np.int64), z["eff_dst"].astype(np.int64)
    sv, dv = z["src_valid"], z["dst_valid"]
    ok = (sv & dv).astype(bool)
    csr = _routes(ctx, route, n, src, dst)
    try:
        for options in (REF, None):
            out, valid, _ = csr.reachability(es, ed, sv, dv, options)
            assert np.array_equal(valid.astype(bool), ok)
            # is_variant = false: the answers do not depend on the batches, re-run rows included
            assert np.array_equal(out[ok], z["reach0"][ok])
        _check_ref(csr, n, es, ed, sv, dv)
    finally:
        csr.free()


# ---- default mode = iterativelength's rows -----------------------------------------------------------------------

@pytest.mark.parametrize("name", ["rmat10", "rmat12", "rmat12u", "rmat14"])
@pytest.mark.parametrize("opt", ["auto", "lanes64", "lanes256", "no_dedup", "no_prune", "push", "pull"])
def test_default_equals_iterativelength(ctx, name, opt):
    n, s, d = _graph(name)
    options = {"auto": None, "lanes64": pgq.Options(64), "lanes256": pgq.Options(256),
               "no_dedup": pgq.Options(no_dedup=True), "no_prune": pgq.Options(no_prune=True),
               "push": pgq.Options(direction=1), "pull": pgq.Options(direction=2)}[opt]
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        ps, pd = datagen.hashed_pairs(2048, n)
        _check_default(csr, ps, pd, options=options)
        _check_default(csr, *_pairs(n, 2048, n), options=options)
    finally:
        csr.free()


# ---- reference batching = the restatement ------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["rmat10", "rmat10u", "rmat12", "rmat12u", "rmat14", "rmat14u", "rmat16"])
def test_reference_batching_on_rmat(ctx, name):
    n, s, d = _graph(name)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        ps, pd = datagen.hashed_pairs(2048, n)
        _, _, st = _check_ref(csr, n, ps, pd)
        assert st["batches"] == len(orr.reference_batch_starts(ps)) >= 2
        _check_ref(csr, n, *_pairs(n, 2048, n))
        # the counters are the plain traversal's: a lane's seen set = its source + what it reaches
        out, _, _ = csr.reachability(ps, pd)
        ref_out, _, _ = csr.reachability(ps, pd, options=REF)
        assert np.array_equal(out, ref_out)
    finally:
        csr.free()


@pytest.fixture(scope="module")
def rmat12(ctx):
    n, s, d = datagen.rmat_edges(12, seed=12)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    yield n, csr
    csr.free()


@pytest.mark.parametrize("k", [1, 511, 512, 513, 1024, 1025])
def test_distinct_sources_around_the_batch(rmat12, k):
    n, csr = rmat12
    rng = np.random.default_rng(k)
    src = rng.permutation(n)[:k]
    dst = rng.integers(0, n, k)
    _, _, st = _check_ref(csr, n, src, dst)
    assert st["batches"] == (k + 511) // 512 and st["searches"] == k


def test_repeated_source_across_the_boundary(rmat12):
    """Sources 0 .. 511 fill the first batch; rows with sources 0 and 5 behind it open lanes in the second one, and a
    source repeated inside a batch shares its lane."""
    n, csr = rmat12
    src = np.concatenate([np.arange(512), [0, 5, 0, 5, 7]])
    dst = np.concatenate([np.arange(512)[::-1], [1, 2, 3, 4, 7]])
    out, _, st = _check_ref(csr, n, src, dst)
    assert st["batches"] == 2 and st["searches"] == 512 + 3 and st["search_rows"] == len(src)
    assert out[-1] == 1


def test_trivial_rows_take_lanes(rmat12):
    n, csr = rmat12
    # only src == dst rows, 600 distinct sources: two batches, every row true
    src = np.arange(600)
    out, valid, st = _check_ref(csr, n, src, src.copy())
    assert out.all() and valid.all() and st["batches"] == 2 and st["searches"] == 600
    # without the reference's batches they need no lane
    out, valid, st = _check_default(csr, src, src.copy())
    assert out.all() and st["searches"] == 0
    # a trivial row's source is the lane of the non-trivial rows after it
    src = np.array([3, 3, 9, 3])
    dst = np.array([3, 100, 9, 200])
    _, _, st = _check_ref(csr, n, src, dst)
    assert st["searches"] == 2 and st["batches"] == 1


def test_empty_call(rmat12):
    _, csr = rmat12
    for options in (REF, None):
        out, valid, st = csr.reachability(np.zeros(0, np.int64), np.zeros(0, np.int64), options=options)
        assert len(out) == 0 and len(valid) == 0 and st["batches"] == 0 and st["levels"] == 0


def test_null_sources_and_destinations(rmat12):
    n, csr = rmat12
    rng = np.random.default_rng(1)
    for p in (600, 1100, 2048):
        src, dst = rng.integers(0, n, p), rng.integers(0, n, p)
        src = rng.permutation(n)[:p] if p <= n else src
        sv = (rng.random(p) > 0.1).astype(np.uint8)
        dv = (rng.random(p) > 0.1).astype(np.uint8)
        sv[-1] = 0  # a trailing NULL source: the reference would never finish
        dst[dv == 0] = n + 5  # under a NULL the value is not read
        out, valid, st = _check_ref(csr, n, src, dst, sv, dv)
        assert not valid[sv == 0].any() and not valid[dv == 0].any() and not out[valid == 0].any()
        # NULL sources take no lane, NULL destinations keep theirs
        assert st["searches"] == len(np.unique(src[sv == 1]))
        _check_default(csr, src, dst, sv, dv)
    # all NULL
    z = np.zeros(5, np.uint8)
    for options in (REF, None):
        out, valid, st = csr.reachability(np.arange(5), np.arange(5), z, None, options)
        assert not valid.any() and st["batches"] == 0


def test_errors(rmat12):
    n, csr = rmat12
    good = np.array([0, 1]), np.array([1, 2])
    for options in (REF, None):
        for src, dst in ((np.array([0, n]), np.array([1, 2])), (np.array([0, 1]), np.array([-1, 2]))):
            with pytest.raises(pgq.InvalidInputException) as ex:
                csr.reachability(src, dst, options=options)
            assert ex.value.status == pgq.PGQ_ERR_RANGE
        with pytest.raises(pgq.PgqError) as ex:
            csr.reachability(*good, options=pgq.Options(shard_index=0, shard_count=2,
                                                        reference_batching=options is REF))
        assert ex.value.status == pgq.PGQ_ERR_UNSUPPORTED
        # a NULL id is not checked
        out, valid, _ = csr.reachability(np.array([n + 1, 0]), np.array([0, -4]), np.array([0, 1], np.uint8),
                                         np.array([1, 0], np.uint8), options)
        assert not valid.any()
    for lanes in (64, 128, 256, 100):
        with pytest.raises(pgq.InvalidInputException) as ex:
            csr.reachability(*good, options=pgq.Options(lanes, reference_batching=True))
        assert ex.value.status == pgq.PGQ_ERR_INVALID_ARG
    _check_ref(csr, n, *good, options=pgq.Options(512, reference_batching=True))


@pytest.mark.parametrize("schedule", ["b", "p", "t", "bp", "pb", "tbp", "ppb"])
def test_forced_schedules(ctx, monkeypatch, schedule):
    monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
    for name in ("rmat12", "rmat12u"):
        n, s, d = _graph(name)
        csr = pgq.DeviceCSR.build(ctx, n, s, d)
        try:
            _check_ref(csr, n, *_pairs(n, 1300, 3))
            _check_default(csr, *_pairs(n, 1300, 4))
        finally:
            csr.free()


def test_dirty_workspace(ctx):
    """One context, calls of every BFS consumer in turn on two CSRs: each must find its workspace as it needs it."""
    graphs = [_graph("rmat12"), _graph("rmat10u")]
    csrs = [pgq.DeviceCSR.build(ctx, n, s, d) for n, s, d in graphs]
    try:
        hv = [c.download() for c in csrs]
        for rnd in range(3):
            for k, ((n, _, _), csr, (v, e, ids)) in enumerate(zip(graphs, csrs, hv)):
                src, dst, sv, dv = _pairs(n, 1500, 10 * rnd + k)
                _check_ref(csr, n, src, dst, sv, dv)
                lo, lv, _ = csr.iterativelength(src, dst, sv)
                eo, ev, _ = orc.iterativelength(n, v, e, src, dst, sv, 512)
                assert np.array_equal(lv, ev) and np.array_equal(lo[lv == 1], eo[ev == 1])
                _check_default(csr, src, dst, sv, dv)
                paths, _ = csr.shortestpath(src[:300], dst[:300])
                epaths, _ = orc.shortestpath(n, v, e, ids, src[:300], dst[:300])
                assert paths == epaths
                bo, bv, _ = csr.iterativelengthbidirectional(src, dst, sv, dv)
                ebo, ebv, _ = orb.iterativelengthbidirectional(n, v, e, src, dst, sv, dv, 512)
                assert np.array_equal(bv, ebv) and np.array_equal(bo, ebo)
                _check_ref(csr, n, src, dst, sv, dv)
    finally:
        for c in csrs:
            c.free()


def test_sql_mirror(ctx):
    n, s, d = datagen.rmat_edges(9, seed=2)
    state = pgq.DuckPGQState(ctx)
    state.csr_list[0] = pgq.DeviceCSR.build(ctx, n, s, d)
    src, dst, sv, dv = _pairs(n, 700, 9)
    out, valid = pgq.reachability(state, 0, True, n, src, dst, sv, dv)
    v, e, _ = state.csr_list[0].download()
    eo, ew, _ = orr.reachability(n, v, e, src, dst, sv, dv)
    assert out.dtype == bool and np.array_equal(valid, ew) and np.array_equal(out, eo.astype(bool))
    assert 0 in state.csr_to_delete
    with pytest.raises(pgq.ConstraintException, match="CSR not found with ID 3"):
        pgq.reachability(state, 3, False, n, src, dst)
    with pytest.raises(pgq.InvalidInputException):
        pgq.reachability(state, 0, False, n + 1, src, dst)
    state.query_end()
