"""iterativelengthbidirectional on the device CSR against the oracle's loop-for-loop restatement, at 512 lanes.

Results, validity and the counters batches / levels (= iterations of both sides) / edges_traversed must be the
oracle's exactly: the answers of a batch are coupled (a lane that has met keeps expanding and keeps the batch alive), so
any difference in lane composition, iteration order or the stopping rule shows up here."""
import glob
import os
import re

import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "refb_*.npz")))
TRACE = re.compile(r"\[pgq\] batch (\d+) iteration (\d+) (src|dst) side (push|pull|tail)")


@pytest.fixture(scope="module")
def ctx():
    return pgq.default_context(0)


def _pairs(n, p, seed, nulls=True):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, max(n, 1), p)
    dst = rng.integers(0, max(n, 1), p)
    if p > 4:
        dst[::7] = src[::7]              # src == dst
        src[3::11], dst[3::11] = src[0], dst[0]  # repeated pairs
    sv = dv = None
    if nulls:
        sv = (rng.random(p) > 0.05).astype(np.uint8)
        dv = (rng.random(p) > 0.05).astype(np.uint8)
    return src, dst, sv, dv


def _check(csr, n, src, dst, sv=None, dv=None, options=None):
    v, e, _ = csr.download()
    out, valid, st = csr.iterativelengthbidirectional(src, dst, sv, dv, options)
    eo, ev, ost = orb.iterativelengthbidirectional(n, v, e, src, dst, sv, dv, 512)
    assert np.array_equal(valid, ev), np.nonzero(valid != ev)[0][:10]
    assert np.array_equal(out, eo), np.nonzero(out != eo)[0][:10]
    assert (st["batches"], st["levels"], st["edges_traversed"]) == (ost.batches, ost.iterations, ost.edges_traversed)
    assert st["lanes"] == 512
    return out, valid


def _undirected(src, dst):
    return np.concatenate([src, dst]), np.concatenate([dst, src])


def _graph(name):
    if name.startswith("rmat"):
        scale = int(name[4:6])
        n, s, d = datagen.rmat_edges(scale, seed=scale)
        return (n,) + (_undirected(s, d) if name.endswith("u") else (s, d))
    if name == "star":
        n = 3000
        return n, np.zeros(n - 1, np.int64), np.arange(1, n)
    if name == "path":
        n = 1500
        return n, np.arange(n - 1), np.arange(1, n)
    if name == "edgeless":
        return 50, np.zeros(0, np.int64), np.zeros(0, np.int64)
    if name == "loops":  # self-loops and parallel edges
        rng = np.random.default_rng(5)
        n = 700
        s = rng.integers(0, n, 4000)
        d = rng.integers(0, n, 4000)
        s = np.concatenate([s, s[:500], np.arange(0, n, 3)])
        d = np.concatenate([d, d[:500], np.arange(0, n, 3)])
        return n, s, d
    raise KeyError(name)


GRAPHS = ["rmat10", "rmat10u", "rmat12", "rmat12u", "rmat14", "rmat14u", "rmat16", "rmat16u", "star", "path",
          "edgeless", "loops"]


@pytest.mark.parametrize("name", GRAPHS)
def test_generated_graphs(ctx, name):
    n, s, d = _graph(name)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        src, dst, sv, dv = _pairs(n, 2048, GRAPHS.index(name))
        _check(csr, n, src, dst, sv, dv)
    finally:
        csr.free()


@pytest.mark.parametrize("p", [1, 2, 63, 511, 512, 513, 1024, 1100, 2048])
def test_multi_batch_rows(ctx, p):
    n, s, d = datagen.rmat_edges(11, seed=3)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        _check(csr, n, *_pairs(n, p, p))
        _check(csr, n, *_pairs(n, p, p + 1, nulls=False))
    finally:
        csr.free()


def test_coupling_across_lanes(ctx):
    """Row X = (a, b) with a sink source and the edge b -> a: alone its source side dies at iteration 0 and it is NULL;
    next to a row Y whose source side keeps growing, the destination side reaches a at iteration 1 and X is 2."""
    n = 10
    a, b, c, d2 = 0, 1, 2, 3
    csr = pgq.DeviceCSR.build(ctx, n, np.array([b, c, d2, 4]), np.array([a, d2, 4, 5]))
    try:
        out, valid = _check(csr, n, np.array([a]), np.array([b]))
        assert valid[0] == 0
        out, valid = _check(csr, n, np.array([c, a]), np.array([9, b]))
        assert valid[1] == 1 and out[1] == 2
        # the same rows in different batches: X is in the second batch alone again
        src = np.concatenate([[c], np.full(511, c), [a]])
        dst = np.concatenate([[9], np.full(511, 8), [b]])
        out, valid = _check(csr, n, src, dst)
        assert valid[-1] == 0
    finally:
        csr.free()


@pytest.mark.parametrize("route", ["build", "build_device", "upload", "create", "keys", "clone"])
def test_construction_routes(ctx, route):
    import torch
    n, s, d = datagen.rmat_edges(12, seed=12)
    base = pgq.DeviceCSR.build(ctx, n, s, d)
    v, e, _ = base.download()  # (upload's input)
    if route == "build":
        csr = pgq.DeviceCSR.build(ctx, n, s, d)
    elif route == "build_device":
        ts = torch.as_tensor(s, dtype=torch.int32, device="cuda:0")
        td = torch.as_tensor(d, dtype=torch.int32, device="cuda:0")
        csr = pgq.DeviceCSR.build_device(ctx, n, len(s), ts.data_ptr(), td.data_ptr())
        torch.cuda.synchronize()
    elif route == "upload":
        csr = pgq.DeviceCSR.upload(ctx, n, v, e)
    elif route == "create":
        csr = pgq.DeviceCSR.create(ctx, n)
        csr.add_vertex_counts(np.arange(n), np.bincount(s, minlength=n))
        for o in range(0, len(s), 2048):
            csr.add_edges(len(s), len(s), s[o:o + 2048], d[o:o + 2048], np.arange(o, min(o + 2048, len(s))))
        csr.finalize()
    elif route == "keys":
        keys = np.arange(n, dtype=np.int64) * 7 + 3
        csr = pgq.DeviceCSR.build_from_keys(ctx, keys, keys[s], keys[d])
    else:
        csr = base.clone(ctx)
    try:
        dv_, de_, _ = csr.download()
        assert np.array_equal(dv_, v) and np.array_equal(np.sort(de_), np.sort(e))
        _check(csr, n, *_pairs(n, 1500, 7))
    finally:
        csr.free()
        base.free()


@pytest.mark.parametrize("schedule", ["b", "p", "t", "a", "bp", "pb"])
@pytest.mark.parametrize("name", ["rmat12", "rmat12u", "loops", "path"])
def test_forced_schedules(ctx, monkeypatch, capfd, name, schedule):
    monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    n, s, d = _graph(name)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        capfd.readouterr()
        _check(csr, n, *_pairs(n, 1100, 11))
        lines = [TRACE.match(x) for x in capfd.readouterr().err.splitlines()]
        lines = [x for x in lines if x]
        assert lines
        for mt in lines:
            it, side, kind = int(mt.group(2)), mt.group(3), mt.group(4)
            assert side == ("dst" if it & 1 else "src")
            want = schedule[it % len(schedule)]
            if want == "p":
                assert kind == "push"
            elif want == "b" and len(s) > 0:
                assert kind == "pull"
    finally:
        csr.free()


@pytest.mark.parametrize("direction", [0, 1, 2])
def test_directions_and_undirected_equals_iterativelength(ctx, direction):
    n, s, d = datagen.rmat_edges(13, seed=13)
    s, d = _undirected(s, d)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        src, dst, sv, _ = _pairs(n, 2048, 13)
        out, valid = _check(csr, n, src, dst, sv, None, pgq.Options(512, direction=direction))
        lo, lv, _ = csr.iterativelength(src, dst, sv)
        assert np.array_equal(valid, lv) and np.array_equal(out, lo)
    finally:
        csr.free()


def test_interleaved_with_other_consumers(ctx):
    n, s, d = datagen.rmat_edges(12, seed=4)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    v, e, ids = csr.download()
    try:
        src, dst, sv, dv = _pairs(n, 1300, 21)
        for rnd in range(2):
            _check(csr, n, src, dst, sv, dv)
            out, valid, st = csr.iterativelength(src, dst, sv, pgq.Options(512, reference_batching=True))
            eo, ev, _ = orc.iterativelength(n, v, e, src, dst, sv, 512)
            assert np.array_equal(out, eo) and np.array_equal(valid, ev)
            _check(csr, n, src[:700], dst[:700])
            paths, _ = csr.shortestpath(src[:100], dst[:100])
            epaths, _ = orc.shortestpath(n, v, e, ids, src[:100], dst[:100])
            assert paths == epaths
            out, valid, _ = csr.iterativelength(src, dst, sv)
            assert np.array_equal(out, eo) and np.array_equal(valid, ev)
            csr.local_clustering_coefficient(np.arange(min(n, 300)))
    finally:
        csr.free()


def test_abi_errors(ctx):
    n, s, d = datagen.rmat_edges(8, seed=8)
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    try:
        src, dst = np.array([0, 1]), np.array([2, 3])
        for lanes in (64, 128, 256, 100):
            with pytest.raises(pgq.PgqError) as ei:
                csr.iterativelengthbidirectional(src, dst, options=pgq.Options(lanes))
            assert ei.value.status == pgq.PGQ_ERR_INVALID_ARG
        with pytest.raises(pgq.PgqError) as ei:
            csr.iterativelengthbidirectional(src, dst, options=pgq.Options(512, reference_batching=True))
        assert ei.value.status == pgq.PGQ_ERR_UNSUPPORTED
        with pytest.raises(pgq.PgqError) as ei:
            csr.iterativelengthbidirectional(src, dst, options=pgq.Options(512, shard_index=0, shard_count=2))
        assert ei.value.status == pgq.PGQ_ERR_UNSUPPORTED
        with pytest.raises(pgq.PgqError) as ei:
            csr.iterativelengthbidirectional(np.array([0]), np.array([n]))
        assert ei.value.status == pgq.PGQ_ERR_RANGE
        with pytest.raises(pgq.PgqError) as ei:
            csr.iterativelengthbidirectional(np.array([-1]), np.array([0]))
        assert ei.value.status == pgq.PGQ_ERR_RANGE
        # out-of-range ids under a NULL, and src == dst, take no lane and raise nothing
        out, valid, _ = csr.iterativelengthbidirectional(np.array([n + 5, 3]), np.array([0, 3]), np.array([0, 1]))
        assert list(valid) == [0, 1] and list(out) == [-1, 0]
    finally:
        csr.free()
    fresh = pgq.DeviceCSR.create(ctx, 10)
    try:
        with pytest.raises(pgq.PgqError) as ei:
            fresh.iterativelengthbidirectional(np.array([0]), np.array([1]))
        assert ei.value.status == pgq.PGQ_ERR_NOT_INITIALIZED
    finally:
        fresh.free()


def test_module_function_lookup_texts(ctx):
    state = pgq.DuckPGQState(ctx)
    with pytest.raises(pgq.ConstraintException, match="Invalid ID"):
        pgq.iterativelengthbidirectional(state, 0, 10, np.array([0]), np.array([1]))
    n, s, d = datagen.rmat_edges(9, seed=9)
    state.csr_list[0] = pgq.DeviceCSR.build(ctx, n, s, d)
    src, dst, sv, dv = _pairs(n, 600, 9)
    out, valid = pgq.iterativelengthbidirectional(state, 0, n, src, dst, sv, dv)
    v, e, _ = state.csr_list[0].download()
    eo, ev, _ = orb.iterativelengthbidirectional(n, v, e, src, dst, sv, dv)
    assert np.array_equal(out, eo) and np.array_equal(valid, ev)
    assert 0 in state.csr_to_delete
    state.query_end()


def _golden_csr(ctx, route, n, s, d):
    if route == "build":
        return pgq.DeviceCSR.build(ctx, n, s, d)
    if route == "build_device":
        import torch
        ts = torch.as_tensor(s, dtype=torch.int32, device="cuda:0")
        td = torch.as_tensor(d, dtype=torch.int32, device="cuda:0")
        csr = pgq.DeviceCSR.build_device(ctx, n, len(s), ts.data_ptr(), td.data_ptr())
        torch.cuda.synchronize()
        return csr
    if route == "upload":
        v, e, _ = orc.csr_build(n, s, d)
        return pgq.DeviceCSR.upload(ctx, n, v, e)
    if route == "create":
        csr = pgq.DeviceCSR.create(ctx, n)
        csr.add_vertex_counts(np.arange(n), np.bincount(s, minlength=n))
        for o in range(0, len(s), 2048):
            csr.add_edges(len(s), len(s), s[o:o + 2048], d[o:o + 2048], np.arange(o, min(o + 2048, len(s))))
        csr.finalize()
        return csr
    keys = np.arange(n, dtype=np.int64) * 5 + 11
    return pgq.DeviceCSR.build_from_keys(ctx, keys, keys[s], keys[d])


@pytest.mark.parametrize("route", ["build", "build_device", "upload", "create", "keys"])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[5:-4] for p in GOLDEN])
def test_reference_goldens(ctx, path, route):
    """The reference binary's rows (tests/golden/make_golden_bidir.py: the ids it searched are the byte view of its key
    columns, eff_src / eff_dst), for CSRs from every construction route; counters against the restatement."""
    z = np.load(path)
    n = int(z["n"])
    s, d = z["src"].astype(np.int64), z["dst"].astype(np.int64)
    if len(s) == 0 and route in ("build_device", "create"):
        pytest.skip("no edge rows to feed this route")
    csr = _golden_csr(ctx, route, n, s, d)
    try:
        src, dst = z["eff_src"].astype(np.int64), z["eff_dst"].astype(np.int64)
        out, valid = _check(csr, n, src, dst, z["src_valid"])
        assert np.array_equal(valid, z["length_valid"])
        assert np.array_equal(out, z["length"].astype(np.int64))
    finally:
        csr.free()


def test_empty_trailing_batch_is_counted(ctx):
    """1024 lane rows followed by trivial and NULL rows: the reference's loop starts a third batch that finds no lane."""
    n = 10
    csr = pgq.DeviceCSR.build(ctx, n, np.array([1, 2, 3, 4]), np.array([0, 3, 4, 5]))
    try:
        src = np.concatenate([np.full(1024, 2), np.full(100, 5), np.full(30, 1)])
        dst = np.concatenate([np.full(1024, 8), np.full(100, 5), np.full(30, 0)])
        sv = np.concatenate([np.ones(1124, np.uint8), np.zeros(30, np.uint8)])
        _check(csr, n, src, dst, sv)
        _, _, st = csr.iterativelengthbidirectional(src, dst, sv)
        assert st["batches"] == 3
        _, _, st = csr.iterativelengthbidirectional(src[:1024], dst[:1024])
        assert st["batches"] == 2
    finally:
        csr.free()
