"""BASELINE.json's full-size configurations, checked through size-independent properties (the
oracle needs minutes there): independence of lane width / direction / batch composition, path
validity against the CSR, hop count == path length, plus a direct oracle comparison on a sample
small enough for the CPU."""
import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc

pytestmark = pytest.mark.gpu


def check_paths_valid(v, e, ids, ps, pd, paths, lengths, valid):
    """every hop of every path is a CSR edge carrying that edge id; len(path)//2 == hop count"""
    for s, d, path, ln, ok in zip(ps, pd, paths, lengths, valid):
        if path is None:
            assert not ok
            continue
        assert ok and len(path) == 2 * ln + 1 and path[0] == s and path[-1] == d
        for k in range(ln):
            a, eid, b = path[2 * k], path[2 * k + 1], path[2 * k + 2]
            row = slice(v[a], v[a + 1])
            hits = np.nonzero((e[row] == b) & (ids[row] == eid))[0]
            assert hits.size > 0, (a, eid, b)


def test_c2_rmat22_1024_pairs(gpu_ctx):
    """configs[1]: RMAT scale-22 (4M v / 64M e), 1024 hashed pairs, 1 x H100."""
    n, src, dst = datagen.rmat_edges_cached(22)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    ps, pd = datagen.hashed_pairs(1024, n)
    ps[5] = pd[5]  # a src == dst row
    base, bvalid, st = csr.iterativelength(ps, pd)
    assert base[5] == 0 and bvalid[5] == 1
    assert 150 < int(bvalid.sum()) < 400  # ~ 23 % of hashed pairs are connected on directed R-MAT
    for opts in (pgq.Options(64), pgq.Options(512), pgq.Options(256, 1), pgq.Options(256, 2),
                 pgq.Options(128, reference_batching=True)):
        out, valid, st2 = csr.iterativelength(ps, pd, None, opts)
        assert np.array_equal(out, base) and np.array_equal(valid, bvalid), opts
    # the restatement on a 64-pair sample (one batch) -- incl. the work counter W
    v, e, ids = csr.download()
    exp, expv, ost = orc.iterativelength(n, v, e, ps[:64], pd[:64], None, 64)
    out, valid, st3 = csr.iterativelength(ps[:64], pd[:64], None, pgq.Options(64, reference_batching=True))
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    assert st3["edges_traversed"] == ost.edges_traversed and st3["levels"] == ost.levels
    # paths for the first 128 pairs: valid edges, same lengths
    paths, _ = csr.shortestpath(ps[:128], pd[:128], None, pgq.Options(64))
    check_paths_valid(v, e, ids, ps[:128], pd[:128], paths, base[:128], bvalid[:128])
    csr.free()


def test_c4_snb_shaped_sf10_shortestpath(gpu_ctx):
    """configs[3]: SNB-shaped SF10 Person-knows-Person (65 645 v, ~3.9 M directed edge rows of the
    undirected CSR), ANY SHORTEST with path reconstruction for 2048 pairs."""
    n, src, dst, eid = datagen.snb_shaped_edges()
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst, eid)
    v, e, ids = csr.download()
    rng = np.random.default_rng(10)
    ps, pd = rng.integers(0, n, 2048), rng.integers(0, n, 2048)
    lengths, valid, _ = csr.iterativelength(ps, pd)
    paths, st = csr.shortestpath(ps, pd)
    check_paths_valid(v, e, ids, ps, pd, paths, lengths, valid)
    paths2, _ = csr.shortestpath(ps, pd, None, pgq.Options(64, 1, reference_batching=True))
    assert paths2 == paths  # tie-break independent of lanes / direction / batching
    # exact equality with the restatement on a sample (the reference's tie-break)
    exp, _ = orc.shortestpath(n, v, e, ids, ps[:64], pd[:64], None, 64)
    assert paths[:64] == exp
    csr.free()


def _device_rmat_csr(gpu_ctx, scale):
    import torch
    n, src, dst = datagen.rmat_edges_device(scale)
    torch.cuda.synchronize()
    csr = pgq.DeviceCSR.build_device(gpu_ctx, n, src.numel(), src.data_ptr(), dst.data_ptr())
    del src, dst
    torch.cuda.empty_cache()
    return n, csr


def _oracle_sample(n, csr, ps, pd, lanes, count):
    """Exact equality with the restatement (OpenMP level loop: same results and counters, see
    oracle/pgq_oracle.c) for the first `count` rows under the reference's batch composition, lengths AND
    the work counters W / levels."""
    v, e, _ = csr.download_ve()
    exp, expv, ost, _ = orc.iterativelength_ex(n, v, e, ps[:count], pd[:count], None, lanes, omp=True)
    out, valid, st = csr.iterativelength(ps[:count], pd[:count], None, pgq.Options(lanes, reference_batching=True))
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
        ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices)
    return v, e


def test_c2_rmat22_all_pairs_vs_oracle(gpu_ctx):
    """configs[1] again, every one of the 1024 pairs against the restatement (two 512-lane batches with the
    reference's batch composition, OpenMP level loop), incl. W and the level count."""
    n, src, dst = datagen.rmat_edges_cached(22)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    ps, pd = datagen.hashed_pairs(1024, n)
    v, e = _oracle_sample(n, csr, ps, pd, 512, 1024)
    # the default composition (degree shortcut + one lane per distinct source) recomputed by the oracle
    exp, expv, ost, lanes_used = orc.iterativelength_ex(n, v, e, ps, pd, None, 256, prune=True, dedup=True, omp=True)
    out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(256))
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    assert st["searches"] == lanes_used and st["edges_traversed"] == ost.edges_traversed and st["levels"] == ost.levels
    csr.free()


def test_c3_rmat24_4096_pairs(gpu_ctx):
    """configs[2]'s graph and pair set on one GPU: RMAT scale-24 (16.8M v / 268M e, built on the device),
    4096 hashed pairs; lane-width / direction / batching invariance, and one 256-lane batch + the first
    1024 rows against the restatement."""
    n, csr = _device_rmat_csr(gpu_ctx, 24)
    ps, pd = datagen.hashed_pairs(4096, n)
    base, bvalid, st = csr.iterativelength(ps, pd)
    assert 600 < int(bvalid.sum()) < 1600
    for opts in (pgq.Options(64), pgq.Options(512), pgq.Options(256, 2), pgq.Options(128, reference_batching=True)):
        out, valid, _ = csr.iterativelength(ps, pd, None, opts)
        assert np.array_equal(out, base) and np.array_equal(valid, bvalid), opts
    out, valid, _ = csr.iterativelength(ps[:512], pd[:512], None, pgq.Options(256, 1))  # top-down only
    assert np.array_equal(out, base[:512]) and np.array_equal(valid, bvalid[:512])
    v, e = _oracle_sample(n, csr, ps, pd, 256, 1024)
    exp, expv, _, _ = orc.iterativelength_ex(n, v, e, ps, pd, None, 512, prune=True, dedup=True, omp=True)
    assert np.array_equal(base, exp) and np.array_equal(bvalid, expv)  # all 4096 pairs
    csr.free()


def test_c5_rmat26_512_lanes(gpu_ctx):
    """configs[4] at single-GPU size: RMAT scale-26 (67M v / 1.07G e; positions beyond 2^30 exercise the
    int32 adjacency offsets), one 512-lane multi-source BFS; lane-width invariance and a 64-lane batch
    with the reference's batch composition against the restatement (lengths, W, levels)."""
    n, csr = _device_rmat_csr(gpu_ctx, 26)
    ps, pd = datagen.hashed_pairs(512, n)
    base, bvalid, st = csr.iterativelength(ps, pd, None, pgq.Options(512, reference_batching=True))
    assert st["batches"] == 1 and st["lanes"] == 512
    for opts in (pgq.Options(0), pgq.Options(128), pgq.Options(256, 2)):
        out, valid, _ = csr.iterativelength(ps, pd, None, opts)
        assert np.array_equal(out, base) and np.array_equal(valid, bvalid), opts
    v, e = _oracle_sample(n, csr, ps, pd, 64, 64)
    del v, e
    csr.free()
