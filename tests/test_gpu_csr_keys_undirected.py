"""pgq_csr_build_keys_undirected / _device: the undirected CSR CTE over key columns on the device, against the oracle's
restatement (oracle/pgq_oracle_keys_undirected), the reference's own output (tests/golden/refu_*.npz), pgq_csr_build
and the consumers of the CSR."""
import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb
from oracle import pgq_oracle_keys_undirected as orcu
from oracle import pgq_oracle_reach as orr
from test_oracle_keys_undirected_golden import load_undirected_golden, rows_as_sets, undirected_golden_names

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def build_both(ctx, vkey, src, dst, vvalid=None, svalid=None, dvalid=None):
    """(device arrays, oracle arrays); both sides raise their ConstraintException alike"""
    try:
        ref = orcu.csr_build_keys_undirected(vkey, src, dst, vvalid, svalid, dvalid)
    except orc.ConstraintError:
        ref = None
    if ref is None:
        with pytest.raises(pgq.ConstraintException) as ex:
            pgq.DeviceCSR.build_from_keys(ctx, vkey, src, dst, vvalid, svalid, dvalid, undirected=True)
        assert str(ex.value) == orc.CONSTRAINT_TEXT
        return None, None
    csr = pgq.DeviceCSR.build_from_keys(ctx, vkey, src, dst, vvalid, svalid, dvalid, undirected=True)
    got = csr.download()
    csr.free()
    return got, ref


def assert_same(got, ref):
    for a, b in zip(got, ref):
        assert np.asarray(a).dtype == np.asarray(b).dtype and np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _cases():
    rng = np.random.default_rng(8)
    out = {}
    for name in undirected_golden_names():
        g = load_undirected_golden(name)
        out[f"golden_{name}"] = (g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    keys = rng.permutation(3000) * 7 - 9000
    out["random20000"] = (keys, rng.choice(keys, 20000), rng.choice(keys, 20000), None, None, None)
    keys = rng.permutation(200)
    s = rng.choice(keys[:40], 6000)
    out["heavy_duplication"] = (keys, s, np.where(rng.random(6000) < 0.5, s, rng.choice(keys[:40], 6000)), None, None,
                                None)
    out["empty_edges"] = (keys, [], [], None, None, None)
    out["empty_vertex_table"] = ([], [1, 2], [2, 1], None, None, None)
    out["single_vertex_loops"] = ([I64_MIN], [I64_MIN] * 5, [I64_MIN] * 5, None, None, None)
    out["all_unmatched"] = (np.arange(100), np.arange(200, 300), np.arange(300, 400), None, None, None)
    out["all_null_ends"] = (np.arange(10), np.arange(10), np.arange(10), None, np.zeros(10), np.zeros(10))
    out["extremes"] = (np.array([I64_MIN, -1, 0, I64_MAX]), [I64_MIN, I64_MAX, -1, 0], [I64_MAX, I64_MIN, 0, 0], None,
                       None, None)
    keys = np.arange(500) * 2
    vvalid = (rng.random(500) > 0.2).astype(np.uint8)
    live = keys[vvalid == 1]
    out["null_vertex_keys"] = (keys, rng.choice(live, 3000), rng.choice(live, 3000), vvalid, None, None)
    out["balanced_well_formed"] = ([1, 1, 2], [1, 2], [2, 9], None, None, None)
    out["balanced_ill_formed"] = ([1, 1, 2, 3], [1, 3], [2, 9], None, None, None)
    out["null_end_balanced"] = ([1, 1, 2], [1, 2], [2, 0], None, None, [1, 0])
    out["duplicate_key"] = ([1, 1, 2], [1], [2], None, None, None)
    out["dangling_only"] = (np.arange(10), [1, 2], [20, 30], None, None, None)
    return out


CASES = _cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_oracle(gpu_ctx, name):
    got, ref = build_both(gpu_ctx, *CASES[name])
    if ref is not None:
        assert_same(got, ref)


@pytest.mark.parametrize("name", undirected_golden_names())
def test_device_equals_reference(gpu_ctx, name):
    g = load_undirected_golden(name)
    args = (g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    if g["constraint"] or g["ill_formed"]:
        with pytest.raises(pgq.ConstraintException):
            pgq.DeviceCSR.build_from_keys(gpu_ctx, *args, undirected=True)
        return
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, *args, undirected=True)
    v, e, ids = csr.download()
    csr.free()
    assert np.array_equal(v, g["csr_v"])
    assert rows_as_sets(v, e) == rows_as_sets(g["csr_v"], g["csr_e"])
    for p in range(len(g["vkey"])):
        for pos in range(v[p], v[p + 1]):
            k, q = ids[pos], e[pos]
            ks, kd, kp, kq = g["src"][k], g["dst"][k], g["vkey"][p], g["vkey"][q]
            assert (ks == kp and kd == kq) or (ks == kq and kd == kp)


def test_result_is_symmetric_and_ordered(gpu_ctx):
    rng = np.random.default_rng(5)
    keys = rng.choice(np.arange(-10**9, 10**9), 2000, replace=False)
    src, dst = rng.choice(keys, 30000), rng.choice(keys, 30000)
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, src, dst, undirected=True)
    v, e, ids = csr.download()
    csr.free()
    pair_id = {}
    for p in range(len(keys)):
        row = e[v[p]:v[p + 1]]
        assert np.all(np.diff(row) > 0)  # ascending, no repeats
        for pos in range(v[p], v[p + 1]):
            pair_id[(p, int(e[pos]))] = int(ids[pos])
    for (p, q), k in pair_id.items():
        assert pair_id[(q, p)] == k


def test_keys_equal_to_rowids_give_the_rowid_build(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    s, d = src.astype(np.int64), dst.astype(np.int64)
    pairs = np.unique(np.concatenate([s * n + d, d * n + s]))
    a = pgq.DeviceCSR.build_from_keys(gpu_ctx, np.arange(n), src, dst, undirected=True)
    got = a.download()
    a.free()
    b = pgq.DeviceCSR.build(gpu_ctx, n, pairs // n, pairs % n)
    want = b.download()
    b.free()
    assert_same(got[:2], want[:2])  # (the edge ids differ: pgq_csr_build numbers the rows)


def test_host_and_device_columns_agree(gpu_ctx):
    import torch
    rng = np.random.default_rng(3)
    vkey = rng.permutation(4096) * 5 - 9000
    vvalid = (rng.random(4096) > 0.1).astype(np.uint8)
    live = vkey[vvalid == 1]
    src, dst = rng.choice(live, 50000), rng.choice(live, 50000)
    svalid = dvalid = np.ones(50000, dtype=np.uint8)
    host = pgq.DeviceCSR.build_from_keys(gpu_ctx, vkey, src, dst, vvalid, svalid, dvalid, undirected=True)
    arrays = (vkey, src, dst, vvalid, svalid, dvalid)
    cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    dev = pgq.DeviceCSR.build_from_keys_device(gpu_ctx, 4096, 50000, *(c.data_ptr() for c in cols), undirected=True)
    ref = orcu.csr_build_keys_undirected(*arrays)
    assert_same(host.download(), ref)
    assert_same(dev.download(), ref)
    host.free()
    dev.free()
    for c, a in zip(cols, arrays):  # the columns are left as they were
        assert np.array_equal(c.cpu().numpy(), a)


def test_too_many_rows_before_deduplication_is_a_range_error(gpu_ctx):
    # 40000 rows share key 0: each of 27000 edges 0 -> 1 expands to 40000 rows each way, 2.16e9 > 2^31 in all
    keys = np.concatenate([np.zeros(40000, dtype=np.int64), [1]])
    with pytest.raises(pgq.InvalidInputException):
        pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, np.zeros(27000), np.ones(27000), undirected=True)


def test_consumers_on_a_key_built_undirected_rmat16(gpu_ctx):
    n, src, dst = datagen.rmat_edges(16)
    rng = np.random.default_rng(16)
    keys = rng.choice(np.arange(-(2**45), 2**45, 1000003), n, replace=False)
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[src], keys[dst], undirected=True)
    v, e, ids = orcu.csr_build_keys_undirected(keys, keys[src], keys[dst])
    assert_same(csr.download(), (v, e, ids))
    ps, pd = datagen.hashed_pairs(3000, n)
    out, valid, _ = csr.iterativelength(ps, pd)
    exp, expv, _ = orc.iterativelength(n, v, e, ps, pd)
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    paths, _ = csr.shortestpath(ps[:500], pd[:500])
    epaths, _ = orc.shortestpath(n, v, e, ids, ps[:500], pd[:500])
    assert paths == epaths
    bo, bv, _ = csr.iterativelengthbidirectional(ps[:1024], pd[:1024])
    eo, ev, _ = orb.iterativelengthbidirectional(n, v, e, ps[:1024], pd[:1024], None, None, 512)
    assert np.array_equal(bv, ev) and np.array_equal(bo[bv == 1], eo[ev == 1])
    ro, rv, _ = csr.reachability(ps[:1024], pd[:1024])
    eo, ew, _ = orr.reachability(n, v, e, ps[:1024], pd[:1024])
    assert np.array_equal(rv, ew) and np.array_equal(ro, eo)
    ids_all = np.arange(n)
    got = csr.local_clustering_coefficient(ids_all)[0]
    want = orc.local_clustering_coefficient(n, v, e, ids_all)[0]
    assert np.array_equal(got, want)
    assert np.array_equal(csr.weakly_connected_component(ids_all)[0], orc.weakly_connected_component(n, v, e, ids_all)[0])
    assert np.array_equal(csr.pagerank(ids_all)[0], orc.pagerank(n, v, e, ids_all)[0])
    csr.free()


def test_rmat20_build_equals_oracle(gpu_ctx):
    n, src, dst = datagen.rmat_edges(20)
    keys = np.random.default_rng(20).permutation(n).astype(np.int64) * 3 - n
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[src], keys[dst], undirected=True)
    assert_same(csr.download(), orcu.csr_build_keys_undirected(keys, keys[src], keys[dst]))
    csr.free()


def test_key_build_leaves_the_search_masks_alone(monkeypatch):
    """One workspace.  A search whose sources have no in-edges (their mask rows lie beyond the rows a workspace keeps
    known to be zero), then host-column key builds whose columns are all -1 bytes and small enough that no workspace
    slot grows, then the same search: its answers must not change."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        n_src, n_dst = 4000, 1000
        n = n_src + n_dst
        rng = np.random.default_rng(9)
        src = np.arange(n_src)
        dst = n_src + rng.integers(0, n_dst, n_src)
        chain = n_src + np.arange(n_dst - 1)
        src, dst = np.concatenate([src, chain]), np.concatenate([dst, chain + 1])
        csr = pgq.DeviceCSR.build(ctx, n, src, dst)
        v, e, _ = csr.download()
        ps = rng.integers(0, n_src, 2000)
        pd = rng.integers(0, n, 2000)
        first = csr.iterativelength(ps, pd)
        exp, expv, _ = orc.iterativelength(n, v, e, ps, pd)
        assert np.array_equal(first[0], exp) and np.array_equal(first[1], expv)
        m = 12000
        ones = np.ones(m, dtype=np.uint8)
        for undirected in (False, True):
            k = pgq.DeviceCSR.build_from_keys(ctx, [-1], np.full(m, -1), np.full(m, -1), None, ones, ones,
                                              undirected=undirected)
            k.free()
            again = csr.iterativelength(ps, pd)
            assert np.array_equal(again[0], exp) and np.array_equal(again[1], expv)
        csr.free()
    finally:
        ctx.close()
