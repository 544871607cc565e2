"""pgq_csr_build_keys / pgq_csr_build_keys_device: the directed CSR CTE over key columns on the device, against the
oracle's restatement (oracle/pgq_oracle_keys), the reference's own output (tests/golden/refk_*.npz) and pgq_csr_build."""
import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys as orck
from test_oracle_keys_golden import keys_golden_names, load_keys_golden, rows_as_multisets

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def build_both(ctx, vkey, src, dst, vvalid=None, svalid=None, dvalid=None):
    """(device arrays, oracle arrays); both sides raise their ConstraintException alike"""
    try:
        ref = orck.csr_build_keys(vkey, src, dst, vvalid, svalid, dvalid)
    except orc.ConstraintError:
        ref = None
    if ref is None:
        with pytest.raises(pgq.ConstraintException) as ex:
            pgq.DeviceCSR.build_from_keys(ctx, vkey, src, dst, vvalid, svalid, dvalid)
        assert str(ex.value) == orc.CONSTRAINT_TEXT
        return None, None
    csr = pgq.DeviceCSR.build_from_keys(ctx, vkey, src, dst, vvalid, svalid, dvalid)
    got = csr.download()
    csr.free()
    return got, ref


def assert_same(got, ref):
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)


def _cases():
    rng = np.random.default_rng(7)
    out = {}
    keys = rng.permutation(3000)
    out["shuffled"] = (keys, rng.choice(keys, 20000), rng.choice(keys, 20000), None, None, None)
    keys = rng.choice(np.arange(-10**15, 10**15, 1000003), 2000, replace=False)
    out["sparse_signed"] = (keys, rng.choice(keys, 9000), rng.choice(keys, 9000), None, None, None)
    keys = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], dtype=np.int64)
    out["extremes"] = (keys, rng.choice(keys, 300), rng.choice(keys, 300), None, None, None)
    keys = np.concatenate([rng.integers(0, 50, 400), 1000 + np.arange(100)])  # sources repeat up to ~20 times
    out["dup_sources"] = (keys, rng.choice(keys[:400], 3000), 1000 + rng.integers(0, 100, 3000), None, None, None)
    keys = np.arange(500) * 2
    vvalid = (rng.random(500) > 0.2).astype(np.uint8)
    live = keys[vvalid == 1]
    out["null_vertex_keys"] = (keys, rng.choice(live, 4000), rng.choice(live, 4000), vvalid, None, None)
    m = 4000
    src, dst = rng.choice(keys, m), rng.choice(keys, m)
    svalid = (rng.random(m) > 0.3).astype(np.uint8)
    out["null_src_keys"] = (keys, src, np.where(svalid == 1, dst, 12345), None, svalid, None)
    dvalid = (rng.random(m) > 0.3).astype(np.uint8)
    out["null_dst_keys_behind_unmatched_src"] = (keys, np.where(dvalid == 1, src, -7), dst, None, None, dvalid)
    out["empty_edges"] = (keys, [], [], None, None, None)
    out["single_vertex"] = ([I64_MIN], [I64_MIN] * 5, [I64_MIN] * 5, None, None, None)
    out["single_vertex_no_edges"] = ([3], [], [], None, None, None)
    out["empty_vertex_table"] = ([], [1, 2], [2, 1], None, None, None)
    out["no_key_matches"] = (np.arange(100), np.arange(200, 300), np.arange(0, 100), None, None, None)
    # what must be refused
    out["dangling_dst"] = (np.arange(10), [1, 2, 3], [2, 3, 10], None, None, None)
    out["duplicate_dst"] = (np.array([0, 1, 2, 2]), [0, 1], [1, 2], None, None, None)
    out["dangling_balanced_by_duplicate"] = (np.array([0, 1, 2, 2]), [0, 1], [7, 2], None, None, None)
    out["null_dst_behind_matched_src"] = (np.arange(10), [1, 2], [2, 3], None, None, [1, 0])
    out["dst_is_null_vertex_key"] = (np.arange(10), [1, 2], [2, 3], np.array([1, 1, 1, 0, 1, 1, 1, 1, 1, 1]), None, None)
    return out


CASES = _cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_oracle(gpu_ctx, name):
    got, ref = build_both(gpu_ctx, *CASES[name])
    if ref is not None:
        assert_same(got, ref)


@pytest.mark.parametrize("name", keys_golden_names())
def test_device_equals_reference(gpu_ctx, name):
    g = load_keys_golden(name)
    if g["constraint"]:
        with pytest.raises(pgq.ConstraintException):
            pgq.DeviceCSR.build_from_keys(gpu_ctx, g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
        return
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    v, e, _ = csr.download()
    csr.free()
    assert np.array_equal(v, g["csr_v"])
    assert rows_as_multisets(v, e) == rows_as_multisets(g["csr_v"], g["csr_e"])


def test_keys_equal_to_rowids_give_the_rowid_build(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    a = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    b = pgq.DeviceCSR.build_from_keys(gpu_ctx, np.arange(n), src, dst)
    for x, y in zip(a.download(), b.download()):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
    a.free()
    b.free()


def test_too_many_join_rows_is_a_range_error(gpu_ctx):
    # 50000 vertex rows share key 0: 44000 edges 0 -> 1 expand to 2.2e9 rows, beyond the int32 CSR
    keys = np.concatenate([np.zeros(50000, dtype=np.int64), [1]])
    with pytest.raises(pgq.InvalidInputException):
        pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, np.zeros(44000), np.ones(44000))


def test_host_and_device_columns_agree(gpu_ctx):
    import torch
    rng = np.random.default_rng(3)
    vkey = rng.permutation(4096) * 5 - 9000
    vvalid = (rng.random(4096) > 0.1).astype(np.uint8)
    live = vkey[vvalid == 1]
    src, dst = rng.choice(vkey, 50000), rng.choice(live, 50000)
    svalid = ((rng.random(50000) > 0.1) & np.isin(src, live)).astype(np.uint8)
    dvalid = np.ones(50000, dtype=np.uint8)
    host = pgq.DeviceCSR.build_from_keys(gpu_ctx, vkey, src, dst, vvalid, svalid, dvalid)
    cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (vkey, src, dst, vvalid, svalid, dvalid)]
    dev = pgq.DeviceCSR.build_from_keys_device(gpu_ctx, 4096, 50000, *(c.data_ptr() for c in cols))
    ref = orck.csr_build_keys(vkey, src, dst, vvalid, svalid, dvalid)
    assert_same(host.download(), ref)
    assert_same(dev.download(), ref)
    host.free()
    dev.free()
    # the columns are left as they were; without validity columns every key is valid
    assert np.array_equal(cols[0].cpu().numpy(), vkey)
    keys = rng.permutation(1000)
    cols = [torch.from_numpy(a).cuda() for a in (keys, keys[rng.integers(0, 1000, 8000)], keys[rng.integers(0, 1000, 8000)])]
    dev = pgq.DeviceCSR.build_from_keys_device(gpu_ctx, 1000, 8000, *(c.data_ptr() for c in cols))
    assert_same(dev.download(), orck.csr_build_keys(*(c.cpu().numpy() for c in cols)))
    dev.free()


def test_paths_on_a_key_built_rmat16(gpu_ctx):
    n, src, dst = datagen.rmat_edges(16)
    rng = np.random.default_rng(16)
    keys = rng.choice(np.arange(-(2**45), 2**45, 1000003), n, replace=False)
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[src], keys[dst])
    v, e, ids = orck.csr_build_keys(keys, keys[src], keys[dst])
    assert_same(csr.download(), (v, e, ids))
    ps, pd = datagen.hashed_pairs(3000, n)
    out, valid, _ = csr.iterativelength(ps, pd)
    exp, expv, _ = orc.iterativelength(n, v, e, ps, pd)
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    paths, _ = csr.shortestpath(ps[:500], pd[:500])
    epaths, _ = orc.shortestpath(n, v, e, ids, ps[:500], pd[:500])
    assert paths == epaths
    csr.free()


def test_rmat20_build_equals_oracle(gpu_ctx):
    n, src, dst = datagen.rmat_edges(20)
    keys = np.random.default_rng(20).permutation(n).astype(np.int64) * 3 - n
    csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[src], keys[dst])
    assert_same(csr.download(), orck.csr_build_keys(keys, keys[src], keys[dst]))
    csr.free()
