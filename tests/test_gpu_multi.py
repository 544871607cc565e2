"""Several GPUs from one process (pgq_multi_*, SURVEY.md section 8e): CSR replicas by peer copy, the search lanes
of a call dealt over the devices, no collective.  The multi-device cases need >= 2 visible GPUs and skip
otherwise; the replica itself is also exercised on one GPU."""
import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc

pytestmark = pytest.mark.gpu


def test_csr_clone_is_a_full_replica(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    eid = np.arange(len(src), dtype=np.int64) * 2 + 1
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst, eid)
    other = pgq.Context(pgq.device_count() - 1)  # the last device (= device 0 on a one-GPU box)
    rep = csr.clone(other)
    for a, b in zip(csr.download(), rep.download()):
        assert np.array_equal(a, b)
    ps, pd = datagen.hashed_pairs(700, n)
    o1, v1, s1 = csr.iterativelength(ps, pd)
    o2, v2, s2 = rep.iterativelength(ps, pd)
    assert np.array_equal(o1, o2) and np.array_equal(v1, v2) and s1["edges_traversed"] == s2["edges_traversed"]
    p1, _ = csr.shortestpath(ps[:100], pd[:100])
    p2, _ = rep.shortestpath(ps[:100], pd[:100])
    assert p1 == p2
    rep.free()
    csr.free()
    other.close()


@pytest.mark.parametrize("ndev", [2, 4, 8])
def test_multi_device_iterativelength(gpu_ctx, ndev):
    if pgq.device_count() < ndev:
        pytest.skip(f"needs {ndev} GPUs")
    n, src, dst = datagen.rmat_edges(14)
    v, e, ids = orc.csr_build(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    multi = pgq.MultiDeviceCSR(csr, list(range(ndev)))
    ps, pd = datagen.hashed_pairs(5000, n)
    sv = (np.arange(5000) % 13 != 0).astype(np.uint8)
    exp, expv, _ = orc.iterativelength(n, v, e, ps, pd, sv, 512)
    out, valid, sts = multi.iterativelength(ps, pd, sv)
    assert np.array_equal(out, exp) and np.array_equal(valid, expv)
    _, _, one = csr.iterativelength(ps, pd, sv)
    searches = [s["searches"] for s in sts]
    assert sum(searches) == one["searches"] and max(searches) - min(searches) <= 1  # lanes dealt evenly
    out, valid, _ = multi.iterativelength(ps[:3], pd[:3])  # fewer searches than devices
    e3, v3, _ = orc.iterativelength(n, v, e, ps[:3], pd[:3], None, 512)
    assert np.array_equal(out, e3) and np.array_equal(valid, v3)
    multi.free()
    csr.free()
