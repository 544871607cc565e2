"""The oracle's restatement of the directed CSR CTE over key columns (oracle/pgq_oracle_keys) against what the reference
binary built from the same tables (tests/golden/refk_*.npz, made by tests/golden/make_golden_keys.py), plus the
cases the reference cannot show: NULL vertex keys and a dangling destination balanced by a duplicated one."""
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys as orck


def keys_golden_names():
    return sorted(os.path.basename(f)[5:-4] for f in glob.glob(os.path.join(GOLDEN, "refk_*.npz")))


def load_keys_golden(name):
    z = np.load(os.path.join(GOLDEN, f"refk_{name}.npz"))
    g = {k: z[k] for k in z.files}
    g["constraint"] = bool(int(g["constraint"]))
    return g


def rows_as_multisets(v, e):
    """the adjacency of every CSR row as a sorted list: DuckDB's join output order is not part of its contract"""
    v, e = np.asarray(v), np.asarray(e)
    return [sorted(e[v[i]:v[i + 1]].tolist()) for i in range(len(v) - 1)]


def test_every_case_is_there():
    assert len(keys_golden_names()) >= 8


@pytest.mark.parametrize("name", keys_golden_names())
def test_oracle_matches_reference(name):
    g = load_keys_golden(name)
    if g["constraint"]:
        with pytest.raises(orc.ConstraintError):
            orck.csr_build_keys(g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
        return
    v, e, ids = orck.csr_build_keys(g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    assert np.array_equal(v, g["csr_v"])
    assert rows_as_multisets(v, e) == rows_as_multisets(g["csr_v"], g["csr_e"])
    # every edge id in a row is an edge whose src key is the row's key and whose dst key is the neighbour's key
    for a in range(len(g["vkey"])):
        for pos in range(v[a], v[a + 1]):
            k = ids[pos]
            assert g["src"][k] == g["vkey"][a] and g["dst"][k] == g["vkey"][e[pos]]


def test_duplicate_sources_keep_edge_rowid_order():
    # rows 0 and 2 share key 7: edges 0 and 2 go under both, in edge rowid order, with their own rowids
    v, e, ids = orck.csr_build_keys([7, 8, 7, 9], [7, 8, 7], [8, 9, 9])
    assert v.tolist() == [0, 2, 3, 5, 5, 5]
    assert e.tolist() == [1, 3, 3, 1, 3]
    assert ids.tolist() == [0, 2, 1, 0, 2]


def test_null_vertex_key_matches_nothing():
    # row 1's key is NULL: it keeps its place (n = 3 rows), has no edges and is no edge's endpoint
    v, e, ids = orck.csr_build_keys([1, 2, 3], [1, 3], [3, 1], vertex_valid=[1, 0, 1])
    assert v.tolist() == [0, 1, 1, 2, 2]
    assert e.tolist() == [2, 0] and ids.tolist() == [0, 1]
    with pytest.raises(orc.ConstraintError):  # an edge into it is dangling
        orck.csr_build_keys([1, 2, 3], [1], [2], vertex_valid=[1, 0, 1])


def test_dangling_destination_balanced_by_duplicate_is_rejected():
    # S = 2 = C: edge 0 has md = 0, edge 1 has md = 2 -- the reference's count check passes, the per-edge one does not
    with pytest.raises(orc.ConstraintError):
        orck.csr_build_keys([1, 2, 2], [1, 1], [9, 2])
