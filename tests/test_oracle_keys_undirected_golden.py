"""The oracle's restatement of the undirected CSR CTE over key columns (oracle/pgq_oracle_keys_undirected) against what
the reference binary built from the same tables (tests/golden/refu_*.npz, made by
tests/golden/make_golden_keys_undirected.py) and against an independent numpy restatement on random inputs."""
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys_undirected as orcu


def undirected_golden_names():
    return sorted(os.path.basename(f)[5:-4] for f in glob.glob(os.path.join(GOLDEN, "refu_*.npz")))


def load_undirected_golden(name):
    z = np.load(os.path.join(GOLDEN, f"refu_{name}.npz"))
    g = {k: z[k] for k in z.files}
    g["constraint"] = bool(int(g["constraint"]))
    g["ill_formed"] = bool(int(g["ill_formed"]))
    return g


def rows_as_sets(v, e):
    """the adjacency of every CSR row as a sorted list: DuckDB's GROUP BY output order is not part of its contract"""
    v, e = np.asarray(v), np.asarray(e)
    return [sorted(e[v[i]:v[i + 1]].tolist()) for i in range(len(v) - 2)]


def sql_neighbours(vkey, src, dst, sv=None, dv=None):
    """row p -> the sorted distinct rows q of edges_cte UNION ALL its reverse, from numpy alone"""
    vkey, src, dst = (np.asarray(a, dtype=np.int64) for a in (vkey, src, dst))
    m = src.shape[0]
    sv = np.ones(m, bool) if sv is None else np.asarray(sv, bool)
    dv = np.ones(m, bool) if dv is None else np.asarray(dv, bool)
    a, c = [], []
    for k in np.nonzero(sv & dv)[0]:
        for x in np.nonzero(vkey == src[k])[0]:
            for y in np.nonzero(vkey == dst[k])[0]:
                a += [x, y]
                c += [y, x]
    pairs = np.unique(np.stack([np.asarray(a, dtype=np.int64), np.asarray(c, dtype=np.int64)]), axis=1) \
        if a else np.zeros((2, 0), dtype=np.int64)
    return [sorted(pairs[1][pairs[0] == p].tolist()) for p in range(vkey.shape[0])]


def numpy_restatement(vkey, src, dst, vv=None, sv=None, dv=None):
    """(v, e, ids) or None for the ConstraintException, with np.unique over the stacked pairs and the two defined
    choices; the degrees count distinct (row, other end) pairs, a NULL other end as one more value"""
    vkey, src, dst = (np.asarray(a, dtype=np.int64) for a in (vkey, src, dst))
    n, m = vkey.shape[0], src.shape[0]
    vv = np.ones(n, bool) if vv is None else np.asarray(vv, bool)
    sv = np.ones(m, bool) if sv is None else np.asarray(sv, bool)
    dv = np.ones(m, bool) if dv is None else np.asarray(dv, bool)
    rows = {x: np.nonzero(vv & (vkey == x))[0] for x in set(src.tolist()) | set(dst.tolist())}
    trip = [(p, q, k) for k in range(m) if sv[k] and dv[k]
            for a in rows[src[k]] for c in rows[dst[k]] for p, q in ((a, c), (c, a))]
    t = np.array(trip, dtype=np.int64).reshape(-1, 3)
    t = t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]
    _, first = np.unique(t[:, :2], axis=0, return_index=True)
    u = t[np.sort(first)]
    ends = set()
    for k in range(m):
        for jv, jk, ov, ok in ((sv[k], src[k], dv[k], dst[k]), (dv[k], dst[k], sv[k], src[k])):
            if jv:
                for a in rows[jk]:
                    ends.add((int(a), bool(ov), int(ok) if ov else 0))
    cnt = np.bincount(np.array([e[0] for e in ends], dtype=np.int64), minlength=n)[:n]
    deg = np.bincount(u[:, 0], minlength=n)[:n]
    if not np.array_equal(cnt, deg):
        return None
    v = np.zeros(n + 2, dtype=np.int64)
    v[1:n + 1] = np.cumsum(deg)
    v[n + 1] = v[n]
    return v, u[:, 1].copy(), u[:, 2].copy()


def test_every_case_is_there():
    assert len(undirected_golden_names()) >= 10


@pytest.mark.parametrize("name", undirected_golden_names())
def test_oracle_matches_reference(name):
    g = load_undirected_golden(name)
    args = (g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    if g["constraint"] or g["ill_formed"]:
        with pytest.raises(orc.ConstraintError):
            orcu.csr_build_keys_undirected(*args)
        return
    v, e, ids = orcu.csr_build_keys_undirected(*args)
    assert np.array_equal(v, g["csr_v"])
    assert rows_as_sets(v, e) == rows_as_sets(g["csr_v"], g["csr_e"])
    # every edge id joins its pair in one direction or the other
    for p in range(len(g["vkey"])):
        for pos in range(v[p], v[p + 1]):
            k, q = ids[pos], e[pos]
            ks, kd, kp, kq = g["src"][k], g["dst"][k], g["vkey"][p], g["vkey"][q]
            assert (ks == kp and kd == kq) or (ks == kq and kd == kp)


def test_the_reference_scatters_the_ill_formed_balanced_case_out_of_place():
    # rows 0, 1 hold key 1, row 2 key 2, row 3 key 3; edges (1,2), (3,9): S = R = 4 but R(row 2) = 2 != 1
    # the reference accepts it: its row 2 gets two entries, the second in row 3's place, so row 3's offsets run
    # backwards and no row set of the reference's CSR is row 3's (empty) SQL neighbour set
    g = load_undirected_golden("balanced_ill_formed")
    assert not g["constraint"] and g["ill_formed"]
    v, e = g["csr_v"], g["csr_e"]
    want = sql_neighbours(g["vkey"], g["src"], g["dst"])
    assert [p for p in range(len(want)) if v[p + 1] < v[p] or sorted(e[v[p]:v[p + 1]].tolist()) != want[p]]
    with pytest.raises(orc.ConstraintError):
        orcu.csr_build_keys_undirected(g["vkey"], g["src"], g["dst"])


def test_the_balanced_well_formed_case_is_built():
    # rows 0, 1 hold key 1, row 2 key 2; edges (1,2), (2,9): cnt = R(p) for every row
    v, e, ids = orcu.csr_build_keys_undirected([1, 1, 2], [1, 2], [2, 9])
    assert v.tolist() == [0, 1, 2, 4, 4] and e.tolist() == [2, 2, 0, 1] and ids.tolist() == [0, 0, 0, 0]


def test_defined_choices():
    # parallel and reciprocal edges collapse onto the smallest edge rowid; a self-loop stays once
    v, e, ids = orcu.csr_build_keys_undirected([5, 6, 7], [5, 5, 6, 7, 6], [6, 6, 5, 7, 7])
    assert v.tolist() == [0, 1, 3, 5, 5]
    assert e.tolist() == [1, 0, 2, 1, 2] and ids.tolist() == [0, 0, 4, 4, 3]


def test_random_inputs_against_numpy():
    rng = np.random.default_rng(44)
    accepted = refused = 0
    for _ in range(300):
        n, m = int(rng.integers(0, 14)), int(rng.integers(0, 30))
        pool = np.arange(-4, 12)
        vkey = rng.choice(pool, n) if rng.random() < 0.5 else rng.permutation(pool)[:n]
        src, dst = rng.choice(pool, m), rng.choice(pool, m)
        vv = (rng.random(n) > 0.1).astype(np.uint8)
        sv, dv = ((rng.random(m) > 0.1).astype(np.uint8) for _ in range(2))
        want = numpy_restatement(vkey, src, dst, vv, sv, dv)
        if want is None:
            refused += 1
            with pytest.raises(orc.ConstraintError):
                orcu.csr_build_keys_undirected(vkey, src, dst, vv, sv, dv)
            continue
        accepted += 1
        got = orcu.csr_build_keys_undirected(vkey, src, dst, vv, sv, dv)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
    assert accepted > 20 and refused > 20
