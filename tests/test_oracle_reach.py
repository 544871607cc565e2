"""The oracle's restatement of reachability (oracle/pgq_oracle_reach.c) on the CPU: the properties its contract states,
checked against scipy, and the two places where the reference's loop leaves defined ground (the NULL restart and the
visit_list that is kept across batches)."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import shortest_path

from duckpgq_extension_b200 import datagen
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_reach as orr


def _hops(n, s, d, sources):
    """BFS hop counts from every source (inf = unreachable), scipy"""
    g = sp.csr_matrix((np.ones(len(s)), (s, d)), shape=(n, n))
    return shortest_path(g, unweighted=True, directed=True, indices=sources)


def _graph(kind, seed):
    if kind == "rmat":
        return datagen.rmat_edges(9, seed=seed)
    rng = np.random.default_rng(seed)
    n = 300
    m = {"sparse": 330, "dense": 3000}[kind]
    return n, rng.integers(0, n, m), rng.integers(0, n, m)


def _expected(n, s, d, src, dst):
    uniq, inv = np.unique(src, return_inverse=True)
    hops = _hops(n, s, d, uniq)
    return np.isfinite(hops[inv, dst]).astype(np.uint8), uniq, hops


@pytest.mark.parametrize("kind,seed", [("rmat", 1), ("rmat", 2), ("sparse", 3), ("dense", 4), ("sparse", 5)])
@pytest.mark.parametrize("restart", [False, True])
def test_plain_traversal_is_reachability(kind, seed, restart):
    n, s, d = _graph(kind, seed)
    v, e, _ = orc.csr_build(n, s, d)
    rng = np.random.default_rng(seed)
    p = 1500
    src, dst = rng.integers(0, n, p), rng.integers(0, n, p)
    dst[::9] = src[::9]
    out, written, st = orr.reachability(n, v, e, src, dst, restart=restart)
    exp, _, _ = _expected(n, s, d, src, dst)
    assert written.all() and np.array_equal(out, exp)
    # batches: the first appearances of 512 distinct sources cut the rows
    assert st.batches == len(orr.reference_batch_starts(src))


def test_counters_of_one_batch():
    """One batch: a level per BFS distance reached by any lane, plus the one that adds nothing; each level expands the
    vertices that some lane reached at the previous distance."""
    n, s, d = datagen.rmat_edges(10, seed=7)
    v, e, _ = orc.csr_build(n, s, d)
    rng = np.random.default_rng(7)
    src, dst = rng.integers(0, n, 400), rng.integers(0, n, 400)
    out, _, st = orr.reachability(n, v, e, src, dst)
    exp, uniq, hops = _expected(n, s, d, src, dst)
    assert np.array_equal(out, exp) and st.batches == 1
    finite = np.where(np.isfinite(hops), hops, -1).astype(np.int64)
    ecc = int(finite.max())
    deg = np.diff(v[: n + 1])
    w = sum(int(deg[np.nonzero((finite == k).any(axis=0))[0]].sum()) for k in range(ecc + 1))
    assert (st.levels, st.edges_traversed) == (ecc + 1, w)


@pytest.mark.parametrize("kind,seed", [("rmat", 11), ("sparse", 12), ("dense", 13), ("rmat", 14)])
def test_variant_answers_on_single_batch_calls(kind, seed):
    n, s, d = _graph(kind, seed)
    v, e, _ = orc.csr_build(n, s, d)
    rng = np.random.default_rng(seed)
    src, dst = rng.integers(0, n, 2048), rng.integers(0, n, 2048)
    src = src % 200  # at most 200 distinct sources: one batch
    dst[::5] = src[::5]
    a, _, sa = orr.reachability(n, v, e, src, dst)
    b, _, sb = orr.reachability(n, v, e, src, dst, is_variant=True)
    assert np.array_equal(a, b) and sa.batches == sb.batches == 1 and sb.stale_starts == 0


def test_variant_mode_two_is_reached_and_still_answers():
    """A frontier of more than input_size / 2 vertices switches the variant to its full-scan mode (FindMode mode 2)."""
    n = 40
    s = np.concatenate([[0], np.full(30, 1), np.arange(2, 32)])
    d = np.concatenate([[1], np.arange(2, 32), np.arange(3, 33)])
    v, e, _ = orc.csr_build(n, s, d)
    src, dst = np.array([0, 0, 0, 5]), np.array([1, 32, 39, 33])
    a, _, sa = orr.reachability(n, v, e, src, dst)
    b, _, sb = orr.reachability(n, v, e, src, dst, is_variant=True)
    assert list(a) == [1, 1, 0, 0] and np.array_equal(a, b)
    assert sb.levels == sa.levels and sb.edges_traversed >= sa.edges_traversed


def _stale_case():
    # 0 -> 1 -> {2 .. 9}: the second level finds 8 > input_size / 2 = 5 vertices, so the third runs in mode 2, finds
    # nothing, and the batch ends with visit_list = {2 .. 9}
    n = 10
    v, e, _ = orc.csr_build(n, np.array([0] + [1] * 8), np.arange(1, 10))
    src, dst = np.array([7, 0, 0]), np.array([7, 1, 5])
    sv = np.array([0, 1, 1], np.uint8)
    return n, v, e, src, dst, sv


def test_stale_visit_list_is_reproduced():
    """The NULL first row makes the reference start a second batch at row 2 (result_size += 2 valid rows).  With
    is_variant that batch starts in mode 1 over the visit_list the first batch left behind, which holds none of its
    sources: it expands nothing and overwrites row 2's true with false."""
    n, v, e, src, dst, sv = _stale_case()
    plain, written, sp_ = orr.reachability(n, v, e, src, dst, sv, restart=True)
    assert list(written) == [0, 1, 1] and list(plain[1:]) == [1, 1] and sp_.batches == 2
    var, _, st = orr.reachability(n, v, e, src, dst, sv, restart=True, is_variant=True)
    assert list(var[1:]) == [1, 0] and st.batches == 2 and st.stale_starts == 1
    # without the restart there is one batch, and the variant answers as the plain traversal
    var1, _, st1 = orr.reachability(n, v, e, src, dst, sv, is_variant=True)
    assert list(var1[1:]) == [1, 1] and st1.batches == 1 and st1.stale_starts == 0


def test_restart_and_hang():
    n, s, d = datagen.rmat_edges(8, seed=3)
    v, e, _ = orc.csr_build(n, s, d)
    src, dst = np.arange(20) % n, (np.arange(20) * 7) % n
    sv = np.ones(20, np.uint8)
    sv[[2, 5]] = 0
    # two NULLs: the second batch starts at row 18 and re-runs rows 18, 19
    assert orr.reference_batch_starts(src, sv) == [0, 18]
    a, wa, sa = orr.reachability(n, v, e, src, dst, sv, restart=True)
    b, wb, sb = orr.reachability(n, v, e, src, dst, sv)
    assert np.array_equal(a, b) and np.array_equal(wa, wb) and (sa.batches, sb.batches) == (2, 1)
    # a NULL last row: the batch that starts there finds no valid source and never ends
    sv[19] = 0
    with pytest.raises(orr.ReferenceHang):
        orr.reference_batch_starts(src, sv)
    with pytest.raises(orr.ReferenceHang):
        orr.reachability(n, v, e, src, dst, sv, restart=True)
    _, written, st = orr.reachability(n, v, e, src, dst, sv)
    assert st.batches == 1 and list(np.nonzero(written == 0)[0]) == [2, 5, 19]


def test_defined_batches():
    """513 distinct sources: the row that opens lane 512 ends the batch; a repeat of a first-batch source after it opens
    a lane in the second; NULL sources neither take lanes nor move the start; NULL destinations keep their lane."""
    n, s, d = datagen.rmat_edges(10, seed=5)
    v, e, _ = orc.csr_build(n, s, d)
    src = np.concatenate([np.arange(512), [0, 600]])
    dst = np.concatenate([np.arange(512)[::-1], [3, 600]])
    out, written, st = orr.reachability(n, v, e, src, dst)
    exp, _, _ = _expected(n, s, d, src, dst)
    assert np.array_equal(out, exp) and st.batches == 2
    sv = np.ones(len(src), np.uint8)
    sv[10] = 0
    dv = np.ones(len(src), np.uint8)
    dv[20] = 0
    out2, written2, st2 = orr.reachability(n, v, e, src, dst, sv, dv)
    # (without source 10 the first batch has room for rows 512 and 513)
    assert st2.batches == 1 and written2[10] == 0 and written2[20] == 0
    ok = written2 == 1
    assert np.array_equal(out2[ok], exp[ok])
    with pytest.raises(ValueError):
        orr.reachability(n, v, e, np.array([n]), np.array([0]))
