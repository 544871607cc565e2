"""Long rows that cross a range boundary of the bottom-up layout and become finished, against the oracle.

k_pull_finish runs behind every fused bottom-up level.  In one launch it applies the level update to the long rows
that cross a 1024-position range boundary (marking the ones every live lane has seen as finished), and it zeroes the
frontier entries of rows newly set in the finished-rows bitmap since the snapshot of two levels ago (DESIGN §3).  The
graph here makes such crossing rows finish in a bottom-up level that more bottom-up levels follow:

  sources -> layer A (1500 vertices) -> 8 hubs, each with an in-edge from every vertex of A (in-degree 1500) -> chain
  -> layer B (1500 vertices) -> 6 more hubs of in-degree 1500 -> chain

plus sources whose only out-edge ends at a vertex without out-edges, so that their lanes die after level 1 and the
hubs are finished as soon as the other lanes have them.  Every level is forced bottom-up (PGQ_B200_SCHEDULE=b), with
the skip of finished rows on and off; lengths, validity and work counters must equal the oracle's."""
import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc

pytestmark = pytest.mark.gpu

N_SRC, N_DEAD = 600, 50
A0, NA = 1000, 1500
H0, NH = 2500, 8
C0, NC = 2600, 12
B0, NB = 3000, 1500
G0, NG = 4500, 6
D0, ND = 4600, 10
N = 4700


def _graph():
    rng = np.random.default_rng(20261016)
    src, dst = [], []

    def edges(s, d):
        src.append(np.asarray(s, dtype=np.int64).ravel())
        dst.append(np.asarray(d, dtype=np.int64).ravel())

    a = np.arange(A0, A0 + NA)
    b = np.arange(B0, B0 + NB)
    edges(np.repeat(np.arange(N_SRC), 3), rng.choice(a, 3 * N_SRC))        # sources -> A
    dead = np.arange(N_SRC, N_SRC + N_DEAD)
    edges(dead, dead + N_DEAD)                                             # lanes that die after level 1
    edges(np.repeat(a, 2), rng.choice(a, 2 * NA))                          # short rows inside A
    for h in range(H0, H0 + NH):                                           # hubs: in-degree 1500, crossing rows
        edges(rng.permutation(a), np.full(NA, h))
    edges(np.arange(H0, H0 + NH), np.full(NH, C0))
    edges(np.arange(C0, C0 + NC - 1), np.arange(C0 + 1, C0 + NC))          # chain behind the hubs
    edges(np.full(NB, C0 + 5), b)                                          # chain -> B
    for h in range(G0, G0 + NG):                                           # a second set of hubs, later levels
        edges(rng.permutation(b), np.full(NB, h))
    edges(np.arange(G0, G0 + NG), np.full(NG, D0))
    edges(np.arange(D0, D0 + ND - 1), np.arange(D0 + 1, D0 + ND))
    perm = rng.permutation(N)  # (ids shuffled: the internal renumbering must not matter)
    return np.concatenate(src), np.concatenate(dst), perm


@pytest.fixture(scope="module")
def graph(gpu_ctx):
    s, d, perm = _graph()
    s, d = perm[s], perm[d]
    eid = np.arange(len(s), dtype=np.int64)
    csr = pgq.DeviceCSR.build(gpu_ctx, N, s, d, eid)
    v, e, ids = csr.download()
    ov, oe, oids = orc.csr_build(N, s, d, eid)
    assert np.array_equal(v, ov) and np.array_equal(e, oe) and np.array_equal(ids, oids)
    indeg = np.bincount(d, minlength=N)
    assert (indeg[perm[np.arange(H0, H0 + NH)]] > 1024).all()  # every hub row spans more than one range
    yield csr, v, e, ids, perm
    csr.free()


def _pairs(perm, k, seed):
    rng = np.random.default_rng(seed)
    srcs = rng.permutation(N_SRC + N_DEAD)[:k]
    targets = np.concatenate([np.arange(H0, H0 + NH), np.arange(C0, C0 + NC), np.arange(G0, G0 + NG),
                              np.arange(D0, D0 + ND), rng.integers(0, N, 40)])
    dsts = rng.choice(targets, k)
    return perm[srcs], perm[dsts]


@pytest.mark.parametrize("skip", ["1", "0"])
@pytest.mark.parametrize("lanes", [64, 128, 256, 512])
@pytest.mark.parametrize("schedule", ["b", "bbbbbp", "pbbb"])
def test_crossing_rows_finish_under_bottom_up_levels(graph, monkeypatch, schedule, lanes, skip):
    csr, v, e, _, perm = graph
    monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
    monkeypatch.setenv("PGQ_B200_PULL_SKIP", skip)
    for k, rb in ((lanes, False), (650, True), (lanes // 2 + 1, True)):
        ps, pd = _pairs(perm, k, seed=lanes + k + len(schedule))
        out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes, reference_batching=rb))
        if rb:
            exp, expv, ost = orc.iterativelength(N, v, e, ps, pd, None, lanes)
        else:
            exp, expv, ost, _ = orc.iterativelength_ex(N, v, e, ps, pd, None, lanes, prune=True, dedup=True)
        assert np.array_equal(valid, expv) and np.array_equal(out, exp)
        assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
            ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices)
        assert st["pull_levels"] >= 6  # the hubs are finished early, bottom-up levels follow
        assert int(valid.sum()) > 0


@pytest.mark.parametrize("lanes", [64, 512])
def test_crossing_rows_finish_paths(graph, monkeypatch, lanes):
    """The path mode finishes crossing rows with a warp per row."""
    csr, v, e, ids, perm = graph
    monkeypatch.setenv("PGQ_B200_SCHEDULE", "b")
    ps, pd = _pairs(perm, 97, seed=lanes)
    got, _ = csr.shortestpath(ps, pd, None, pgq.Options(lanes))
    exp, _ = orc.shortestpath(N, v, e, ids, ps, pd, None, 512)
    assert got == exp
