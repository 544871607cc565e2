"""shortest_k_groups: every path of the k shortest lengths of a row, SQL/PGQ's SHORTEST k GROUP (include/duckpgq_b200.h,
pgq_shortest_k_groups / pgq_shortest_k_groups_count).

The CPU tests pin the oracle (oracle/pgq_oracle_kgroups.c) against a brute-force enumeration on random multigraphs with
self-loops and parallel edges: walk counts (A^h)[s, t] in Python integers and the walks themselves, each mode's paths,
grouped by length.  They check the identities with shortest_k_paths[_mode] at k = N, with all_shortest_paths and
shortest_path_count at k = 1, and show that each case of the catalogue reaches what it is named after.  The GPU tests
require the device's lists, counts, groups, completeness and batch counters to equal the oracle's.
"""
import threading

import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_INVALID_ARG, PGQ_ERR_NOT_INITIALIZED, PGQ_ERR_RANGE, PGQ_ERR_UNSUPPORTED
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_kgroups as okg
from oracle import pgq_oracle_kpaths_modes as okm
from oracle import pgq_oracle_kshortest as oks

MODES = ("WALK", "TRAIL", "ACYCLIC", "SIMPLE")
PATH_MAX = 65533
INT64_MAX = 2 ** 63 - 1
WALK_COUNTERS = ("batches", "lanes", "searches", "levels", "push_levels")
MODE_COUNTERS = ("batches", "lanes", "searches", "levels")
# the reference's top_k.test / path_modes.test graph, edges in rowid order
TOPK = {"n": 5, "src": [0, 0, 0, 3, 1, 1, 2, 4], "dst": [1, 2, 3, 0, 2, 3, 3, 3]}


def ref_csr(n, src, dst, eid=None):
    return orc.csr_build(n, np.asarray(src, np.int64), np.asarray(dst, np.int64), eid)


def random_multigraph(seed, n_hi=7, m_hi=12):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, n_hi))
    m = int(rng.integers(0, m_hi))
    src, dst = rng.integers(0, n, m), rng.integers(0, n, m)
    if m > 2:  # a parallel edge and a self-loop
        src[1], dst[1] = src[0], dst[0]
        dst[2] = src[2]
    return n, src.astype(np.int64), dst.astype(np.int64)


def all_rows(n):
    ps, pd = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    return ps.ravel().astype(np.int64), pd.ravel().astype(np.int64)


# ---- brute force -----------------------------------------------------------------------------------------------------
def walk_counts(n, v, e, s, t, hmax):
    """(A^h)[s, t] for h = 0 .. hmax in Python integers"""
    row = [0] * n
    row[s] = 1
    out = [row[t]]
    for _ in range(hmax):
        nxt = [0] * n
        for u in range(n):
            if row[u]:
                for idx in range(v[u], v[u + 1]):
                    nxt[int(e[idx])] += row[u]
        row = nxt
        out.append(row[t])
    return out


def group_lengths(counts, k):
    return [h for h, c in enumerate(counts) if c > 0][:k]


def brute_walks(n, v, e, ids, s, t, lengths):
    """every walk s -> t whose length is in `lengths`, sorted by (h, steps from t back to s), a step being (parent,
    the edge's position in the parent's adjacency)"""
    hmax = max(lengths, default=0)
    back = [[0] * n for _ in range(hmax + 1)]  # back[j][u]: walks u -> t of j edges
    back[0][t] = 1
    for j in range(1, hmax + 1):
        for u in range(n):
            back[j][u] = sum(back[j - 1][int(e[idx])] for idx in range(v[u], v[u + 1]))
    out = []

    def go(u, left, elems, steps):
        if left == 0:
            out.append(((len(steps), list(reversed(steps))), list(elems)))
            return
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            if back[left - 1][w]:
                go(w, left - 1, elems + [int(ids[idx]), w], steps + [(u, idx - int(v[u]))])

    for h in sorted(lengths):
        if back[h][s]:
            go(s, h, [s], [])
    return [el for _, el in sorted(out, key=lambda x: x[0])]


def brute_mode_paths(n, v, e, ids, s, t, mode):
    """every path s -> t of the mode (TRAIL, ACYCLIC, SIMPLE), sorted like brute_walks"""
    out = []

    def walk(u, elems, steps, used, visited):
        if u == t:
            out.append(((len(steps), list(reversed(steps))), list(elems)))
            if mode != "TRAIL" and (len(steps) > 0 or mode == "ACYCLIC" or s != t):
                return
        for idx in range(v[u], v[u + 1]):
            w = int(e[idx])
            if mode == "TRAIL":
                if idx in used:
                    continue
            elif w in visited and not (mode == "SIMPLE" and w == s == t):
                continue
            walk(w, elems + [int(ids[idx]), w], steps + [(u, idx - int(v[u]))], used | {idx}, visited | {w})

    walk(s, [s], [], frozenset(), frozenset([s]))
    return [el for _, el in sorted(out, key=lambda x: x[0])]


def h_of(path):
    return (len(path) - 1) // 2


def expected_mode_row(paths, k, max_paths):
    """(listed, count, ngroups, last_len, complete) from a row's sorted mode paths"""
    lengths = sorted({h_of(p) for p in paths})[:k]
    full = [p for p in paths if h_of(p) in lengths]
    listed = full[:max_paths] if max_paths else full
    complete = len(listed) == len(full)
    return (listed, len(full) if complete else -1, len({h_of(p) for p in listed}),
            h_of(listed[-1]) if listed else -1, complete)


# ---- the oracle against brute force ----------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(30))
def test_oracle_is_the_brute_force_enumeration(seed):
    n, src, dst = random_multigraph(seed)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = all_rows(n)
    for mode in MODES:
        if mode == "WALK":
            counts = [walk_counts(n, v, e, int(s), int(t), 8 * n) for s, t in zip(ps, pd)]
        else:
            brute = [brute_mode_paths(n, v, e, ids, int(s), int(t), mode) for s, t in zip(ps, pd)]
        for k in range(1, 7):
            for max_paths in (0, 1, 3):
                paths, rows, _ = okg.shortest_k_groups(n, v, e, ids, ps, pd, k, max_paths, mode)
                for i in range(len(ps)):
                    where = (mode, k, max_paths, int(ps[i]), int(pd[i]))
                    got = paths[i] or []
                    if mode == "WALK":
                        lengths = group_lengths(counts[i], k)
                        N = sum(counts[i][h] for h in lengths)
                        assert rows["count"][i] == min(N, INT64_MAX), where
                        assert rows["ngroups"][i] == len(lengths), where
                        assert rows["last_len"][i] == (lengths[-1] if lengths else -1), where
                        nl = min(N, max_paths) if max_paths else N
                        assert rows["npaths"][i] == nl and len(got) == nl, where
                        assert rows["complete"][i] == (nl == N), where
                        if N <= 400:
                            assert got == brute_walks(n, v, e, ids, int(ps[i]), int(pd[i]), lengths)[:nl], where
                    else:
                        listed, cnt, ng, last, complete = expected_mode_row(brute[i], k, max_paths)
                        assert got == listed, where
                        assert (rows["count"][i], rows["ngroups"][i], rows["last_len"][i], rows["complete"][i]) == \
                            (cnt, ng, last, complete), where
                    assert rows["valid"][i] == (len(got) > 0), where


@pytest.mark.parametrize("seed", range(15))
def test_identities(seed):
    n, src, dst = random_multigraph(500 + seed)
    v, e, ids = ref_csr(n, src, dst)
    ps, pd = all_rows(n)
    sp_count = oas.shortest_path_count(n, v, e, ids, ps, pd)[0]
    for mode in MODES:
        for k in (1, 2, 4):
            paths, rows, _ = okg.shortest_k_groups(n, v, e, ids, ps, pd, k, 0, mode)
            for i in range(len(ps)):
                N = int(rows["count"][i])
                if N == 0:
                    assert paths[i] is None
                    continue
                if mode == "WALK":  # the first N walks of shortest_k_paths
                    ks = oks.shortest_k_paths(n, v, e, ids, ps[i:i + 1], pd[i:i + 1], N)[0][0]
                else:
                    ks = okm.shortest_k_paths_mode(n, v, e, ids, ps[i:i + 1], pd[i:i + 1], N, mode)[0][0]
                assert paths[i] == ks, (mode, k, i)
            if k == 1:  # ALL SHORTEST for s != t
                for max_paths in (0, 2):
                    ap = oas.all_shortest_paths(n, v, e, ids, ps, pd, max_paths)[0]
                    one, _, _ = okg.shortest_k_groups(n, v, e, ids, ps, pd, 1, max_paths, mode)
                    assert all(one[i] == ap[i] for i in range(len(ps)) if ps[i] != pd[i])
                if mode == "WALK":
                    assert all(rows["count"][i] == sp_count[i] for i in range(len(ps)) if ps[i] != pd[i])
        # count-only is the full call's counts
        _, full, _ = okg.shortest_k_groups(n, v, e, ids, ps, pd, 3, 0, "WALK")
        _, cnt, _ = okg.shortest_k_groups(n, v, e, ids, ps, pd, 3, 0, "WALK", count_only=True)
        for key in ("count", "ngroups", "last_len", "valid"):
            assert np.array_equal(cnt[key], full[key])


# ---- the catalogue ---------------------------------------------------------------------------------------------------
def case_bipartite():  # an undirected 4-cycle: every walk 0 -> 2 has even length
    src = [0, 1, 1, 2, 2, 3, 3, 0]
    dst = [1, 0, 2, 1, 3, 2, 0, 3]
    return {"n": 4, "src": src, "dst": dst, "ps": [0, 0, 1], "pd": [2, 0, 2], "ks": [3], "mps": [0, 4]}


def case_dag():  # lengths 1, 2 and 3 only
    return {"n": 4, "src": [0, 0, 0, 1, 1, 2], "dst": [1, 2, 3, 2, 3, 3], "ps": [0, 1], "pd": [3, 3], "ks": [6],
            "mps": [0, 2]}


def case_self_loop_trap():  # s reaches the self-loop at 2, which does not reach t = 1
    return {"n": 3, "src": [0, 0, 2], "dst": [1, 2, 2], "ps": [0], "pd": [1], "ks": [3], "mps": [0]}


def case_cycle_behind_chain():  # a 2-cycle at 0 behind the chain 0 -> 1 -> ... -> 12
    src = list(range(12)) + [0, 13]
    dst = list(range(1, 13)) + [13, 0]
    return {"n": 14, "src": src, "dst": dst, "ps": [0, 13], "pd": [12, 12], "ks": [3], "mps": [0, 2]}


def case_diamonds(count=64):  # `count` diamonds in a row: 2^count shortest walks, and a way back for longer ones
    src, dst = [], []
    for d in range(count):
        a = 3 * d
        src += [a, a, a + 1, a + 2]
        dst += [a + 1, a + 2, a + 3, a + 3]
    end = 3 * count
    src.append(end)
    dst.append(0)
    return {"n": end + 1, "src": src, "dst": dst, "ps": [0], "pd": [end], "ks": [2], "mps": [5]}


def case_closed():  # s == t on the top_k graph, every mode
    return {"n": TOPK["n"], "src": TOPK["src"], "dst": TOPK["dst"], "ps": [0, 3, 4], "pd": [0, 3, 4], "ks": [1, 3],
            "mps": [0, 2]}


def case_null_unreachable():  # rows with a NULL id, an unreachable target, an isolated vertex
    return {"n": 5, "src": [0, 1, 2], "dst": [1, 2, 0], "ps": [0, 9, 0, 4, 4, 3], "pd": [2, 1, 9, 0, 4, 3],
            "sv": [1, 0, 1, 1, 1, 1], "dv": [1, 1, 0, 1, 1, 1], "ks": [2], "mps": [0, 1]}


def case_cut():  # the top_k graph from 0 to 3: a max_paths that cuts a group
    return {"n": TOPK["n"], "src": TOPK["src"], "dst": TOPK["dst"], "ps": [0, 0], "pd": [3, 3], "ks": [2, 3],
            "mps": [1, 2, 3]}


def case_rows(p, seed=3):  # p rows on a random graph
    rng = np.random.default_rng(seed)
    n = 200
    src, dst = rng.integers(0, n, 1200), rng.integers(0, n, 1200)
    ps = rng.choice(np.unique(src), p)
    pd = (ps + 1 + rng.integers(0, n - 1, p)) % n
    return {"n": n, "src": src.tolist(), "dst": dst.tolist(), "ps": ps.tolist(), "pd": pd.tolist(), "ks": [1, 2],
            "mps": [0, 3]}


CATALOGUE = {
    "bipartite": case_bipartite,
    "dag": case_dag,
    "self_loop_trap": case_self_loop_trap,
    "cycle_behind_chain": case_cycle_behind_chain,
    "diamonds": case_diamonds,
    "closed": case_closed,
    "null_unreachable": case_null_unreachable,
    "cut": case_cut,
    **{f"rows{p}": (lambda p=p: case_rows(p)) for p in (63, 65, 513)},
}


def run_oracle(c, k, max_paths, mode, lanes=0, count_only=False):
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    return okg.shortest_k_groups(c["n"], v, e, ids, c["ps"], c["pd"], k, max_paths, mode, c.get("sv"), c.get("dv"),
                                 lanes, count_only)


def test_catalogue_bipartite():
    c = case_bipartite()
    paths, rows, _ = run_oracle(c, 3, 0, "WALK")
    assert rows["last_len"].tolist() == [6, 4, 5] and rows["ngroups"].tolist() == [3, 3, 3]
    assert {h_of(p) for p in paths[0]} == {2, 4, 6}  # the odd lengths are skipped
    assert rows["count"][0] == 2 + 8 + 32
    paths, rows, _ = run_oracle(c, 3, 0, "TRAIL")
    assert {h_of(p) for p in paths[0]} == {2, 4, 6} and rows["ngroups"][0] == 3


def test_catalogue_dag():
    paths, rows, _ = run_oracle(case_dag(), 6, 0, "WALK")
    assert rows["ngroups"].tolist() == [3, 2] and rows["count"].tolist() == [4, 2]  # fewer than k groups
    assert rows["complete"].tolist() == [1, 1]
    for mode in ("TRAIL", "ACYCLIC", "SIMPLE"):
        mpaths, mrows, _ = run_oracle(case_dag(), 6, 0, mode)
        assert mpaths == paths and mrows["count"].tolist() == [4, 2]


def test_catalogue_self_loop_trap():
    paths, rows, st = run_oracle(case_self_loop_trap(), 3, 0, "WALK")
    assert paths == [[[0, 0, 1]]] and rows["ngroups"][0] == 1
    assert st["levels"] == 2  # the counts die on B(t) at h = 2: the self-loop at 2 is not counted


def test_catalogue_cycle_behind_chain():
    c = case_cycle_behind_chain()
    paths, rows, _ = run_oracle(c, 3, 0, "WALK")
    assert rows["last_len"].tolist() == [16, 17] and rows["count"].tolist() == [3, 3]
    assert [h_of(p) for p in paths[0]] == [12, 14, 16]
    _, rows, _ = run_oracle(c, 3, 0, "TRAIL")
    assert rows["ngroups"].tolist() == [2, 1]  # the cycle once, then no more trails


def test_catalogue_diamonds_saturate():
    c = case_diamonds()
    with pytest.raises(orc.OracleError) as ex:
        run_oracle(c, 1, 0, "WALK")
    assert ex.value.code == okg.ERR_UNSUPPORTED
    paths, rows, _ = run_oracle(c, 2, 5, "WALK")
    assert rows["count"][0] == INT64_MAX and rows["npaths"][0] == 5 and rows["complete"][0] == 0
    assert rows["ngroups"][0] == 2 and rows["last_len"][0] == 128 + 129
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    assert paths[0] == oks.shortest_k_paths(c["n"], v, e, ids, [0], [c["pd"][0]], 5)[0][0]
    _, cnt, _ = run_oracle(c, 2, 0, "WALK", count_only=True)  # counting alone does not list
    assert cnt["count"][0] == INT64_MAX


def test_catalogue_closed():
    c = case_closed()
    out = {m: run_oracle(c, 3, 0, m) for m in MODES}
    assert out["ACYCLIC"][0][0] == [[0]]
    assert out["SIMPLE"][0][0][0] == [0] and out["TRAIL"][0][0][0] == [0]
    # the closed walks through 0: 0 -> 3 -> 0, then two of 3 edges; groups h = 0, 2, 3
    for m in ("WALK", "TRAIL", "SIMPLE"):
        assert out[m][1]["last_len"][0] == 3 and out[m][1]["ngroups"][0] == 3 and out[m][1]["count"][0] == 4
    for m in MODES:
        paths, rows, st = run_oracle(c, 1, 0, m)
        assert paths == [[[0]], [[3]], [[4]]] and rows["count"].tolist() == [1, 1, 1]
        assert st["levels"] == 0  # k = 1: [s], no search


def test_catalogue_nulls():
    paths, rows, _ = run_oracle(case_null_unreachable(), 2, 0, "WALK")
    assert paths[:4] == [[[0, 0, 1, 1, 2], [0, 0, 1, 1, 2, 2, 0, 0, 1, 1, 2]], None, None, None]
    assert paths[4] == [[4]]
    assert rows["count"].tolist()[:4] == [2, 0, 0, 0] and rows["last_len"][1] == -1 and rows["complete"][1] == 1
    _, rows, _ = run_oracle(case_null_unreachable(), 2, 0, "TRAIL")
    assert rows["ngroups"].tolist() == [1, 0, 0, 0, 1, 1]


def test_catalogue_cut_by_max_paths():
    c = case_cut()
    for mode in ("TRAIL", "ACYCLIC", "SIMPLE"):
        paths, rows, _ = run_oracle(c, 2, 1, mode)
        assert len(paths[0]) == 1 and rows["complete"][0] == 0 and rows["count"][0] == -1
        assert rows["ngroups"][0] == 1 and rows["last_len"][0] == 1  # only the listed paths' groups
        _, rows, _ = run_oracle(c, 2, 3, mode)  # exactly N = 3 listed: complete
        assert rows["complete"][0] == 1 and rows["count"][0] == 3 and rows["ngroups"][0] == 2
    _, rows, _ = run_oracle(c, 2, 1, "WALK")
    assert rows["complete"][0] == 0 and rows["count"][0] == 3 and rows["ngroups"][0] == 2


def cycle_walk_limit():
    """a 256-cycle: the walks 0 -> 253 have lengths 253 + 256 j, one per group, the 256th exactly 65533 edges"""
    n = 256
    src, dst = np.arange(n), (np.arange(n) + 1) % n
    return n, src, dst


def test_catalogue_walk_limit():
    n, src, dst = cycle_walk_limit()
    v, e, ids = ref_csr(n, src, dst)
    paths, rows, _ = okg.shortest_k_groups(n, v, e, ids, [0], [253], 256, 0, "WALK")
    assert rows["last_len"][0] == PATH_MAX and rows["ngroups"][0] == 256 and h_of(paths[0][-1]) == PATH_MAX
    for count_only in (False, True):  # a 257th group lies one cycle past the limit
        with pytest.raises(orc.OracleError) as ex:
            okg.shortest_k_groups(n, v, e, ids, [0], [253], 257, 0, "WALK", count_only=count_only)
        assert ex.value.code == okg.ERR_UNSUPPORTED
    # the modes on a chain (their restatement keeps no count layers)
    n = PATH_MAX + 2
    v, e, ids = ref_csr(n, np.arange(n - 1), np.arange(1, n))
    paths, rows, _ = okg.shortest_k_groups(n, v, e, ids, [0], [PATH_MAX], 3, 0, "ACYCLIC")
    assert rows["last_len"][0] == PATH_MAX and len(paths[0]) == 1
    with pytest.raises(orc.OracleError) as ex:
        okg.shortest_k_groups(n, v, e, ids, [0], [PATH_MAX + 1], 1, 0, "ACYCLIC")
    assert ex.value.code == okg.ERR_UNSUPPORTED


def test_oracle_errors():
    v, e, ids = ref_csr(3, [0, 1], [1, 2])
    for kw, code in (({"k": 0}, okg.ERR_ARG), ({"max_paths": -1}, okg.ERR_ARG), ({"mode": "ANY"}, okg.ERR_ARG),
                     ({"mode": "TRAIL", "count_only": True}, okg.ERR_ARG), ({"lanes": 96}, okg.ERR_ARG),
                     ({"dst": [3]}, okg.ERR_RANGE)):
        args = {"src": [0], "dst": [1], "k": 1, **kw}
        with pytest.raises(orc.OracleError) as ex:
            okg.shortest_k_groups(3, v, e, ids, args.pop("src"), args.pop("dst"), args.pop("k"), **args)
        assert ex.value.code == code


# ---- GPU: the device against the oracle ------------------------------------------------------------------------------
def compare(csr, n, v, e, ids, ps, pd, k, max_paths, mode, sv=None, dv=None, options=None):
    paths, cnt, ng, last, comp, st = csr.shortest_k_groups(ps, pd, k, max_paths, sv, dv, options, mode)
    lanes = options.lanes if options else 0
    opaths, orows, ost = okg.shortest_k_groups(n, v, e, ids, ps, pd, k, max_paths, mode, sv, dv, lanes)
    assert paths == opaths
    assert np.array_equal(cnt, orows["count"]) and np.array_equal(ng, orows["ngroups"])
    assert np.array_equal(comp, orows["complete"]) and np.array_equal(last, orows["last_len"])
    counters = WALK_COUNTERS if mode == "WALK" else MODE_COUNTERS
    assert {x: st[x] for x in counters} == {x: ost[x] for x in counters}
    if mode == "WALK":
        ccnt, cng, clast, cvalid, cst = csr.shortest_k_groups_count(ps, pd, k, sv, dv, options)
        assert np.array_equal(ccnt, cnt) and np.array_equal(cng, ng) and np.array_equal(clast, last)
        assert np.array_equal(cvalid, (cnt > 0).astype(np.uint8))
        assert {x: cst[x] for x in counters} == {x: ost[x] for x in counters}
    return paths, st


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    c = CATALOGUE[name]()
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))
    for mode in MODES:
        for k in sorted(set(c["ks"]) | {1}):
            for max_paths in c["mps"]:
                if name == "diamonds" and mode == "WALK" and max_paths == 0:
                    with pytest.raises(pgq.PgqError) as ex:
                        csr.shortest_k_groups(c["ps"], c["pd"], k, 0)
                    assert ex.value.status == PGQ_ERR_UNSUPPORTED
                    continue
                if name == "diamonds" and mode != "WALK" and max_paths == 0:
                    continue  # 2^64 trails
                compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], k, max_paths, mode, c.get("sv"), c.get("dv"))
    csr.free()


@pytest.mark.gpu
def test_device_walk_limit_and_layer_budget(gpu_ctx, monkeypatch):
    n = PATH_MAX + 2
    src, dst = np.arange(n - 1), np.arange(1, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    # a group at the limit: counted (its layers are over the budget for a list), and listed in a mode
    cnt, ng, last, _, _ = csr.shortest_k_groups_count([0], [PATH_MAX], 3)
    assert (cnt.tolist(), ng.tolist(), last.tolist()) == ([1], [1], [PATH_MAX])
    paths, _ = compare(csr, n, v, e, ids, [0], [PATH_MAX], 3, 0, "ACYCLIC")
    assert h_of(paths[0][0]) == PATH_MAX
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_groups([0], [PATH_MAX], 1)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED  # the layer budget
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_groups_count([0], [PATH_MAX + 1], 1)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    for mode in ("WALK", "ACYCLIC"):
        with pytest.raises(pgq.PgqError) as ex:
            csr.shortest_k_groups([0], [PATH_MAX + 1], 1, mode=mode)
        assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()
    # the 256th group of a 256-cycle is exactly 65533 edges long, the 257th is past it
    n, src, dst = cycle_walk_limit()
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    paths, _ = compare(csr, n, v, e, ids, [0], [253], 256, 0, "WALK")
    assert h_of(paths[0][-1]) == PATH_MAX
    for call in (lambda: csr.shortest_k_groups([0], [253], 257), lambda: csr.shortest_k_groups_count([0], [253], 257)):
        with pytest.raises(pgq.PgqError) as ex:
            call()
        assert ex.value.status == PGQ_ERR_UNSUPPORTED
    csr.free()
    # the storing pass regroups its rows under a lower layer budget
    c = case_rows(65)
    v, e, ids = ref_csr(c["n"], c["src"], c["dst"])
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], np.asarray(c["src"]), np.asarray(c["dst"]))
    base, st = compare(csr, c["n"], v, e, ids, c["ps"], c["pd"], 3, 0, "WALK")
    last = csr.shortest_k_groups(c["ps"], c["pd"], 3)[3]
    assert (last >= 0).sum() > 2
    n_ab = len(set(np.asarray(c["dst"]).tolist()))  # the vertices with in-edges
    one_row = (int(last.max()) + 1) * n_ab * 8
    monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(one_row * 2))  # a row of the longest walk shares with one more
    paths, _, _, _, _, st2 = csr.shortest_k_groups(c["ps"], c["pd"], 3)
    assert paths == base
    assert st2["kernel_launches"] > st["kernel_launches"]  # (every extra group recomputes its layers)
    monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", "64")
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_groups(c["ps"], c["pd"], 3)
    assert ex.value.status == PGQ_ERR_UNSUPPORTED
    # counting alone keeps no layers, so the budget does not bound it
    ocount = okg.shortest_k_groups(c["n"], v, e, ids, c["ps"], c["pd"], 3)[1]["count"]
    assert np.array_equal(csr.shortest_k_groups_count(c["ps"], c["pd"], 3)[0], ocount)
    csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [12, 14])
def test_device_rmat(gpu_ctx, scale):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(512 if scale == 12 else 256, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    for mode in MODES:
        for k, max_paths in ((1, 0), (2, 16), (3, 8)) if mode == "WALK" else ((1, 0), (2, 8)):
            compare(csr, n, v, e, ids, ps, pd, k, max_paths, mode)
    csr.free()


@pytest.mark.gpu
def test_device_rmat16(gpu_ctx):
    n, src, dst = datagen.rmat_edges(16)
    ps, pd = datagen.hashed_pairs(512, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    ap, apc, _ = csr.all_shortest_paths(ps, pd, 6)
    pick = np.arange(0, len(ps), 37)
    for mode in ("WALK", "TRAIL", "ACYCLIC"):
        paths, cnt = csr.shortest_k_groups(ps, pd, 1, 6, mode=mode)[:2]
        assert all(paths[i] == ap[i] for i in range(len(ps)) if ps[i] != pd[i])
        if mode == "WALK":
            assert np.array_equal(cnt, apc)
        paths, cnt = csr.shortest_k_groups(ps, pd, 2, 6, mode=mode)[:2]
        opaths, orows, _ = okg.shortest_k_groups(n, v, e, ids, ps[pick], pd[pick], 2, 6, mode)
        assert [paths[i] for i in pick] == opaths and np.array_equal(cnt[pick], orows["count"])
    csr.free()


@pytest.mark.gpu
def test_device_lane_widths_and_row_order(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(700, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    for mode in ("WALK", "ACYCLIC"):
        base, _ = compare(csr, n, v, e, ids, ps, pd, 2, 8, mode)
        for lanes in range(64, 513, 64):
            paths, st = compare(csr, n, v, e, ids, ps, pd, 2, 8, mode, options=pgq.Options(lanes))
            assert paths == base and st["lanes"] == lanes
        perm = np.random.default_rng(1).permutation(len(ps))
        assert csr.shortest_k_groups(ps[perm], pd[perm], 2, 8, mode=mode)[0] == [base[i] for i in perm]
    csr.free()


@pytest.mark.gpu
def test_device_construction_routes(gpu_ctx):
    import torch
    n, src, dst = datagen.rmat_edges(10)
    ps, pd = datagen.hashed_pairs(300, n)
    v, e, ids = ref_csr(n, src, dst)
    for csr in (pgq.DeviceCSR.build(gpu_ctx, n, src, dst), pgq.DeviceCSR.upload(gpu_ctx, n, v, e, ids)):
        for mode in MODES:
            compare(csr, n, v, e, ids, ps, pd, 2, 6, mode)
        csr.free()
    vk = np.random.default_rng(4).permutation(n).astype(np.int64) * 3
    cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (vk, vk[src], vk[dst])]
    routes = [pgq.DeviceCSR.build_from_keys(gpu_ctx, vk, vk[src], vk[dst], undirected=u) for u in (False, True)]
    routes.append(pgq.DeviceCSR.build_from_keys_device(gpu_ctx, n, len(src), *(c.data_ptr() for c in cols)))
    for csr in routes:
        kv, ke, kids = csr.download()
        for mode in MODES:
            compare(csr, csr.n, kv, ke, kids, ps % csr.n, pd % csr.n, 2, 6, mode)
        csr.free()


@pytest.mark.gpu
def test_device_shortest_k_paths_unchanged(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(300, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    csr.shortest_k_groups(ps, pd, 2, 4, mode="TRAIL")  # (in between, on the same workspace)
    for mode in MODES:
        paths, npaths, _ = csr.shortest_k_paths(ps, pd, 6, mode=mode)
        if mode == "WALK":
            opaths, onp, _ = oks.shortest_k_paths(n, v, e, ids, ps, pd, 6)
        else:
            opaths, onp, _ = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, 6, mode)
        assert paths == opaths and np.array_equal(npaths, onp)
    csr.free()


@pytest.mark.gpu
def test_device_errors(gpu_ctx):
    csr = pgq.DeviceCSR.build(gpu_ctx, 4, np.array([0, 1, 2]), np.array([1, 2, 0]))
    with pytest.raises(pgq.InvalidInputException):
        csr.shortest_k_groups([0], [1], 2, mode="cheapest")
    for mode in MODES:
        for call, status in ((lambda: csr.shortest_k_groups([0, 4], [1, 1], 2, mode=mode), PGQ_ERR_RANGE),
                             (lambda: csr.shortest_k_groups([0], [1], 0, mode=mode), PGQ_ERR_INVALID_ARG),
                             (lambda: csr.shortest_k_groups([0], [1], 2, -1, mode=mode), PGQ_ERR_INVALID_ARG),
                             (lambda: csr.shortest_k_groups([0], [1], 2, options=pgq.Options(96), mode=mode),
                              PGQ_ERR_INVALID_ARG),
                             (lambda: csr.shortest_k_groups([0], [1], 2, options=pgq.Options(
                                 0, shard_index=0, shard_count=2), mode=mode), PGQ_ERR_UNSUPPORTED)):
            with pytest.raises(pgq.PgqError) as ex:
                call()
            assert ex.value.status == status
        paths, cnt, ng, last, comp, _ = csr.shortest_k_groups([0, 9], [9, 1], 3, 0, [1, 0], [0, 1], mode=mode)
        assert last.tolist() == [-1, -1]
        assert paths == [None, None] and cnt.tolist() == [0, 0] and ng.tolist() == [0, 0] and comp.tolist() == [1, 1]
        paths, st = csr.shortest_k_groups([], [], 3, mode=mode)[::5]
        assert paths == [] and st["batches"] == 0
    with pytest.raises(pgq.PgqError) as ex:
        csr.shortest_k_groups_count([0, 4], [1, 1], 2)
    assert ex.value.status == PGQ_ERR_RANGE
    csr.free()
    un = pgq.DeviceCSR.create(gpu_ctx, 3)
    for mode in ("WALK", "TRAIL"):
        with pytest.raises(pgq.PgqError) as ex:
            un.shortest_k_groups([0], [1], 2, mode=mode)
        assert ex.value.status == PGQ_ERR_NOT_INITIALIZED
    un.free()


@pytest.mark.gpu
def test_udf_mirror(gpu_ctx):
    state = pgq.DuckPGQState(gpu_ctx)
    pgq.create_csr_vertex(state, 0, 4, np.arange(4), np.array([2, 1, 1, 1]))
    pgq.create_csr_edge(state, 0, 4, 5, 5, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], [10, 11, 12, 13, 14])
    v, e, ids = ref_csr(4, [0, 0, 1, 2, 3], [1, 2, 3, 3, 0], np.arange(10, 15))
    assert pgq.shortest_k_groups(state, 0, 4, [0, 0], [3, 0], 1, 0, mode="acyclic") == \
        [[[0, 10, 1, 12, 3], [0, 11, 2, 13, 3]], [[0]]]
    for mode in MODES:
        assert pgq.shortest_k_groups(state, 0, 4, [0, 0], [3, 0], 2, 3, mode=mode) == \
            okg.shortest_k_groups(4, v, e, ids, [0, 0], [3, 0], 2, 3, mode)[0]
    counts, valid = pgq.shortest_k_groups_count(state, 0, 4, [0, 1], [3, 0], 2)
    assert counts.tolist() == [2 + 4, 1 + 2] and valid.tolist() == [1, 1]  # lengths 2 and 5 through the cycle
    with pytest.raises(pgq.InvalidInputException):
        pgq.shortest_k_groups(state, 0, 4, [0], [3], 2, mode="ANY")
    state.query_end()


@pytest.mark.gpu
def test_one_workspace_in_turn(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(300, n)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)

    def calls():
        return (csr.shortest_k_groups(ps, pd, 2, 8)[:2], csr.shortest_k_groups(ps, pd, 2, 8, mode="TRAIL")[:2],
                csr.shortest_k_paths(ps, pd, 8)[0], csr.shortest_k_groups_count(ps, pd, 3)[0].tolist())

    alone = calls()
    for _ in range(2):
        again = calls()
        assert again[0][0] == alone[0][0] and np.array_equal(again[0][1], alone[0][1])
        assert again[1][0] == alone[1][0] and again[2] == alone[2] and again[3] == alone[3]
    csr.free()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    n, src, dst = datagen.rmat_edges(12)
    ps, pd = datagen.hashed_pairs(200, n)
    v, e, ids = ref_csr(n, src, dst)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    exp = {m: okg.shortest_k_groups(n, v, e, ids, ps, pd, 2, 6, m)[0] for m in MODES}
    out = [None] * 8

    def work(i):
        out[i] = csr.shortest_k_groups(ps, pd, 2, 6, mode=MODES[i % 4])[0]

    ths = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(out[i] == exp[MODES[i % 4]] for i in range(8))
