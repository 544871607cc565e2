"""The BFS level loop under forced direction schedules, against the oracle.

The answers of iterativelength / shortestpath -- and the work counters, which the frontier sets define -- must not
depend on how each level was computed (DESIGN §3).  The heuristic alone rarely takes some of the direction changes
the mask-cleaning protocol exists for, so PGQ_B200_SCHEDULE forces them: character (level - 1) % len of the string
decides each level, b bottom-up, p top-down, t k_tail where eligible (top-down otherwise), a the heuristic.  Every
call runs with PGQ_B200_TRACE=1 and its per-level trace is checked against the schedule.
Also here: the depth limit of the path mode, and the device-pointer entry point that bench.py times."""
import re

import numpy as np
import pytest

from duckpgq_extension_b200 import datagen, pgq
from oracle import pgq_oracle as orc

pytestmark = pytest.mark.gpu

FIXED = ["b", "p", "t", "bp", "pb", "tb", "bt", "bbp", "pbb", "bpt", "tbp", "ppbb", "bbbt", "tttb"]
_r = np.random.default_rng(20261015)
RANDOM = ["".join(_r.choice(list("bpta"), size=int(_r.integers(2, 9)))) for _ in range(20)]
SCHEDULES = FIXED + RANDOM
GRAPHS = ["indeg", "outdeg", "tail", "rmat10", "rmat12", "snb"]
COUNTS = [1, 63, 64, 65, 511, 512, 513, 700]
LANES = [0, 64, 128, 256, 512]
CONFIGS = [(k, lanes, rb) for k in COUNTS for lanes in LANES for rb in (False, True)]
TRACE = re.compile(r"\[pgq\] batch (\d+) level (\d+) (push|pull|tail) frontier_v=(\d+) frontier_e=(\d+) items=(-?\d+)")


# ---- graphs: each family aims at a boundary of a kernel -------------------------------------------------------------
def _indeg_ladder():
    """Rows of the bottom-up layout: long rows (in-degree >= 32) of every size around the 256-position chunks and
    1024-position ranges, a short-row count that is not a multiple of 32, parallel edges, self-loops, and shuffled
    ids so that the internal renumbering matters.  Most vertices have no in-edges (outside n_reach)."""
    rng = np.random.default_rng(101)
    n = 5000
    ladder = [1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 2049, 4100]
    src, dst = [], []
    heads = rng.choice(n, 3 * len(ladder) + 1001, replace=False)
    for i, d in enumerate(ladder * 3):
        pool = rng.choice(n, max(2, d // 3), replace=False)  # sources drawn with replacement: parallel edges
        src.append(rng.choice(pool, d))
        dst.append(np.full(d, heads[i]))
    for h in heads[3 * len(ladder):]:  # 1001 short rows
        d = int(rng.integers(1, 32))
        src.append(rng.integers(0, n, d))
        dst.append(np.full(d, h))
    loops = rng.choice(heads, 40, replace=False)
    src.append(loops)
    dst.append(loops)
    src, dst = np.concatenate(src), np.concatenate(dst)
    perm = rng.permutation(n)
    return n, perm[src], perm[dst]


def _outdeg_ladder():
    """Top-down work items of <= 256 edges and the narrow / wide choice at fe < 8 * n_items."""
    rng = np.random.default_rng(102)
    n = 4000
    src, dst = [rng.integers(0, n, 6000)], [rng.integers(0, n, 6000)]
    hubs = rng.choice(n, 30, replace=False)
    for i, d in enumerate([1, 7, 8, 9, 255, 256, 257, 512, 513, 1100] * 3):
        src.append(np.full(d, hubs[i]))
        dst.append(rng.integers(0, n, d))
    return n, np.concatenate(src), np.concatenate(dst)


def _tail_thresholds():
    """Sources whose level-1 frontier is exactly at or one past k_tail's limits (256 items, 1024 out-edges), and
    chains around PGQ_TAIL_MAX = 32 levels.  Ids are not shuffled: TAIL_HUBS / TAIL_CHAINS name the sources."""
    rng = np.random.default_rng(103)
    src, dst = [], []
    nxt = [0]

    def new(k):
        a = np.arange(nxt[0], nxt[0] + k)
        nxt[0] += k
        return a

    chains = {}
    for length in (31, 32, 33, 64, 65):
        c = new(length)
        src.append(c[:-1])
        dst.append(c[1:])
        chains[length] = int(c[0])
    pool = new(300)
    src.append(pool)
    dst.append(rng.choice(list(chains.values()), 300))
    hubs = {}
    for name, leaves, degs in (("v256", 256, None), ("v257", 257, None), ("e1024", 128, 8), ("e1025", 128, 8)):
        h = new(1)
        lv = new(leaves)
        src.append(np.repeat(h, leaves))
        dst.append(lv)
        for j, leaf in enumerate(lv):
            d = 1 if degs is None else degs + (1 if name == "e1025" and j == 0 else 0)
            src.append(np.full(d, leaf))
            dst.append(rng.choice(pool, d, replace=False))
        hubs[name] = int(h[0])
    return nxt[0], np.concatenate(src), np.concatenate(dst), hubs, chains


_, _, _, TAIL_HUBS, TAIL_CHAINS = _tail_thresholds()


def _make(name):
    if name == "indeg":
        return _indeg_ladder()
    if name == "outdeg":
        return _outdeg_ladder()
    if name == "tail":
        return _tail_thresholds()[:3]
    if name.startswith("rmat"):
        return datagen.rmat_edges(int(name[4:]))
    n, src, dst, _ = datagen.snb_shaped_edges(1500, 16.0, seed=4)  # undirected: finished rows saturate early
    return n, src, dst


class Graph:
    def __init__(self, ctx, name):
        n, src, dst = _make(name)
        eid = np.arange(len(src), dtype=np.int64) * 3 + 11
        self.n = n
        self.csr = pgq.DeviceCSR.build(ctx, n, src, dst, eid)
        self.v, self.e, self.ids = self.csr.download()
        ov, oe, oids = orc.csr_build(n, src, dst, eid)
        assert np.array_equal(self.v, ov) and np.array_equal(self.e, oe) and np.array_equal(self.ids, oids)


@pytest.fixture(scope="module")
def graphs(gpu_ctx):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Graph(gpu_ctx, name)
        return cache[name]

    yield get
    for g in cache.values():
        g.csr.free()


def make_pairs(g, k, seed):
    """k distinct sources, a quarter of them (when there are) without in-edges, plus rows that repeat a source,
    src == dst rows and NULL sources, in shuffled order.  Three in four destinations have in-edges."""
    rng = np.random.default_rng(seed)
    n = g.n
    outdeg = np.diff(g.v[: n + 1])
    indeg = np.bincount(g.e, minlength=n)
    no_in = rng.permutation(np.flatnonzero((indeg == 0) & (outdeg > 0)))[: k // 4]
    rest = rng.permutation(np.setdiff1d(np.arange(n), no_in))[: k - len(no_in)]
    srcs = np.concatenate([no_in, rest])
    if k == 1:
        return srcs, rng.integers(0, n, 1), None
    has_in = np.flatnonzero(indeg > 0)
    dsts = np.where(rng.random(k) < 0.75, rng.choice(has_in, k), rng.integers(0, n, k))
    extra = k // 8 + 3
    rep = rng.choice(srcs, extra)
    same = rng.choice(srcs, 3)
    null = rng.integers(0, n, 3)
    ps = np.concatenate([srcs, rep, same, null])
    pd = np.concatenate([dsts, rng.integers(0, n, extra), same, rng.integers(0, n, 3)])
    sv = np.concatenate([np.ones(k + extra + 3, np.uint8), np.zeros(3, np.uint8)])
    order = rng.permutation(len(ps))
    return ps[order], pd[order], sv[order]


def check_trace(text, schedule, no_tail=False):
    """Every level line of the trace ran what the schedule asked for; returns the level-to-level transitions seen.
    A t level runs top-down only where k_tail is not eligible.  After a fused bottom-up level the frontier has no
    item list yet, and eligibility is judged on the bound fv + fe / 256 of its length."""
    lines = [(int(b), int(lv), kind, int(fv), int(fe), int(items)) for b, lv, kind, fv, fe, items in TRACE.findall(text)]
    seen = set()
    prev = None
    for b, lv, kind, fv, fe, items in lines:
        after_pull = prev is not None and prev[:2] == (b, lv - 1) and prev[2] == "pull"
        if after_pull:
            items = fv + fe // 256
        want = schedule[(lv - 1) % len(schedule)]
        if want == "b":
            assert kind == "pull", (schedule, b, lv, kind)
        elif want == "p":
            assert kind == "push", (schedule, b, lv, kind)
        elif want == "t" and kind != "tail":
            assert kind == "push" and (no_tail or items > 256 or fe > 1024), (schedule, b, lv, kind, items, fe)
        if lv == 1:
            seen.add(("start", kind))
        elif prev is not None and prev[0] == b and prev[1] == lv - 1:
            seen.add((prev[2], kind))
        prev = (b, lv, kind)
    return seen, lines


def run_lengths(g, ps, pd, sv, lanes, rb, **opt):
    """Device iterativelength == oracle: lengths, validity, and (explicit lane width) the work counters."""
    out, valid, st = g.csr.iterativelength(ps, pd, sv, pgq.Options(lanes, reference_batching=rb, **opt))
    if rb:
        exp, expv, ost = orc.iterativelength(g.n, g.v, g.e, ps, pd, sv, lanes or 512)
    else:
        exp, expv, ost, _ = orc.iterativelength_ex(g.n, g.v, g.e, ps, pd, sv, lanes or 512, prune=True, dedup=True)
    assert np.array_equal(valid, expv) and np.array_equal(out, exp)
    if lanes:
        assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
            ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices)
    return st


def run_paths(g, ps, pd, sv, lanes, rb):
    got, _ = g.csr.shortestpath(ps, pd, sv, pgq.Options(lanes, reference_batching=rb))
    exp, _ = orc.shortestpath(g.n, g.v, g.e, g.ids, ps, pd, sv, 512)
    assert got == exp


def _set_env(monkeypatch, schedule, streams=1, **extra):
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", str(streams))
    if schedule is None:
        monkeypatch.delenv("PGQ_B200_SCHEDULE", raising=False)
    else:
        monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
    for k, val in extra.items():
        monkeypatch.setenv(k, val)


# ---- every schedule on every graph family ---------------------------------------------------------------------------
@pytest.mark.parametrize("schedule", SCHEDULES)
@pytest.mark.parametrize("graph", GRAPHS)
def test_schedule_matches_oracle(graphs, monkeypatch, capfd, graph, schedule):
    case = GRAPHS.index(graph) * len(SCHEDULES) + SCHEDULES.index(schedule)
    g = graphs(graph)
    _set_env(monkeypatch, schedule, streams=1 + case % 2)
    capfd.readouterr()
    for c in (2 * case, 2 * case + 1):
        k, lanes, rb = CONFIGS[c % len(CONFIGS)]
        ps, pd, sv = make_pairs(g, k, seed=c)
        run_lengths(g, ps, pd, sv, lanes, rb)
    ps, pd, sv = make_pairs(g, 65, seed=case)
    run_paths(g, ps, pd, sv, [0, 64, 512][case % 3], case % 2 == 0)
    _, lines = check_trace(capfd.readouterr().err, schedule)
    assert lines


@pytest.mark.parametrize("alpha", [1, 3, 64, 1 << 30])
@pytest.mark.parametrize("graph", GRAPHS)
def test_alpha_matches_oracle(graphs, monkeypatch, graph, alpha):
    """The heuristic's cost ratio moves the direction changes to other levels; answers and counters stay."""
    g = graphs(graph)
    _set_env(monkeypatch, None)
    for k, lanes, rb in ((700, 64, False), (513, 256, True), (65, 0, False)):
        ps, pd, sv = make_pairs(g, k, seed=alpha + k)
        run_lengths(g, ps, pd, sv, lanes, rb, alpha=alpha)


VARIANT_SCHEDULES = ["bp", "pb", "tb", "bt", "bbp", "tbp", "bbbt", "ppbb"] + RANDOM[:4]
VARIANTS = [{"PGQ_B200_PULL_SKIP": "0"}, {"PGQ_B200_NO_TAIL": "1"}]


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "-".join(f"{k[9:]}={x}" for k, x in v.items()))
@pytest.mark.parametrize("schedule", VARIANT_SCHEDULES)
@pytest.mark.parametrize("graph", ["indeg", "snb", "rmat12"])
def test_variant_schedule_matches_oracle(graphs, monkeypatch, capfd, graph, schedule, variant):
    """Without skipping finished rows, and without k_tail."""
    g = graphs(graph)
    _set_env(monkeypatch, schedule, **variant)
    capfd.readouterr()
    seed = VARIANT_SCHEDULES.index(schedule)
    for k, lanes, rb in ((700, 64, False), (513, 128, True)):
        ps, pd, sv = make_pairs(g, k, seed=seed + k)
        run_lengths(g, ps, pd, sv, lanes, rb)
    ps, pd, sv = make_pairs(g, 64, seed=seed)
    run_paths(g, ps, pd, sv, 64, seed % 2 == 0)
    check_trace(capfd.readouterr().err, schedule, no_tail="PGQ_B200_NO_TAIL" in variant)


@pytest.mark.parametrize("schedule", ["a", "t", "pt", "tb", "bt", "p"])
def test_tail_thresholds(graphs, monkeypatch, capfd, schedule):
    """One source per call: a level-1 frontier of exactly 256 / 257 items or 1024 / 1025 out-edges, and chains
    of 31 ... 65 vertices.  Under t the second level is k_tail exactly when it is within both limits."""
    g = graphs("tail")
    _set_env(monkeypatch, schedule)
    eligible = {"v256": True, "v257": False, "e1024": True, "e1025": False}
    for name, hub in TAIL_HUBS.items():
        capfd.readouterr()
        run_lengths(g, [hub] * 5, [hub + 1, (hub + 300) % g.n, 0, 40, 200], None, 64, True)
        run_paths(g, [hub] * 3, [hub + 1, 30, 100], None, 64, False)
        _, lines = check_trace(capfd.readouterr().err, schedule)
        if schedule in ("t", "pt"):
            level2 = [kind for b, lv, kind, fv, fe, items in lines if lv == 2]
            assert level2 and set(level2) == {"tail" if eligible[name] else "push"}, (name, level2)
    for length, head in TAIL_CHAINS.items():
        ps = np.array([head] * 3)
        pd = np.array([head + length - 1, head + length // 2, head + 1])
        run_lengths(g, ps, pd, None, 64, True)
        run_lengths(g, ps, pd, None, 64, False)
        run_paths(g, ps, pd, None, 64, True)
    check_trace(capfd.readouterr().err, schedule)


def test_every_transition_is_forced(graphs, monkeypatch, capfd):
    """The trace shows each change of direction the cleaning protocol has to survive."""
    seen = set()
    g = graphs("tail")
    chain = TAIL_CHAINS[65]
    for schedule in ("bp", "bt", "tb", "pbb", "tttb"):
        _set_env(monkeypatch, schedule)
        capfd.readouterr()
        run_lengths(g, [chain, chain], [chain + 64, chain + 10], None, 64, True)
        run_lengths(g, [TAIL_HUBS["v256"]], [TAIL_CHAINS[33] + 32], None, 64, False)
        seen |= check_trace(capfd.readouterr().err, schedule)[0]
    g = graphs("indeg")
    for schedule in ("bp", "pb", "b"):
        _set_env(monkeypatch, schedule)
        capfd.readouterr()
        ps, pd, sv = make_pairs(g, 513, seed=7)
        run_lengths(g, ps, pd, sv, 64, False)
        seen |= check_trace(capfd.readouterr().err, schedule)[0]
    for t in [("pull", "push"), ("push", "pull"), ("pull", "tail"), ("tail", "pull"), ("start", "pull")]:
        assert t in seen, (t, sorted(seen))


# ---- several batches, pooled workspaces ------------------------------------------------------------------------------
SEQUENCE = [  # (graph, schedule, pairs, lanes, reference batching): lane width, CSR and schedule change call to call
    ("indeg", "b", 700, 64, False), ("indeg", "bp", 700, 64, True), ("indeg", "bt", 513, 128, False),
    ("snb", "bbp", 700, 64, False), ("snb", "pbb", 511, 128, True), ("indeg", "tbp", 700, 64, False),
    ("indeg", "b", 513, 256, True), ("rmat12", "bbbt", 700, 64, False), ("snb", "bpt", 700, 64, False),
    ("indeg", "ppbb", 700, 128, False), ("indeg", "b", 700, 64, False),
]


@pytest.mark.parametrize("streams", [1, 2])
@pytest.mark.parametrize("fresh", [False, True], ids=["pooled", "one-workspace"])
def test_consecutive_calls_reuse_workspaces(gpu_ctx, graphs, monkeypatch, capfd, streams, fresh):
    """Later batches on a workspace clear only the first n_reach rows of the mask arrays ("known clean"): whatever
    a batch leaves behind beyond them reaches the next batch.  With a fresh context that may hold one workspace,
    every batch of every call runs on the same arrays."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0) if fresh else gpu_ctx
    local = {}
    try:
        for i, (name, schedule, k, lanes, rb) in enumerate(SEQUENCE):
            if fresh:
                if name not in local:
                    local[name] = Graph(ctx, name)
                g = local[name]
            else:
                g = graphs(name)
            _set_env(monkeypatch, schedule, streams=streams)
            capfd.readouterr()
            ps, pd, sv = make_pairs(g, k, seed=100 + i)
            st = run_lengths(g, ps, pd, sv, lanes, rb)
            assert st["batches"] > 1
            if i % 3 == 0:
                run_paths(g, ps[:200], pd[:200], sv[:200], lanes, rb)
            check_trace(capfd.readouterr().err, schedule)
    finally:
        for g in local.values():
            g.csr.free()
        if fresh:
            ctx.close()


# ---- path-mode depth limit --------------------------------------------------------------------------------------------
DEPTH_OK = 65533  # DESIGN §7: shortestpath supports BFS depths < 65 534


def _chain(ctx, vertices):
    src = np.arange(vertices - 1, dtype=np.int64)
    return pgq.DeviceCSR.build(ctx, vertices, src, src + 1, src * 2 + 5)


def _chain_path(d):
    out = [0]
    for i in range(d):
        out += [2 * i + 5, i + 1]
    return out


@pytest.mark.parametrize("schedule", ["a", "b"])
def test_path_depth_limit(gpu_ctx, graphs, monkeypatch, schedule):
    """A chain of DEPTH_OK + 1 vertices is the longest shortestpath answers, with and without reference batching
    (which runs the batch on until its frontier is empty, one level deeper); one more vertex is PGQ_ERR_UNSUPPORTED.
    Under a, k_tail runs the levels 32 at a time up to the clamp; under b every level is a bottom-up round trip."""
    _set_env(monkeypatch, schedule)
    monkeypatch.delenv("PGQ_B200_TRACE")
    ok, deep = _chain(gpu_ctx, DEPTH_OK + 1), _chain(gpu_ctx, DEPTH_OK + 2)
    try:
        for rb in (False, True):
            paths, st = ok.shortestpath([0, 5, 0], [DEPTH_OK, DEPTH_OK, 7], None, pgq.Options(reference_batching=rb))
            assert paths[0] == _chain_path(DEPTH_OK)
            assert paths[1] == _chain_path(DEPTH_OK)[10:] and paths[2] == _chain_path(7)
            with pytest.raises(pgq.PgqError) as err:
                deep.shortestpath([0], [DEPTH_OK + 1], None, pgq.Options(reference_batching=rb))
            assert err.value.status == pgq.PGQ_ERR_UNSUPPORTED
            # the context recovers: the same CSR and another one answer ordinary calls
            paths, _ = deep.shortestpath([3, 10], [1000, 12], None, pgq.Options(reference_batching=rb))
            assert paths == [_chain_path(1000)[6:], _chain_path(12)[20:]]
            g = graphs("rmat10")
            ps, pd, sv = make_pairs(g, 65, seed=3)
            run_lengths(g, ps, pd, sv, 64, rb)
            run_paths(g, ps, pd, sv, 64, rb)
        # iterativelength keeps no level array: no depth limit
        for rb in (False, True):
            out, valid, _ = deep.iterativelength([0, 1], [DEPTH_OK + 1, 0], None, pgq.Options(reference_batching=rb))
            assert out.tolist() == [DEPTH_OK + 1, -1] and valid.tolist() == [1, 0]
    finally:
        ok.free()
        deep.free()


def test_iterativelength_long_chain(gpu_ctx, monkeypatch):
    monkeypatch.delenv("PGQ_B200_SCHEDULE", raising=False)
    csr = _chain(gpu_ctx, 70000)
    try:
        for rb in (False, True):
            out, valid, st = csr.iterativelength([0, 5], [69999, 69000], None, pgq.Options(64, reference_batching=rb))
            assert out.tolist() == [69999, 68995] and valid.tolist() == [1, 1]
    finally:
        csr.free()


# ---- device-pointer entry point -------------------------------------------------------------------------------------
def test_iterativelength_device_entry(graphs, monkeypatch):
    """pgq_iterativelength_device (what bench.py times) == the host-pointer entry == the oracle, on the default
    stream and on a side stream whose inputs are written on it right before the call; outputs start as garbage."""
    import torch

    g = graphs("rmat12")
    monkeypatch.delenv("PGQ_B200_SCHEDULE", raising=False)
    ps, pd, sv = make_pairs(g, 700, seed=42)
    p = len(ps)
    opts = pgq.Options(64)
    for with_sv in (False, True):
        hsv = sv if with_sv else None
        exp, expv, _ = orc.iterativelength(g.n, g.v, g.e, ps, pd, hsv)
        hout, hvalid, hst = g.csr.iterativelength(ps, pd, hsv, opts)
        assert np.array_equal(hout, exp) and np.array_equal(hvalid, expv) and hst["batches"] > 1
        for side in (False, True):
            stream = torch.cuda.Stream() if side else torch.cuda.default_stream()
            d_src = torch.empty(p, dtype=torch.int64, device="cuda")
            d_dst = torch.empty_like(d_src)
            d_sv = torch.empty(p, dtype=torch.uint8, device="cuda")
            out = torch.empty_like(d_src)
            valid = torch.empty_like(d_sv)
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                d_src.copy_(torch.from_numpy(ps).pin_memory(), non_blocking=True)
                d_dst.copy_(torch.from_numpy(pd).pin_memory(), non_blocking=True)
                d_sv.copy_(torch.from_numpy(sv).pin_memory(), non_blocking=True)
                out.fill_(0x5A5A5A5A5A5A5A5A)
                valid.fill_(0x77)
                st = g.csr.iterativelength_device(d_src.data_ptr(), d_dst.data_ptr(), p, out.data_ptr(),
                                                  valid.data_ptr(), d_sv.data_ptr() if with_sv else 0,
                                                  stream.cuda_stream, opts)
            stream.synchronize()
            assert np.array_equal(out.cpu().numpy(), hout) and np.array_equal(valid.cpu().numpy(), hvalid)
            assert st["batches"] == hst["batches"] and st["levels"] == hst["levels"]
    # p = 0 touches nothing
    out.fill_(0x5A5A5A5A5A5A5A5A)
    g.csr.iterativelength_device(d_src.data_ptr(), d_dst.data_ptr(), 0, out.data_ptr(), valid.data_ptr())
    torch.cuda.synchronize()
    assert (out == 0x5A5A5A5A5A5A5A5A).all()
    # an id outside [0, n) is PGQ_ERR_RANGE
    d_dst[17] = g.n
    with pytest.raises(pgq.InvalidInputException) as err:
        g.csr.iterativelength_device(d_src.data_ptr(), d_dst.data_ptr(), p, out.data_ptr(), valid.data_ptr())
    assert err.value.status == pgq.PGQ_ERR_RANGE
