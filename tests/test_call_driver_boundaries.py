"""The call driver of iterativelength and shortestpath at its own boundaries, against a restatement that shows the lane map.

Every iterativelength and shortestpath call goes through the call driver of csrc/pgq_bfs.cu: k_assign classifies the
rows and hands out one lane per distinct source in first-appearance order (hash table with linear probing, tile counts
plus a block scan, the deal over shards, the rows per 64-lane group), run_call plans the batches (pick_lanes, applied
again to the remainder when lanes = 0), k_init_batch collects a batch's rows, and the k_path_* kernels rebuild the
paths (slot allocator, the walk buffer that grows between batches, the in-list scan for the smallest parent in ORIGINAL
ids, the out-list scan for the FIRST position, list offsets in tiles of 1024 rows).  A wrong lane order or batch plan
changes no answer, only searches / batches / levels / edges_traversed; a wrong tie-break changes a path only where
there is a tie.  So:

- driver_run, a numpy restatement from the edge rows that shows its work: per row the class, the lane and the owning
  shard; per call the counters, the rows per lane group, the batch plan and the trailing-batch rule; per batch and
  level the frontier and the rows answered, with the stop reason; per path every walk step (in-degree and out-degree
  scanned, tied candidates).  It equals oracle/pgq_oracle.c wherever the oracle can express the case (CPU);
- a catalogue of cases that each name what they hit, proven on the CPU from the restatement's output and layout();
- on the GPU every case under the option sets and lane widths that apply, with the per-level trace compared line by
  line, shards, the raw list ABI, the other construction routes, one dirty workspace and eight threads on one CSR."""
import ctypes as C
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import shortest_path as sp_shortest_path

from duckpgq_extension_b200 import _native, pgq
from oracle import pgq_oracle as orc
from test_csr_layout_shapes import ROUTES, _oracle, check_download, layout, make

H100_SMS = 132            # the H100 SXM; the GPU tests read the device's own count
TILE = 1024               # rows per tile of k_assign and of k_path_offsets
WALK_THREADS = 128        # k_path_walk's block: the in-list and out-list scans stride by this
WALK_BLOCKS_PER_SM = 16   # k_path_walk's grid cap
PLACE_BLOCKS = 4096       # k_path_place's grid cap
SHORT_DEG = 32            # in-degree from which a row lies in the long part of the bottom-up layout
REF, NO_DEDUP, NO_PRUNE = 1, 2, 4  # PGQ_OPT_REFERENCE_BATCHING / _NO_DEDUP / _NO_PRUNE
OPTION_SETS = {"default": 0, "no_dedup": NO_DEDUP, "no_prune": NO_PRUNE, "reference_batching": REF}
NULL, TRIVIAL, PRUNED, SEARCH = 0, 1, 2, 3
P_SIZES = [1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049]
LANE_TOTALS = [1, 63, 64, 65, 128, 129, 256, 257, 511, 512, 513, 1024, 1025, 1100]
IN_DEGREES = [1, 127, 128, 129, 3000]
OUT_DEGREES = [1, 128, 129, 3000]


class RangeError(ValueError):
    pass


def options(lanes=0, flags=0, shard_index=0, shard_count=0):
    return pgq.Options(lanes, reference_batching=bool(flags & REF), no_dedup=bool(flags & NO_DEDUP),
                       no_prune=bool(flags & NO_PRUNE), shard_index=shard_index, shard_count=shard_count)


def pick_lanes(lanes, n, searches, path):
    """run_call's lane width: the caller's, or 512 on a graph whose 64 B masks fit 32 MiB (256 otherwise), halved
    while the per-lane level array of path mode exceeds 4 GiB, then while half of it holds the searches."""
    if lanes:
        return lanes
    w = 512 if n * 64 <= (32 << 20) else 256
    if path:
        while w > 64 and n * w * 2 > (4 << 30):
            w >>= 1
    while w > 64 and searches <= w // 2:
        w >>= 1
    return w


def hash_u32(x):
    x = np.asarray(x, dtype=np.uint64) & np.uint64(0xffffffff)
    m = np.uint64(0xffffffff)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7feb352d)) & m
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846ca68b)) & m
    x ^= x >> np.uint64(16)
    return x.astype(np.int64)


def hash_size(p):
    h = 64
    while h < 2 * p:
        h <<= 1
    return h


# ---- the graph as the driver sees it ----------------------------------------------------------------------------------
class Graph:
    """The reference's CSR of the edge rows, the device's internal order (layout()) and the in-lists in the device's
    order: by the tail's internal id, parallel edges in CSR order."""

    def __init__(self, n, src, dst, edge_id=None):
        self.n = n
        self.src, self.dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
        self.edge_id = edge_id
        self.v, self.e, self.ids = orc.csr_build(n, self.src, self.dst, None if isinstance(edge_id, str) else edge_id)
        if isinstance(edge_id, str):  # "position": a CSR uploaded without edge ids reports the CSR position
            self.ids = np.arange(len(self.e), dtype=np.int64)
        self.lay = layout(n, self.src, self.dst)
        self.od, self.ind = self.lay["od"], self.lay["ind"]
        self.perm = np.empty(n, np.int64)  # original id -> internal id
        self.perm[self.lay["inv"]] = np.arange(n)
        self.row = np.repeat(np.arange(n), self.od)
        order = np.lexsort((self.perm[self.row], self.e))
        self.in_src = self.row[order]
        self.in_off = np.concatenate([[0], np.cumsum(self.ind)])
        by_head = np.argsort(self.e, kind="stable")
        self.pull_src = self.row[by_head]
        self.heads, self.starts = np.unique(self.e[by_head], return_index=True)
        self.has_out, self.has_in = np.flatnonzero(self.od > 0), np.flatnonzero(self.ind > 0)
        self.mat = sp.csr_matrix((np.ones(len(self.src)), (self.src, self.dst)), shape=(n, n))
        self._dist, self._walk = {}, {}

    def ins(self, x):
        return self.in_src[self.in_off[x]:self.in_off[x + 1]]

    def outs(self, x):
        return self.e[self.v[x]:self.v[x + 1]]

    def dist(self, s):
        """Hop counts from s (-1 = unreachable), by scipy."""
        if s not in self._dist:
            d = sp_shortest_path(self.mat, method="D", unweighted=True, indices=[s])[0]
            self._dist[s] = np.where(np.isfinite(d), d, -1).astype(np.int64)
        return self._dist[s]

    def walk(self, s, d):
        """The reference's path of (s, d) -> ([src, e1, v1, ..., dst] or None, one dict per walk step): the parent of
        a node reached at level k is the smallest ORIGINAL id among the lane's level k - 1 vertices with an edge to
        it, the edge the FIRST CSR position of the node in the parent's out-list."""
        if (s, d) not in self._walk:
            self._walk[(s, d)] = self._do_walk(s, d)
        return self._walk[(s, d)]

    def _do_walk(self, s, d):
        if s == d:
            return [s], []
        dist = self.dist(s)
        if dist[d] < 0:
            return None, []
        out, steps, cur = [d], [], d
        for k in range(int(dist[d]), 0, -1):
            ins = self.ins(cur)
            match = np.flatnonzero(dist[ins] == k - 1)
            cand = np.unique(ins[match])
            parent = int(cand[0])
            outs = self.outs(parent)
            at = np.flatnonzero(outs == cur)
            steps.append(dict(node=cur, parent=parent, indeg=len(ins), match=match, cand=cand, outdeg=len(outs),
                              edge_pos=int(at[0]), dup=len(at)))
            out += [int(self.ids[self.v[parent] + at[0]]), parent]
            cur = parent
        return out[::-1], steps


def graph(n, src_e, dst_e, edge_id=None):
    return _oracle("call_driver_graph", lambda: Graph(n, src_e, dst_e, edge_id), n, np.asarray(src_e),
                   np.asarray(dst_e), edge_id)


# ---- the restatement that shows its work ------------------------------------------------------------------------------
def driver_run(n, src_e, dst_e, ps, pd, sv=None, lanes=0, flags=0, shard_index=0, shard_count=1, path=False,
               edge_id=None):
    """k_assign, run_call's batch plan and the level loop, restated from the edge rows -> dict:
    per row   cls (NULL / TRIVIAL / PRUNED / SEARCH), ordinal (first-appearance ordinal of its source, or its own
              without dedup; -1 = takes no lane), lane (within this shard, -1 = not this shard's), leaders (the rows
              that open a lane), out / valid (lengths) or paths and steps (path mode);
    per call  searches, pruned, search_rows, grp_rows, plan [(pos, take, width)], lanes, trailing, batches, levels,
              edges, fv;
    per batch runs[b] = dict(rows, rows_ub, levels, stop), and trace = one dict per level (batch, level, fv, fe,
              answered rows)."""
    g = graph(n, src_e, dst_e, edge_id)
    ps, pd = np.asarray(ps, dtype=np.int64), np.asarray(pd, dtype=np.int64)
    p = len(ps)
    ref = bool(flags & REF)
    prune = not (ref or flags & NO_PRUNE)
    dedup = not (ref or flags & NO_DEDUP)
    sc = shard_count if shard_count > 1 else 1
    si = shard_index if sc > 1 else 0
    ok = np.ones(p, bool) if sv is None else np.asarray(sv) != 0
    same = ps == pd
    in_range = (ps >= 0) & (ps < n) & (pd >= 0) & (pd < n)
    if path:  # the range is checked first; src == dst is a list [src], answered on the spot only with the shortcut
        bad = ok & ~in_range
        trivial = ok & in_range & same & prune
    else:     # src == dst is 0 whatever the id
        trivial = ok & same
        bad = ok & ~same & ~in_range
    if bad.any():
        raise RangeError("source or destination outside [0, n)")
    cand = ok & ~trivial
    s0, d0 = np.where(cand, ps, 0), np.where(cand, pd, 0)
    pruned = cand & prune & ~same & ((g.od[s0] == 0) | (g.ind[d0] == 0))
    search = cand & ~pruned
    cls = np.full(p, NULL)
    cls[trivial], cls[pruned], cls[search] = TRIVIAL, PRUNED, SEARCH
    rows = np.flatnonzero(search)
    if dedup and len(rows):
        uniq, first = np.unique(ps[rows], return_index=True)
        rank = np.empty(len(uniq), np.int64)
        rank[np.argsort(first)] = np.arange(len(uniq))
        ord_row = rank[np.searchsorted(uniq, ps[rows])]
        lane_src_all = uniq[np.argsort(first)]
        leaders = rows[np.sort(first)]
    else:
        ord_row, lane_src_all, leaders = np.arange(len(rows)), ps[rows], rows
    ordinal = np.full(p, -1, np.int64)
    ordinal[rows] = ord_row
    lane = np.full(p, -1, np.int64)
    mine = ord_row % sc == si
    lane[rows[mine]] = ord_row[mine] // sc
    lane_src = lane_src_all[si::sc]
    total = len(lane_src)
    res = dict(cls=cls, ordinal=ordinal, lane=lane, leaders=leaders, all_lanes=len(lane_src_all), lane_src=lane_src,
               searches=total, pruned=int(pruned.sum() + (trivial.sum() if path else 0)),
               search_rows=int((lane >= 0).sum()), grp_rows=np.bincount(lane[lane >= 0] >> 6, minlength=p // 64 + 2),
               lanes=pick_lanes(lanes, n, total, path), batches=0, levels=0, edges=0, fv=0, runs=[], trace=[])
    plan, pos = [], 0
    while pos < total:
        w = lanes or pick_lanes(0, n, total - pos, path)
        plan.append((pos, min(total - pos, w), w))
        pos += plan[-1][1]
    res["plan"] = plan
    # the reference's batch loop starts one more batch behind a full last one (or when no row took a lane) if rows
    # without a lane follow; the device counts it only where its batches are the reference's
    res["trailing"] = bool(ref and lanes and sc <= 1 and p > 0 and (not plan or plan[-1][1] == plan[-1][2]) and
                           lane[p - 1] < 0)
    out = np.full(p, -1, np.int64)
    valid = np.zeros(p, np.uint8)
    if not path:
        out[trivial], valid[trivial] = 0, 1
    one = np.uint64(1)
    for b, (pos, take, w) in enumerate(plan):
        words = (take + 63) // 64
        l = np.arange(take)
        visit = np.zeros((n, words), np.uint64)
        seen = np.zeros((n, words), np.uint64)
        np.bitwise_or.at(visit, (lane_src[pos:pos + take], l >> 6), np.left_shift(one, (l & 63).astype(np.uint64)))
        brows = np.flatnonzero((lane >= pos) & (lane < pos + take))
        bl, bd = lane[brows] - pos, pd[brows]
        open_ = np.ones(len(brows), bool)
        path_stop = (not ref) or take == w
        g0, g1 = pos // 64, (pos + take - 1) // 64
        run = dict(rows=brows, rows_ub=int(res["grp_rows"][g0:g1 + 1].sum()), levels=0, stop=None)
        res["runs"].append(run)
        res["batches"] += 1
        it = 1
        while True:
            fr = visit.any(axis=1)
            rec = dict(batch=b, level=it, fv=int(fr.sum()), fe=int(g.od[fr].sum()), answered=np.zeros(0, np.int64))
            res["trace"].append(rec)
            res["levels"] += 1
            res["edges"] += rec["fe"]
            res["fv"] += rec["fv"]
            run["levels"] = it
            nxt = np.zeros((n, words), np.uint64)
            if len(g.heads):
                nxt[g.heads] = np.bitwise_or.reduceat(visit[g.pull_src], g.starts, axis=0)
            nxt &= ~seen
            seen |= nxt
            visit = nxt
            if not nxt.any():
                run["stop"] = "frontier_empty"
                break
            found = ((seen[bd, bl >> 6] >> (bl & 63).astype(np.uint64)) & one) != 0
            if path:
                if path_stop and found.all():
                    run["stop"] = "path_stop"
                    break
            else:
                new = found & open_
                out[brows[new]], valid[brows[new]] = it, 1
                rec["answered"] = brows[new]
                open_ &= ~found
                if not open_.any():
                    run["stop"] = "all_answered"
                    break
            it += 1
    if res["trailing"]:
        res["batches"] += 1
    if path:
        paths, steps = [None] * p, {}
        for r in np.flatnonzero(trivial):
            paths[r] = [int(ps[r])]
        for r in np.flatnonzero(lane >= 0):
            paths[r], steps[int(r)] = g.walk(int(ps[r]), int(pd[r]))
        res["paths"], res["steps"] = paths, steps
    else:
        res["out"], res["valid"] = out, valid
    return res


# ---- shapes -------------------------------------------------------------------------------------------------------------
@dataclass
class DShape:
    n: int
    src: np.ndarray
    dst: np.ndarray
    eid: object = None
    mark: dict = field(default_factory=dict)  # named vertices (original ids)


def _edge_ids(m, seed):
    return np.random.default_rng(seed).permutation(m).astype(np.int64) * 3 + 5


def base_shape():
    """3000 body vertices with 1 .. 4 out-edges into the body and 100 sinks, 100 sources without in-edges, 100
    isolated vertices and a ring of 100 that nothing else touches; ids shuffled, edge rowids non-contiguous."""
    rng = np.random.default_rng(300)
    body, sinks, outs, iso, ring = 3000, 100, 100, 100, 100
    od = rng.integers(1, 5, body)
    s = np.repeat(np.arange(body), od)
    d = rng.integers(0, body + sinks, len(s))
    s2 = np.repeat(np.arange(body + sinks, body + sinks + outs), 2)
    d2 = rng.integers(0, body, len(s2))
    r0 = body + sinks + outs + iso
    s3 = np.arange(r0, r0 + ring)
    d3 = r0 + (np.arange(ring) + 1) % ring
    n = r0 + ring
    perm = rng.permutation(n)
    src, dst = perm[np.concatenate([s, s2, s3])], perm[np.concatenate([d, d2, d3])]
    return DShape(n, src, dst, _edge_ids(len(src), 301), dict(ring=perm[s3], iso=perm[body + sinks + outs:r0]))


def chain_shape():
    """c0 -> c1 -> ... -> c259 with an extra vertex in front of c0 and a few leaves; ids shuffled."""
    rng = np.random.default_rng(310)
    k = 260
    s = np.concatenate([np.arange(k - 1), [k], rng.integers(0, k, 30)])
    d = np.concatenate([np.arange(1, k), [0], np.arange(k + 1, k + 31)])
    n = k + 31
    perm = rng.permutation(n)
    return DShape(n, perm[s], perm[d], _edge_ids(len(s), 311), dict(chain=perm[:k]))


def walk_shape():
    """The shapes k_path_walk's two scans are aimed at, ids as allocated (the internal order of vertices with equal
    class and degree is the original one, so in-list positions are chosen by id):
    in_<k>   S -> mids -> D with in-degree k; the other in-neighbours hang on a vertex S does not reach.  The mids sit
             at the first (127), the last (128) and several (129, 3000) in-list positions;
    out_<k>  S -> P -> C, P with out-degree k; the edge to C at position 0 (128), at the last position (129) and three
             times (3000, the first must be reported);
    tie      S -> A, B -> T with A < B in original ids and B the larger degree, hence the smaller internal id;
    tie_mix  the same with one candidate in the long part of the bottom-up layout (in-degree 40) and one short;
    cyc_<c>  a source on a cycle of length c (1 = a self-loop) with a destination 7 hops away that has a self-loop."""
    src, dst, mark = [], [], {}
    nxt = [0]

    def new(k=1):
        a = np.arange(nxt[0], nxt[0] + k)
        nxt[0] += k
        return a if k > 1 else int(a[0])

    def edge(a, b):
        src.append(int(a))
        dst.append(int(b))

    away = new()  # reaches the fillers; nothing reaches it
    for k, ranks in zip(IN_DEGREES, ([0], [0], [127], [0, 64, 128], [5, 1500, 2999])):
        s, d = new(), new()
        nb = np.atleast_1d(new(k))
        for i, x in enumerate(nb):
            edge(s if i in ranks else away, x)
        for x in nb:
            edge(x, d)
        mark[f"in_{k}"] = (s, d)
    for k, at in zip(OUT_DEGREES, ([0], [0], [128], [10, 2000, 2999])):
        s, par, c = new(), new(), new()
        junk = new()
        edge(s, par)
        for i in range(k):
            edge(par, c if i in at else junk)
        mark[f"out_{k}"] = (s, c)
    s, a, b, t = new(), new(), new(), new()
    for x in (a, b):
        edge(s, x)
        edge(x, t)
    for x in np.atleast_1d(new(5)):
        edge(b, x)
    mark["tie"] = (s, t)
    s, b, a, t = new(), new(), new(), new()  # (a, the long row, has the larger id)
    for x in (a, b):
        edge(s, x)
        edge(x, t)
    for x in np.atleast_1d(new(40)):
        edge(away, x)
        edge(x, a)
    mark["tie_mix"] = (s, t)
    for c in (1, 2, 5):
        cyc = np.atleast_1d(new(c))
        for i in range(c):
            edge(cyc[i], cyc[(i + 1) % c])
        tail = np.atleast_1d(new(7))
        edge(cyc[0], tail[0])
        for i in range(6):
            edge(tail[i], tail[i + 1])
        edge(tail[6], tail[6])
        mark[f"cyc_{c}"] = (int(cyc[0]), int(tail[6]))
    return DShape(nxt[0], np.array(src, np.int64), np.array(dst, np.int64), _edge_ids(len(src), 321), mark)


SHAPES = {"base": base_shape, "chain": chain_shape, "walk": walk_shape}
_shapes = {}


def dshape(name):
    if name not in _shapes:
        _shapes[name] = SHAPES[name]()
    return _shapes[name]


def shape_graph(name):
    sh = dshape(name)
    return graph(sh.n, sh.src, sh.dst, sh.eid)


# ---- the catalogue -----------------------------------------------------------------------------------------------------
@dataclass
class Case:
    shape: str
    ps: np.ndarray
    pd: np.ndarray
    sv: object = None
    path: bool = False          # also asked as shortestpath
    opts: tuple = ("default", "no_dedup", "no_prune", "reference_batching")
    widths: tuple = (0, 64, 512)
    shards: tuple = ()          # shard counts the shard test deals it over
    want: set = field(default_factory=set)
    sms: int = 0


def _other(g, pd, ps):
    """pd with every accidental src == dst moved to the next vertex with in-edges."""
    alt = g.has_in[(np.searchsorted(g.has_in, pd) + 1) % len(g.has_in)]
    return np.where(pd == ps, alt, pd)


def rows_over(g, rng, p, n_src, first_at=(), second=()):
    """p searching rows over a pool of n_src sources (the first n_src rows introduce them where p allows), random
    destinations; every row of first_at starts a source of its own; second = ((a, b), ...): row b repeats row a's
    source."""
    cand = rng.permutation(g.has_out[g.ind[g.has_out] > 0])
    pool, special = cand[:n_src], cand[n_src:n_src + len(first_at)]
    ps = rng.choice(pool, p)
    k = min(p, n_src)
    ps[:k] = pool[:k]
    for r, s in zip(first_at, special):
        ps[r] = s
    for a, b in second:
        ps[b] = ps[a]
    pd = _other(g, rng.choice(g.has_in, p), ps)
    return ps, pd, np.ones(p, np.uint8)


def sprinkle(g, rng, ps, pd, sv, keep=(), every=9):
    """Turns every `every`-th row (but the rows of keep) into, in turn: a NULL row, src == dst, a source without
    out-edges, a destination without in-edges, both, and src == dst on a vertex without edges."""
    ps, pd, sv = ps.copy(), pd.copy(), sv.copy()
    sinks = np.flatnonzero((g.od == 0) & (g.ind > 0))
    tops = np.flatnonzero((g.od > 0) & (g.ind == 0))
    iso = np.flatnonzero((g.od == 0) & (g.ind == 0))
    keep = set(int(x) for x in keep)
    turn = 0
    for r in range(every // 2, len(ps), every):
        if r in keep:
            continue
        kind = turn % 6
        turn += 1
        if kind == 0:
            sv[r] = 0
        elif kind == 1:
            pd[r] = ps[r]
        elif kind == 2:
            ps[r] = rng.choice(sinks)
        elif kind == 3:
            pd[r] = rng.choice(tops)
        elif kind == 4:
            ps[r], pd[r] = rng.choice(sinks), rng.choice(tops)
        else:
            ps[r] = pd[r] = rng.choice(iso)
    return ps, pd, sv


def lanes_case(g, rng, total):
    """`total` distinct sources in lane order, one to three rows each (repeats come later, shuffled)."""
    ps, pd, sv = rows_over(g, rng, total, total)
    extra = rng.choice(ps, min(total, 300))
    ps = np.concatenate([ps, extra])
    pd = _other(g, np.concatenate([pd, rng.choice(g.has_in, len(extra))]), ps)
    return ps, pd, np.ones(len(ps), np.uint8)


def hash_rows(g, rng, wrap):
    """40 rows whose sources share home slots of the 128-slot table: four sources per slot on three slots, or, with
    wrap, on the last slot, so that the probe chain runs over the end of the table."""
    hs = hash_size(40)
    cand = g.has_out[g.ind[g.has_out] > 0]
    home = hash_u32(g.perm[cand]) & (hs - 1)
    slots = [hs - 1, hs - 2, 0] if wrap else [int(x) for x in np.flatnonzero(np.bincount(home, minlength=hs) >= 4)[:3]]
    srcs = np.concatenate([cand[home == s][:4] for s in slots])
    ps = np.concatenate([srcs, rng.choice(srcs, 40 - len(srcs))])
    pd = _other(g, rng.choice(g.has_in, 40), ps)
    return ps, pd, np.ones(40, np.uint8)


def build_case(name, sms):
    rng = np.random.default_rng(sum(map(ord, name)))
    g = shape_graph("base")
    if name.startswith("p_"):
        p = int(name[2:])
        first = [r for r in (31, 32, 1023, 1024) if r < p - 1] + ([p - 1] if p > 1 else [])
        second = ((5, 1030),) if p > 2049 - 1 else ()
        ps, pd, sv = rows_over(g, rng, p, min(p, 20), first, second)
        ps, pd, sv = sprinkle(g, rng, ps, pd, sv, set(first) | {0, 5, 1030})
        want = {f"p_{p}"} | {f"first_appearance_row_{r}" for r in first[:-1]} | \
            ({"first_appearance_last_row"} if p > 1 else set())
        if p >= 1023:
            want |= {f"offsets_p_{p}", "classes_mixed_across_tiles"} if p >= 2047 else {f"offsets_p_{p}"}
        if second:
            want.add("second_appearance_a_tile_before_another_first")
        return Case("base", ps, pd, sv, path=True, want=want)
    if name in ("grid_pass_1", "grid_pass_2"):
        k = 1 if name.endswith("1") else 2
        p = k * sms * TILE + (1 if k == 1 else 5)
        first = [sms * TILE - 1, sms * TILE, p - 1]
        ps, pd, sv = rows_over(g, rng, p, 300, first)
        ps, pd, sv = sprinkle(g, rng, ps, pd, sv, first, every=97)
        want = {"p_beyond_one_grid_pass", "first_appearance_beyond_grid_pass", "first_appearance_last_row"}
        if k == 2:
            want.add("p_beyond_two_grid_passes")
        return Case("base", ps, pd, sv, opts=("default", "no_prune"), widths=(0, 64), want=want, sms=sms)
    if name == "one_source":
        s = g.has_out[0]
        pd = rng.choice(g.has_in[g.has_in != s], 3000)
        return Case("base", np.full(3000, s), pd, None, path=True, opts=("default", "no_prune"), widths=(0, 64),
                    want={"one_source_all_rows", "rows_per_lane_beyond_walk_grid"})
    if name in ("distinct_2048", "distinct_2049"):
        p = int(name[-4:])
        ps, pd, sv = rows_over(g, rng, p, p)
        return Case("base", ps, pd, sv, opts=("default", "reference_batching"), widths=(0, 512),
                    want={"all_distinct_p_pow2" if p == 2048 else "all_distinct_p_pow2_plus_1"})
    if name in ("hash_cluster", "hash_wrap"):
        ps, pd, sv = hash_rows(g, rng, name == "hash_wrap")
        return Case("base", ps, pd, sv, path=True, opts=("default", "no_prune"),
                    want={"hash_shared_home_slot"} | ({"hash_probe_wraps"} if name == "hash_wrap" else set()))
    if name == "class_mix":
        ps, pd, sv = rows_over(g, rng, 1100, 40)
        ps, pd, sv = sprinkle(g, rng, ps, pd, sv, every=3)
        return Case("base", ps, pd, sv, path=True, shards=(2, 3, 8, 64),
                    want={"null_row", "trivial_row", "pruned_src_without_out", "pruned_dst_without_in", "pruned_both",
                          "trivial_on_edgeless_vertex", "classes_mixed_in_one_warp", "classes_mixed_across_tiles",
                          "shard_count_2", "shard_count_3", "shard_count_8", "shard_count_beyond_total",
                          "shards_with_pruned_and_trivial"})
    if name == "no_search":
        ps, pd, sv = rows_over(g, rng, 70, 10)
        sv[::2] = 0
        pd[1::2] = ps[1::2]
        ps[5] = pd[5] = dshape("base").mark["iso"][0]
        return Case("base", ps, pd, sv, path=True, want={"no_row_searches", "no_row_searches_trailing_batch",
                                                        "trivial_on_edgeless_vertex"})
    if name.startswith("lanes_"):
        total = int(name[6:])
        ps, pd, sv = lanes_case(g, rng, total)
        want = {f"lane_total_{total}"} if total in LANE_TOTALS else set()
        want |= {513: {"narrowed_last_64", "batches_even"}, 712: {"narrowed_last_256", "batches_even"},
                 1100: {"narrowed_last_128", "batches_odd"}, 1025: {"narrowed_last_64", "batches_odd"}}.get(total, set())
        return Case("base", ps, pd, sv, path=total in (65, 129, 513), opts=("default", "reference_batching"), want=want)
    if name == "path_lengths":
        c = dshape("chain").mark["chain"]
        pairs = [(c[0], c[0]), (c[0], c[1]), (c[0], c[2]), (c[0], c[120]), (c[5], c[0]), (c[5], c[9]), (c[7], c[7]),
                 (c[30], c[10]), (c[30], c[35])]
        ps, pd = np.array(pairs, np.int64).T
        return Case("chain", ps, pd, None, path=True,
                    want={"path_len_1", "path_len_3", "path_len_5", "path_len_ge_200",
                          "lane_with_unreachable_and_reachable"})
    if name.startswith("walk_"):
        c = dshape("chain").mark["chain"]
        i = np.arange(64)
        short = (c[190 + i], c[192 + i])
        long_ = (c[i], c[i + 150])
        longer = (c[64 + i[:10]], np.full(10, c[259]))
        parts = {"walk_grow2": [short, long_], "walk_grow3": [short, long_, longer], "walk_shrink": [long_, short]}[name]
        ps, pd = (np.concatenate([x[k] for x in parts]) for k in (0, 1))
        want = {"walk_grow2": "walk_buffer_grows_2_batches", "walk_grow3": "walk_buffer_grows_3_batches",
                "walk_shrink": "walk_buffer_long_paths_first"}[name]
        return Case("chain", ps, pd, None, path=True, opts=("default", "reference_batching"), widths=(64,), want={want})
    if name == "scans":
        m = dshape("walk").mark
        keys = [f"in_{k}" for k in IN_DEGREES] + [f"out_{k}" for k in OUT_DEGREES] + ["tie", "tie_mix"]
        ps, pd = np.array([m[k] for k in keys], np.int64).T
        want = {f"walk_indeg_{k}" for k in IN_DEGREES} | {f"walk_outdeg_{k}" for k in OUT_DEGREES} | {
            "match_first_position", "match_last_position", "match_several_positions", "edge_at_position_0",
            "edge_at_last_position", "edge_duplicated_first_wins", "tie_original_and_internal_order_disagree",
            "tie_long_and_short_row_parents", "edge_ids_non_contiguous"}
        return Case("walk", ps, pd, None, path=True, want=want)
    if name == "cycles":
        m = dshape("walk").mark
        ps, pd = np.array([m[f"cyc_{c}"] for c in (1, 2, 5)], np.int64).T
        return Case("walk", ps, pd, None, path=True,
                    want={"source_on_cycle_1", "source_on_cycle_2", "source_on_cycle_5", "dst_self_loop"})
    if name == "many_paths":
        ring = dshape("base").mark["ring"]
        live = rows_over(g, rng, 300, 300)[0]
        live = live[~np.isin(live, ring)][:128]
        srcs = np.concatenate([live[:64], ring[:64], live[64:]])  # lanes 64 .. 127 never leave the ring
        ps = np.concatenate([srcs, rng.choice(live[:50], 5200)])
        pd = _other(g, rng.choice(g.has_in[~np.isin(g.has_in, ring)], len(ps)), ps)
        return Case("base", ps, pd, None, path=True, opts=("default",), widths=(0, 64),
                    want={"rows_with_paths_beyond_place_grid", "lane_group_without_paths_between"})
    raise KeyError(name)


CASES = ([f"p_{p}" for p in P_SIZES] + ["grid_pass_1", "grid_pass_2", "one_source", "distinct_2048", "distinct_2049",
                                        "hash_cluster", "hash_wrap", "class_mix", "no_search"] +
         [f"lanes_{t}" for t in LANE_TOTALS + [712]] +
         ["path_lengths", "walk_grow2", "walk_grow3", "walk_shrink", "scans", "cycles", "many_paths"])
PATH_CASES = [n for n in CASES if n.startswith(("p_", "walk_", "hash_")) or n in (
    "one_source", "class_mix", "no_search", "lanes_65", "lanes_129", "lanes_513", "path_lengths", "scans", "cycles",
    "many_paths")]
RANGE_ROWS = {"range_src_low": (-1, None), "range_src_high": ("n", None), "range_dst_low": (None, -1),
              "range_dst_high": (None, "n")}
_cases = {}


def case(name, sms=H100_SMS):
    key = (name, sms if name.startswith("grid_pass") else 0)
    if key not in _cases:
        _cases[key] = build_case(name, sms)
    return _cases[key]


def restated(c, lanes=0, flags=0, path=False, shard_index=0, shard_count=1, edge_id=None):
    sh = dshape(c.shape)
    eid = sh.eid if edge_id is None else edge_id
    return _oracle("driver_run", lambda: driver_run(sh.n, sh.src, sh.dst, c.ps, c.pd, c.sv, lanes, flags, shard_index,
                                                    shard_count, path, eid),
                   sh.n, sh.src, sh.dst, eid, c.ps, c.pd, c.sv, lanes, flags, shard_index, shard_count, path)


def configs(c, path):
    """(option set name, flags, lane width) of every run of case c."""
    return [(o, OPTION_SETS[o], w) for o in c.opts for w in c.widths]


def range_call(c, which):
    """Case c's rows with one id outside [0, n) in the middle of them."""
    s, d = RANGE_ROWS[which]
    n = dshape(c.shape).n
    ps, pd = c.ps.copy(), c.pd.copy()
    sv = None if c.sv is None else c.sv.copy()
    r = len(ps) // 2
    if sv is not None:
        sv[r] = 1
    if s is not None:
        ps[r] = n if s == "n" else s
    if d is not None:
        pd[r] = n if d == "n" else d
    return ps, pd, sv


def case_hits(name, c):
    """Every boundary of the call driver that case c hits, by name."""
    g = shape_graph(c.shape)
    sms = c.sms or H100_SMS
    p = len(c.ps)
    res = restated(c)
    cls, leaders = res["cls"], res["leaders"]
    out = set()
    if p in P_SIZES:
        out.add(f"p_{p}")
    if p > sms * TILE:
        out.add("p_beyond_one_grid_pass")
    if p > 2 * sms * TILE:
        out.add("p_beyond_two_grid_passes")
    lead = set(leaders.tolist())
    for r in (31, 32, 1023, 1024):
        if r in lead and r < p - 1:
            out.add(f"first_appearance_row_{r}")
    if p > 1 and p - 1 in lead:
        out.add("first_appearance_last_row")
    if len(leaders) and leaders.max() >= sms * TILE:
        out.add("first_appearance_beyond_grid_pass")
    follower = np.flatnonzero((cls == SEARCH) & ~np.isin(np.arange(p), leaders))
    if len(follower) and len(leaders) and (leaders.max() >> 10) > (follower.min() >> 10):
        out.add("second_appearance_a_tile_before_another_first")
    if res["searches"] == 1 and res["search_rows"] == p and p >= TILE:
        out.add("one_source_all_rows")
    if res["searches"] == p and p >= 64:
        if p & (p - 1) == 0:
            out.add("all_distinct_p_pow2")
            assert hash_size(p) == 2 * p
        if (p - 1) & (p - 2) == 0:
            out.add("all_distinct_p_pow2_plus_1")
    if res["searches"]:
        hs = hash_size(p)
        home = hash_u32(g.perm[res["lane_src"]]) & (hs - 1)
        if np.bincount(home).max() >= 3:
            out.add("hash_shared_home_slot")
        if np.count_nonzero(home == hs - 1) >= 2:
            out.add("hash_probe_wraps")
    ok = np.ones(p, bool) if c.sv is None else c.sv != 0
    no_out, no_in = g.od[np.clip(c.ps, 0, g.n - 1)] == 0, g.ind[np.clip(c.pd, 0, g.n - 1)] == 0
    pr = cls == PRUNED
    for nm, m in (("null_row", ~ok), ("trivial_row", cls == TRIVIAL), ("pruned_src_without_out", pr & no_out & ~no_in),
                  ("pruned_dst_without_in", pr & no_in & ~no_out), ("pruned_both", pr & no_in & no_out),
                  ("trivial_on_edgeless_vertex", (cls == TRIVIAL) & no_out & no_in)):
        if m.any():
            out.add(nm)
    kinds = np.where(ok, cls, -1)
    per_warp = [set(kinds[i:i + 32].tolist()) for i in range(0, p, 32)]
    if any(len(s) == 4 for s in per_warp):
        out.add("classes_mixed_in_one_warp")
    if p > TILE and all(len(set(kinds[t:t + TILE].tolist())) >= 3 for t in (0, TILE)):
        out.add("classes_mixed_across_tiles")
    if p and res["searches"] == 0:
        out.add("no_row_searches")
        r64 = restated(c, 64, REF)
        if r64["trailing"] and r64["batches"] == 1 and not restated(c, 0, REF)["batches"]:
            out.add("no_row_searches_trailing_batch")
    if res["searches"] in LANE_TOTALS:
        out.add(f"lane_total_{res['searches']}")
    plan = res["plan"]
    if len(plan) >= 2:
        if plan[-1][2] < plan[0][2]:
            out.add(f"narrowed_last_{plan[-1][2]}")
        out.add("batches_odd" if len(plan) & 1 else "batches_even")
    for k in c.shards:
        out.add("shard_count_beyond_total" if k > res["all_lanes"] else f"shard_count_{k}")
    if c.shards and pr.any() and (cls == TRIVIAL).any():
        out.add("shards_with_pruned_and_trivial")
    if not c.path:
        return out
    rp = restated(c, 0, 0, True)
    paths = rp["paths"]
    lens = np.array([0 if x is None else len(x) for x in paths])
    for k in (1, 3, 5):
        if np.any(lens == k):
            out.add(f"path_len_{k}")
    if np.any(lens >= 200):
        out.add("path_len_ge_200")
    walked = lens > 1
    lane = rp["lane"]
    on_lane = lane >= 0
    if on_lane.any():
        dead = np.bincount(lane[on_lane & (lens == 0)], minlength=rp["searches"])
        alive = np.bincount(lane[on_lane & walked], minlength=rp["searches"])
        if np.any((dead > 0) & (alive > 0)):
            out.add("lane_with_unreachable_and_reachable")
        if alive.max() > sms * WALK_BLOCKS_PER_SM:
            out.add("rows_per_lane_beyond_walk_grid")
        grp = np.add.reduceat(alive, np.arange(0, len(alive), 64)) if len(alive) else np.zeros(0)
        if len(grp) >= 3 and np.any((grp[1:-1] == 0) & (np.maximum.accumulate(grp)[:-2] > 0) &
                                    (np.maximum.accumulate(grp[::-1])[::-1][2:] > 0)):
            out.add("lane_group_without_paths_between")
    if walked.sum() > PLACE_BLOCKS:
        out.add("rows_with_paths_beyond_place_grid")
    if p in (1023, 1024, 1025, 2047, 2048, 2049) and len(set(lens.tolist())) >= 3:
        out.add(f"offsets_p_{p}")
    if not np.array_equal(g.ids, np.arange(len(g.ids))) and walked.any():
        out.add("edge_ids_non_contiguous")
    for r, steps in rp["steps"].items():
        s, d = int(c.ps[r]), int(c.pd[r])
        if steps and d in g.outs(d):
            out.add("dst_self_loop")
        back = g.ins(s)
        if steps and len(back):
            cyc = int(g.dist(s)[back][g.dist(s)[back] >= 0].min()) + 1 if np.any(g.dist(s)[back] >= 0) else 0
            if cyc in (1, 2, 5) and len(steps) > cyc:
                out.add(f"source_on_cycle_{cyc}")
        for st in steps:
            if st["indeg"] in IN_DEGREES:
                out.add(f"walk_indeg_{st['indeg']}")
            if st["outdeg"] in OUT_DEGREES:
                out.add(f"walk_outdeg_{st['outdeg']}")
            if st["indeg"] >= WALK_THREADS - 1:
                if len(st["match"]) == 1 and st["match"][0] == 0:
                    out.add("match_first_position")
                if len(st["match"]) == 1 and st["match"][0] == st["indeg"] - 1:
                    out.add("match_last_position")
                if len(st["match"]) >= 3 and st["match"].max() - st["match"].min() >= WALK_THREADS:
                    out.add("match_several_positions")
            if st["outdeg"] >= WALK_THREADS:
                if st["dup"] == 1 and st["edge_pos"] == 0:
                    out.add("edge_at_position_0")
                if st["dup"] == 1 and st["edge_pos"] == st["outdeg"] - 1:
                    out.add("edge_at_last_position")
                if st["dup"] >= 3:
                    out.add("edge_duplicated_first_wins")
            if len(st["cand"]) >= 2:
                if g.perm[st["cand"]].argmin() != 0:  # (cand is sorted: the reference takes cand[0])
                    out.add("tie_original_and_internal_order_disagree")
                if len(set((g.ind[st["cand"]] >= SHORT_DEG).tolist())) == 2:
                    out.add("tie_long_and_short_row_parents")
    r64 = restated(c, 64, 0, True)
    per_batch = [max([lens[r] for r in run["rows"]] + [0]) for run in r64["runs"]]
    if len(per_batch) in (2, 3) and per_batch[-1] >= 4 * per_batch[0] and min(per_batch) > 1:
        out.add(f"walk_buffer_grows_{len(per_batch)}_batches")
    if len(per_batch) >= 2 and per_batch[0] >= 4 * per_batch[-1] and min(per_batch) > 1:
        out.add("walk_buffer_long_paths_first")
    return out


REQUIRED = (
    {f"p_{p}" for p in P_SIZES}
    | {"p_beyond_one_grid_pass", "p_beyond_two_grid_passes", "first_appearance_beyond_grid_pass"}
    | {f"first_appearance_row_{r}" for r in (31, 32, 1023, 1024)}
    | {"first_appearance_last_row", "second_appearance_a_tile_before_another_first", "one_source_all_rows",
       "all_distinct_p_pow2", "all_distinct_p_pow2_plus_1", "hash_shared_home_slot", "hash_probe_wraps", "null_row",
       "trivial_row", "pruned_src_without_out", "pruned_dst_without_in", "pruned_both", "trivial_on_edgeless_vertex",
       "classes_mixed_in_one_warp", "classes_mixed_across_tiles", "no_row_searches", "no_row_searches_trailing_batch"}
    | set(RANGE_ROWS)
    | {f"lane_total_{t}" for t in LANE_TOTALS}
    | {"narrowed_last_64", "narrowed_last_128", "narrowed_last_256", "batches_odd", "batches_even"}
    | {"shard_count_2", "shard_count_3", "shard_count_8", "shard_count_beyond_total", "shards_with_pruned_and_trivial"}
    | {"path_len_1", "path_len_3", "path_len_5", "path_len_ge_200", "lane_with_unreachable_and_reachable"}
    | {f"walk_indeg_{k}" for k in IN_DEGREES} | {f"walk_outdeg_{k}" for k in OUT_DEGREES}
    | {"match_first_position", "match_last_position", "match_several_positions", "edge_at_position_0",
       "edge_at_last_position", "edge_duplicated_first_wins", "edge_ids_non_contiguous",
       "tie_original_and_internal_order_disagree", "tie_long_and_short_row_parents", "source_on_cycle_1",
       "source_on_cycle_2", "source_on_cycle_5", "dst_self_loop", "rows_per_lane_beyond_walk_grid",
       "rows_with_paths_beyond_place_grid", "lane_group_without_paths_between", "walk_buffer_grows_2_batches",
       "walk_buffer_grows_3_batches", "walk_buffer_long_paths_first"}
    | {f"offsets_p_{p}" for p in (1023, 1024, 1025, 2047, 2048, 2049)}
)


# ---- CPU: the restatement equals the oracle; the catalogue hits what it names ---------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_restatement_equals_the_oracle(name):
    """Lengths: orc.iterativelength (the reference's batches) and orc.iterativelength_ex (shortcut and dedup) at the
    explicit widths, for answers, lanes used and the counters; for lanes = 0 the answers, which no plan changes, and
    scipy's hop counts.  Paths: orc.shortestpath for every list, and its counters under the reference's batches."""
    c = case(name)
    g = shape_graph(c.shape)
    n = g.n
    for oname, flags, w in configs(c, False):
        res = restated(c, w, flags)
        assert len(res["trace"]) == res["levels"] and all(r["stop"] for r in res["runs"])
        width = w or 512
        if flags & REF:
            o, ov, st = _oracle("il", lambda: orc.iterativelength(n, g.v, g.e, c.ps, c.pd, c.sv, width), g.v, g.e,
                                c.ps, c.pd, c.sv, width)
            used = int(np.count_nonzero(res["cls"] == SEARCH))
        else:
            o, ov, st, used = _oracle("ilx", lambda: orc.iterativelength_ex(
                n, g.v, g.e, c.ps, c.pd, c.sv, width, prune=not flags & NO_PRUNE, dedup=not flags & NO_DEDUP),
                g.v, g.e, c.ps, c.pd, c.sv, width, flags)
        assert np.array_equal(res["valid"], ov) and np.array_equal(res["out"], o), (oname, w)
        assert res["searches"] == used, (oname, w)
        if w:
            assert (res["batches"], res["levels"], res["edges"], res["fv"]) == (
                st.batches, st.levels, st.edges_traversed, st.frontier_vertices), (oname, w)
    res = restated(c)
    for r in np.flatnonzero(res["cls"] == SEARCH)[:200]:
        d = g.dist(int(c.ps[r]))[c.pd[r]]
        assert (res["out"][r], res["valid"][r]) == ((d, 1) if d > 0 else (-1, 0))
    if c.path:
        opaths, ost = _oracle("sp", lambda: orc.shortestpath(n, g.v, g.e, g.ids, c.ps, c.pd, c.sv, 64), g.v, g.e, g.ids,
                              c.ps, c.pd, c.sv, 64)
        for oname, flags, w in configs(c, True):
            res = restated(c, w, flags, True)
            assert res["paths"] == opaths, (oname, w)
            if flags & REF and w == 64:
                assert (res["batches"], res["levels"], res["edges"], res["fv"]) == (
                    ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices), (oname, w)
    for k in c.shards:
        whole = restated(c)
        for si in range(k):
            part = restated(c, 0, 0, False, si, k)
            own = part["lane"] >= 0
            assert np.array_equal(own, (whole["ordinal"] >= 0) & (whole["ordinal"] % k == si))
            free = whole["cls"] != SEARCH
            assert np.array_equal(part["out"][own | free], whole["out"][own | free])
            assert not part["valid"][~own & ~free].any()


@pytest.mark.parametrize("name", CASES)
def test_call_driver_catalogue_hits_its_boundaries(name):
    c = case(name)
    got = case_hits(name, c)
    print(f"{name}: p={len(c.ps)} hits {sorted(got)}")
    assert c.want <= got, sorted(c.want - got)


@pytest.mark.parametrize("which", list(RANGE_ROWS))
def test_restatement_refuses_an_id_out_of_range(which):
    c = case("class_mix")
    sh = dshape(c.shape)
    ps, pd, sv = range_call(c, which)
    for path in (False, True):
        with pytest.raises(RangeError):
            driver_run(sh.n, sh.src, sh.dst, ps, pd, sv, path=path, edge_id=sh.eid)


def test_call_driver_catalogue_covers_every_boundary():
    named = set().union(*(case(n).want for n in CASES)) | set(RANGE_ROWS)
    assert REQUIRED <= named, sorted(REQUIRED - named)


def test_pick_lanes_budgets():
    """The 32 MiB rule of the mask arrays and the 4 GiB level array of path mode."""
    assert pick_lanes(0, 1 << 19, 1000, False) == 512 and pick_lanes(0, (1 << 19) + 1, 1000, False) == 256
    assert pick_lanes(0, 1 << 19, 1000, True) == 512 and pick_lanes(0, (1 << 19) + 1, 1000, True) == 256
    assert pick_lanes(0, 1 << 23, 1000, True) == 256 and pick_lanes(0, (1 << 23) + 1, 1000, True) == 128
    assert pick_lanes(0, 1 << 24, 1000, True) == 128 and pick_lanes(0, (1 << 24) + 1, 1000, True) == 64
    assert [pick_lanes(0, 100, s, False) for s in (1, 64, 65, 128, 129, 256, 257)] == [64, 64, 128, 128, 256, 256, 512]
    assert pick_lanes(128, 1 << 26, 1, True) == 128


# ---- GPU -----------------------------------------------------------------------------------------------------------------
LEVEL = re.compile(r"\[pgq\] batch (\d+) level (\d+) (?:push|pull|tail) frontier_v=(\d+) frontier_e=(\d+) ")
CALL = re.compile(r"\[pgq\] call .* lanes=(\d+) searches=(\d+) rows=(\d+) pruned=(\d+)")
COUNTERS = ("searches", "pruned", "search_rows", "lanes", "batches", "levels", "edges_traversed", "frontier_vertices")


def counters(res):
    return (res["searches"], res["pruned"], res["search_rows"], res["lanes"], res["batches"], res["levels"],
            res["edges"], res["fv"])


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def sms():
    return device_sms()


def build_csr(ctx, shape_name):
    sh = dshape(shape_name)
    return pgq.DeviceCSR.build(ctx, sh.n, sh.src, sh.dst, sh.eid)


def check_trace(err, res):
    """One stream: every level line in the restatement's order with its batch, level, frontier vertices and
    out-edges, and the closing call line with lanes / searches / rows / pruned."""
    got = [tuple(int(x) for x in m) for m in LEVEL.findall(err)]
    want = [(r["batch"] + 1, r["level"], r["fv"], r["fe"]) for r in res["trace"]]
    assert got == want, next((i, a, b) for i, (a, b) in enumerate(zip(got + [None], want + [None])) if a != b)
    call = CALL.findall(err)
    assert len(call) == 1 and tuple(int(x) for x in call[0]) == (res["lanes"], res["searches"], res["search_rows"],
                                                               res["pruned"])


def run_case(csr, c, capfd=None, edge_id=None, which=None):
    """Case c on the device under every configuration: answers (paths as whole lists), the eight counters and, with
    capfd, the trace."""
    for path in ((False, True) if c.path else (False,)):
        for oname, flags, w in configs(c, path):
            if which is not None and (oname, w) not in which:
                continue
            res = restated(c, w, flags, path, edge_id=edge_id)
            if capfd:
                capfd.readouterr()
            if path:
                paths, st = csr.shortestpath(c.ps, c.pd, c.sv, options(w, flags))
                assert paths == res["paths"], (oname, w, next(i for i, (a, b) in enumerate(zip(paths, res["paths"]))
                                                              if a != b))
            else:
                out, valid, st = csr.iterativelength(c.ps, c.pd, c.sv, options(w, flags))
                assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"]), (oname, w)
            assert tuple(st[k] for k in COUNTERS) == counters(res), (oname, w, path)
            if capfd:
                check_trace(capfd.readouterr().err, res)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_case_on_the_device(gpu_ctx, monkeypatch, capfd, sms, name):
    """Every case under its option sets and lane widths, for iterativelength and (where it has paths) shortestpath:
    answers, counters and, batch by batch and level by level, the frontier of the restatement's lane order."""
    c = case(name, sms)
    if c.sms:
        assert len(c.ps) > sms * TILE
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", "1")
    csr = build_csr(gpu_ctx, c.shape)
    try:
        run_case(csr, c, capfd)
    finally:
        csr.free()


@pytest.mark.gpu
def test_two_streams_give_the_same_totals(gpu_ctx):
    """The default deal of the batches over two streams and workspaces: odd and even batch counts."""
    csr = build_csr(gpu_ctx, "base")
    try:
        for name in ("lanes_513", "lanes_1025", "lanes_1100", "lanes_712", "class_mix", "distinct_2049"):
            run_case(csr, case(name))
    finally:
        csr.free()


TIMINGS = ("expand_ms", "total_ms", "pull_ms")


@pytest.mark.gpu
def test_two_streams_fold_every_counter(gpu_ctx, monkeypatch):
    """The second stream's counters are folded into the call's: one stream and two give the same answers and every
    stats field but the timings, launches, levels and copied bytes included."""
    csr = build_csr(gpu_ctx, "base")
    try:
        for name in ("lanes_513", "lanes_1025", "lanes_1100", "lanes_712", "class_mix", "distinct_2049"):
            c = case(name)
            for oname, flags, w in configs(c, False):
                runs = []
                for streams in ("1", "2"):
                    monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", streams)
                    runs.append(csr.iterativelength(c.ps, c.pd, c.sv, options(w, flags)))
                (out1, valid1, st1), (out2, valid2, st2) = runs
                assert np.array_equal(valid1, valid2) and np.array_equal(out1, out2), (name, oname, w)
                assert {k: v for k, v in st1.items() if k not in TIMINGS} == \
                       {k: v for k, v in st2.items() if k not in TIMINGS}, (name, oname, w)
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ["iterativelength", "shortestpath"])
@pytest.mark.parametrize("flags", [0, NO_DEDUP])
def test_shards(gpu_ctx, fn, flags):
    """Every shard answers exactly the rows whose lane ordinal is congruent to its index, plus the rows that need no
    search; all other rows are (-1, NULL) or NULL lists; searches per shard are the restatement's; the union of the
    shards is the unsharded answer."""
    c = case("class_mix")
    path = fn == "shortestpath"
    csr = build_csr(gpu_ctx, c.shape)
    try:
        whole = restated(c, 0, flags, path)
        free = whole["cls"] != SEARCH
        for k in c.shards:
            union_valid = np.zeros(len(c.ps), bool)
            union = [None] * len(c.ps)
            for si in range(k):
                res = restated(c, 0, flags, path, si, k)
                own = res["lane"] >= 0
                assert np.array_equal(own, (whole["ordinal"] >= 0) & (whole["ordinal"] % k == si))
                if path:
                    got, st = csr.shortestpath(c.ps, c.pd, c.sv, options(0, flags, si, k))
                    assert got == res["paths"], (k, si)
                    assert all(x is None for x, o, f in zip(got, own, free) if not o and not f)
                    valid = np.array([x is not None for x in got])
                else:
                    out, valid, st = csr.iterativelength(c.ps, c.pd, c.sv, options(0, flags, si, k))
                    assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"]), (k, si)
                    assert not valid[~own & ~free].any() and np.all(out[~own & ~free] == -1)
                    got = out.tolist()
                    valid = valid != 0
                assert tuple(st[x] for x in COUNTERS) == counters(res), (k, si)
                for r in np.flatnonzero(valid):
                    assert not union_valid[r] or union[r] == got[r]
                    union[r] = got[r]
                union_valid |= valid
            if path:
                assert union == whole["paths"]
            else:
                assert np.array_equal(union_valid, whole["valid"] != 0)
                assert [union[r] for r in np.flatnonzero(union_valid)] == whole["out"][union_valid].tolist()
    finally:
        csr.free()


@pytest.mark.gpu
def test_range_error_is_a_status_and_the_workspace_stays_good(monkeypatch):
    """An id outside [0, n) next to valid rows, in all four positions: PGQ_ERR_RANGE from both functions, and the next
    call on the same workspace is right."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    c = case("class_mix")
    try:
        csr = build_csr(ctx, c.shape)
        for which in RANGE_ROWS:
            ps, pd, sv = range_call(c, which)
            for call in (csr.iterativelength, csr.shortestpath):
                with pytest.raises(pgq.InvalidInputException) as ei:
                    call(ps, pd, sv)
                assert ei.value.status == pgq.PGQ_ERR_RANGE
                run_case(csr, c, which={("default", 0)})
        csr.free()
    finally:
        ctx.close()


def raw_shortestpath(csr, ps, pd, sv, opts):
    lib = _native.load()
    p = len(ps)
    ps, pd = np.ascontiguousarray(ps, dtype=np.int64), np.ascontiguousarray(pd, dtype=np.int64)
    sv = None if sv is None else np.ascontiguousarray(sv, dtype=np.uint8)
    offs, lens = np.full(p, -7, np.int64), np.full(p, -7, np.int64)
    ov = np.full(p, 9, np.uint8)
    elems = C.POINTER(C.c_int64)()
    total = C.c_int64(-1)
    o = opts.c()
    p64, pu8 = C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    rc = lib.pgq_shortestpath(csr._h, p, ps.ctypes.data_as(p64), pd.ctypes.data_as(p64),
                              None if sv is None else sv.ctypes.data_as(pu8), C.byref(o), offs.ctypes.data_as(p64),
                              lens.ctypes.data_as(p64), ov.ctypes.data_as(pu8), C.byref(elems), C.byref(total), None)
    assert rc == pgq.PGQ_OK
    flat = np.ctypeslib.as_array(elems, shape=(total.value,)).copy() if total.value else np.zeros(0, np.int64)
    lib.pgq_free(elems)
    return offs, lens, ov, flat, total.value


@pytest.mark.gpu
def test_list_offsets_through_the_raw_abi(gpu_ctx):
    """out_offsets is the exclusive prefix sum of out_lengths in row order across the 1024-row tiles, out_total their
    sum, NULL rows have length 0, and a call whose rows are all NULL returns total 0 and a pointer pgq_free takes."""
    csr = build_csr(gpu_ctx, "base")
    try:
        for name in ("p_1023", "p_1024", "p_1025", "p_2047", "p_2048", "p_2049", "many_paths"):
            c = case(name)
            for w, flags in ((0, 0), (64, REF)):
                res = restated(c, w, flags, True)
                offs, lens, ov, flat, total = raw_shortestpath(csr, c.ps, c.pd, c.sv, options(w, flags))
                want = np.array([0 if x is None else len(x) for x in res["paths"]], np.int64)
                assert np.array_equal(lens, want) and np.array_equal(ov, (want > 0).astype(np.uint8))
                assert np.array_equal(offs, np.concatenate([[0], np.cumsum(want)[:-1]])) and total == want.sum()
                assert flat.tolist() == [x for pth in res["paths"] if pth for x in pth]
        c = case("p_2049")
        offs, lens, ov, flat, total = raw_shortestpath(csr, c.ps, c.pd, np.zeros(len(c.ps), np.uint8), options())
        assert total == 0 and not lens.any() and not offs.any() and not ov.any()
    finally:
        csr.free()


ROUTE_CASES = ["p_1025", "class_mix", "lanes_513", "scans", "cycles", "walk_grow3"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["device_pairs", "chunked8", "upload_noids", "keys", "clone", "udf"])
@pytest.mark.parametrize("name", ROUTE_CASES)
def test_other_routes(gpu_ctx, name, route):
    """The same answers and counters from pairs in HBM on a caller-made stream, from a CSR fed in chunks by eight
    threads, uploaded without edge ids (the lists then carry CSR positions), built from key columns, cloned, and
    through the UDF-style calls of DuckPGQState."""
    import torch
    c = case(name)
    sh = dshape(c.shape)
    one = {("default", c.widths[0]), ("reference_batching", c.widths[-1])}
    live, ctxs = [], []
    try:
        if route == "device_pairs":
            csr = build_csr(gpu_ctx, c.shape)
            live.append(csr)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                     (c.ps, c.pd, np.ones(len(c.ps), np.uint8) if c.sv is None else c.sv)]
                out = torch.empty(len(c.ps), dtype=torch.int64, device="cuda")
                valid = torch.empty(len(c.ps), dtype=torch.uint8, device="cuda")
                for oname, w in sorted(one):
                    res = restated(c, w, OPTION_SETS[oname])
                    st = csr.iterativelength_device(d[0].data_ptr(), d[1].data_ptr(), len(c.ps), out.data_ptr(),
                                                    valid.data_ptr(), d[2].data_ptr(), stream.cuda_stream,
                                                    options(w, OPTION_SETS[oname]))
                    stream.synchronize()
                    assert np.array_equal(valid.cpu().numpy(), res["valid"])
                    assert np.array_equal(out.cpu().numpy(), res["out"])
                    assert tuple(st[k] for k in COUNTERS) == counters(res)
        elif route in ROUTES:
            csr, exp, exact = make(gpu_ctx, sh, route)
            live.append(csr)
            v, e, ids, _ = check_download(csr, sh, exp, exact)
            if exact:  # the order inside a vertex is the reference's: the lists are comparable
                eid = "position" if route == "upload_noids" else ids_of(sh, ids, v, e)
                run_case(csr, c, edge_id=eid, which=one)
            else:
                for oname, w in sorted(one):
                    res = restated(c, w, OPTION_SETS[oname])
                    out, valid, st = csr.iterativelength(c.ps, c.pd, c.sv, options(w, OPTION_SETS[oname]))
                    assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"])
                    assert tuple(st[k] for k in COUNTERS) == counters(res)
        elif route == "keys":
            keys = np.random.default_rng(31).choice(1 << 40, sh.n, replace=False).astype(np.int64) - (1 << 39)
            csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[sh.src], keys[sh.dst])
            live.append(csr)
            run_case(csr, c, edge_id=np.arange(len(sh.src), dtype=np.int64), which=one)
        elif route == "clone":
            ctx_a, ctx_b = pgq.Context(0), pgq.Context(0)
            ctxs += [ctx_a, ctx_b]
            prim = build_csr(ctx_a, c.shape)
            csr = prim.clone(ctx_b)
            live.append(csr)
            prim.free()
            run_case(csr, c, which=one)
        else:
            state = pgq.DuckPGQState(gpu_ctx)
            m = len(sh.src)
            pgq.create_csr_vertex(state, 0, sh.n, np.arange(sh.n), np.bincount(sh.src, minlength=sh.n))
            pgq.create_csr_edge(state, 0, sh.n, m, m, sh.src, sh.dst, sh.eid)
            live.append(state.csr_list[0])
            res = restated(c)
            out, valid = pgq.iterativelength(state, 0, sh.n, c.ps, c.pd, c.sv)
            assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"])
            if c.path:
                assert pgq.shortestpath(state, 0, sh.n, c.ps, c.pd, c.sv) == restated(c, 0, 0, True)["paths"]
    finally:
        for x in live:
            x.free()
        for x in ctxs:
            x.close()


def ids_of(sh, ids, v, e):
    """The edge rowids a route gave the CSR, as an edge_id column in row order (the restatement builds its CSR from the
    rows): rows and CSR positions correspond through the reference's build."""
    _, _, pos = orc.csr_build(sh.n, sh.src, sh.dst, np.arange(len(sh.src), dtype=np.int64))
    eid = np.empty(len(sh.src), np.int64)
    eid[pos] = ids
    return eid


@pytest.mark.gpu
def test_one_dirty_workspace(monkeypatch):
    """One context with one workspace: a long-path shortestpath, a wide iterativelength, a bidirectional call and a
    range error in turn, then every path case again on the buffers they left."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        csrs = {s: build_csr(ctx, s) for s in SHAPES}
        run_case(csrs["chain"], case("walk_grow3"))
        run_case(csrs["base"], case("lanes_1100"), which={("default", 0), ("default", 64)})
        c = case("class_mix")
        csrs["base"].iterativelengthbidirectional(c.ps, c.pd, c.sv)
        with pytest.raises(pgq.InvalidInputException):
            csrs["base"].shortestpath(*range_call(c, "range_dst_high"))
        for name in PATH_CASES:
            c = case(name)
            run_case(csrs[c.shape], c, which={("default", c.widths[0]), ("reference_batching", c.widths[-1])})
        for x in csrs.values():
            x.free()
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["walk_grow2", "walk_grow3", "walk_shrink"])
def test_walk_buffer_grows_in_a_fresh_context(name):
    """A new context's workspace has no walk buffer yet, so every batch's bound reallocates it while it holds the
    earlier batches' paths (on a used workspace the buffer may already be large enough)."""
    ctx = pgq.Context(0)
    try:
        csr = build_csr(ctx, "chain")
        run_case(csr, case(name), which={("default", 64)})
        csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    """Eight threads with different cases on one CSR."""
    names = ["p_1025", "p_2049", "class_mix", "lanes_513", "lanes_257", "hash_wrap", "one_source", "no_search"]
    csr = build_csr(gpu_ctx, "base")
    try:
        for nm in names:  # (the restatements, computed before the threads start)
            c = case(nm)
            for path in ((False, True) if c.path else (False,)):
                for oname, flags, w in configs(c, path):
                    restated(c, w, flags, path)

        def body(nm):
            for _ in range(2):
                run_case(csr, case(nm))
            return nm

        with ThreadPoolExecutor(max_workers=8) as pool:
            assert sorted(pool.map(body, names)) == sorted(names)
    finally:
        csr.free()


@pytest.mark.gpu
def test_path_mode_width_budget(gpu_ctx):
    """Optional (skipped when memory is short): the per-lane level array of path mode may take 4 GiB.  A graph beyond
    2^19 vertices starts at 256 lanes (the 32 MiB rule of the masks), so with lanes = 0 one of 2^23 vertices runs 256
    lanes and one of 2^23 + 1 runs 128."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs 24 GiB of free device memory")
    for n, want in ((1 << 23, 256), ((1 << 23) + 1, 128)):
        s = np.arange(300, dtype=np.int64)
        csr = pgq.DeviceCSR.build(gpu_ctx, n, s, s + 300)
        try:
            paths, st = csr.shortestpath(s, s + 300)
            assert st["lanes"] == want and st["searches"] == 300
            assert paths == [[int(x), int(x), int(x) + 300] for x in s]
        finally:
            csr.free()
