"""cheapest_path_count and all_cheapest_paths at the boundaries of their sweep batches, their tight walk engine and
their infinite-count rule, against two restatements.

all_cheapest_paths runs the walk engine of shortest_k_paths (csrc/pgq_count.cuh) over the edges each lane's
Bellman-Ford distances make tight (csrc/pgq_cheapest.cu, TightWalks), and uses parts of it nothing else reaches: walks
placed batch after batch behind the previous batches' (walk_offsets keeps them and grows its buffers with pgq_ws_grow),
an edge filter read per lane through the storing pass's lane map (TightEdges, lane_map = glane, which skips every lane
without walks), in-lists in step order (step_par) in which the non-tight entries stay as zero terms of k_ks_omega's
128-position chunks and k_ks_unrank's 32-entry windows, and the infinite rule of k_ac_step (counts still alive at
h >= |B_tight(t)|).  So:

- a restatement in Python integers written from the definitions at the top of pgq_cheapest.cu: d(s, .) from the
  oracle's cheapest_path_length, the tight edges (test_all_cheapest_paths.tight_edges), B_tight(t), per-length counts by
  a layered DP over every in-list in full step order, the stopping rule, the listing by test_count_unrank_boundaries'
  unranker, the batch plan of run_bf (L lanes, wd mask words) and the storing groups of walk_store per batch.  It shows
  its work -- per row its kind, B(t), its stop and where it turned infinite, per walk the unranker's steps, per batch
  its lanes, its listed lanes and groups, per call the buffer sizes a fresh workspace takes -- and refuses what the
  device refuses;
- a catalogue whose cases each name the boundaries they hit, proven on the CPU from that record; a coverage test asks
  every boundary to be hit by some case;
- the C oracle (oracle/pgq_oracle_allcheapest.c) equal to the restatement on every case, and the small cases equal to
  the brute-force walks of test_all_cheapest_paths;
- on the GPU, the device equal to both on every case at max_paths 0, 1, the count and the count + 1, path 0 equal to
  cheapest_path; then under row widths and a row permutation, layer budgets that close storing groups at chosen sizes
  (checked in the launch counts), the weighted construction routes, a dirty and a fresh one-workspace context, and
  eight threads on one CSR.

The number of Bellman-Ford sweeps of a call (stats levels) depends on the order of the parallel relaxations; each sweep
is one launch, so launch counts are compared as kernel_launches - levels."""
import threading
from functools import lru_cache

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_OOM, PGQ_ERR_UNSUPPORTED
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allcheapest as oac
from test_all_cheapest_paths import INF_F64, INF_I64, brute_walks, distances, tight_cycle_on_route, tight_edges
from test_all_shortest_paths import diamonds
from test_count_unrank_boundaries import (WINDOW, Builder, Graph, Unsupported, chunk_work, layer_bytes, layout,
                                          store_groups, store_launches, unrank)
from test_count_unrank_boundaries import build as ks_build
from test_count_unrank_boundaries import compare_all as ks_compare_all

INT64_MAX = (1 << 63) - 1
WALK_MAX = 65533
KS_BUDGET = 4 << 30
WIDTHS = (1, 31, 32, 33, 64, 65, 96, 97, 160, 200, 255, 256, 257, 513)
GROUP_SIZES = (1, 31, 32, 33, 64, 65)
HUB_DEGREES = (127, 128, 129, 255, 257, 385)


# ---- the restatement ---------------------------------------------------------------------------------------------------
class WGraph(Graph):
    """Graph with a weight per edge row: the CSR's weights (orc.csr_build_weighted, whose layout equals csr_build's),
    per source the distances and the tight edges, and the device's step-ordered in-lists by in-CSC position (the
    parent's internal id and the edge's CSR index)"""

    def __init__(self, n, src, dst, w):
        super().__init__(n, src, dst)
        v, e, ids, self.w = orc.csr_build_weighted(n, self.src, self.dst, np.asarray(w))
        assert np.array_equal(v, self.v) and np.array_equal(e, self.e) and np.array_equal(ids, self.ids)
        self.is_f = self.w.dtype.kind == "f"
        self.inf = INF_F64 if self.is_f else INF_I64
        self.row = np.repeat(np.arange(n), np.diff(self.v[:n + 1]))
        inv = self.lay["inv"]
        parts = [self.st_idx[self.st_off[u]:self.st_off[u + 1]] for u in inv[:self.n_ab].tolist()]
        self.step_csr = np.concatenate(parts).astype(np.int64) if parts else np.zeros(0, np.int64)
        self.step_in = self.perm[self.row[self.step_csr]]
        self._dist, self._tight, self._inl, self._trace = {}, {}, {}, {}

    def dist(self, s):
        if s not in self._dist:
            self._dist[s] = distances(self.n, self.v, self.e, self.w, s)
        return self._dist[s]

    def tight(self, s):
        """per CSR index: whether the edge is tight under d(s, .)"""
        if s not in self._tight:
            t = np.zeros(len(self.e), bool)
            for _, _, k, _ in tight_edges(self.n, self.v, self.e, self.w, self.dist(s)):
                t[k] = True
            self._tight[s] = t
        return self._tight[s]


def lanes_for(n, p):
    """run_bf's lanes per batch: 256, halved while the distances would pass 2 GiB, at most p rounded up to 32"""
    L = 256
    while L > 32 and L * max(n, 1) * 8 > (2 << 30):
        L >>= 1
    return min(L, (p + 31) // 32 * 32)


def ac_layers(s, inl, B, upto):
    """w_1 .. w_upto of the tight walks from s on B (inl[u]: u's tight parents in step order, one entry per edge),
    saturated, without their zeros"""
    out, prev = [], {s: 1}
    for _ in range(upto):
        prev = {u: min(x, INT64_MAX) for u in B if (x := sum(prev.get(p, 0) for p in inl[u]))}
        out.append(prev)
    return out


class Trace:
    """The layers of one row's counts, from s over the tight edges on B(t), grown on demand: w_h(t) and whether w_h
    is alive.  (The counts are the same whatever the call lists; only where it stops differs.)"""

    def __init__(self, s, t, inl, B):
        self.t, self.B = t, B
        self.out = {}  # the tight edges from each vertex of B into B, one entry per edge
        for u in B:
            for p in inl[u]:
                self.out.setdefault(p, []).append(u)
        self.ct, self.alive, self.cur = [], [], {s: 1}

    def at(self, h):
        while len(self.ct) < h:
            nxt = {}
            for v, x in self.cur.items():
                for u in self.out.get(v, ()):
                    nxt[u] = nxt.get(u, 0) + x
            self.cur = {u: min(x, INT64_MAX) for u, x in nxt.items()}
            self.ct.append(self.cur.get(self.t, 0))
            self.alive.append(bool(self.cur))
        return self.ct[h - 1], self.alive[h - 1]


def ac_row(g, s, t, ok, list_, mp):
    """One row: its kind, B(t), counts per length at t, stop, count, the listed walks (lists) with the unranker's work"""
    r = dict(s=s, t=t, kind="null_id", open=False, B=set(), bsize=0, depth=-1, stop=0, count=0, inf_at=None, ct=[],
             takes=[], npaths=0, elems=0, last=-1, lists=None, work=[], lay=None)
    if not ok:
        return r
    T = g.tight(s)
    if not (s == t or g.dist(s)[t] != g.inf):
        tin = any(T[k] for k in g.st_idx[g.st_off[t]:g.st_off[t + 1]].tolist())
        r["kind"] = "sentinel_only" if tin else "unreachable"
        return r
    r["open"] = True
    if s not in g._inl:
        g._inl[s] = {u: [int(p) for p, k in zip(g.st_par[g.st_off[u]:g.st_off[u + 1]].tolist(),
                                                 g.st_idx[g.st_off[u]:g.st_off[u + 1]].tolist()) if T[k]]
                     for u in range(g.n)}
    inl = g._inl[s]
    depth, q = {t: 0}, [t]
    for u in q:
        for p in inl[u]:
            if p not in depth:
                depth[p] = depth[u] + 1
                q.append(p)
    B = set(depth)
    r.update(B=B, bsize=len(B), depth=max(depth.values()))
    if s not in B:
        r["kind"] = "not_in_b"
        return r
    r["kind"] = "counts"
    key = (s, t)
    if key not in g._trace:
        g._trace[key] = Trace(s, t, inl, B)
    trace = g._trace[key]
    total, listed, inf = (1, 1 if list_ else 0, False) if s == t else (0, 0, False)
    ct, takes = [1 if s == t else 0], [listed]
    for h in range(1, WALK_MAX + 2):
        c, alive = trace.at(h)
        ct.append(c)
        total = min(total + c, INT64_MAX)
        take = 0 if not list_ else min(c, mp - listed) if mp else c
        takes.append(take)
        listed = min(listed + take, INT64_MAX)
        if alive and h >= len(B) and not inf:
            r["inf_at"] = h
        inf = inf or (alive and h >= len(B))
        stop = not alive or total == INT64_MAX or (inf and (not list_ or mp == 0 or listed >= mp))
        if h >= WALK_MAX and not stop:
            raise Unsupported("too_long")
        if stop:
            break
    count = INT64_MAX if inf else total
    r.update(stop=h, count=count, ct=ct, takes=takes)
    if not list_ or (mp == 0 and count == INT64_MAX):
        return r  # (the call refuses a list of INT64_MAX walks)
    lens = [x for x, k in enumerate(takes) if k]
    r.update(npaths=listed, last=lens[-1] if lens else -1,
             elems=sum(min(k * (2 * x + 1), INT64_MAX) for x, k in enumerate(takes)))
    lay = [{s: 1}] + ac_layers(s, inl, B, max(r["last"], 0))
    admit = T[g.st_idx]
    r["lay"] = lay
    r["lists"] = [unrank(g, lay, s, t, x, q_, r["work"], admit) for x, k in enumerate(takes) for q_ in range(k)]
    return r


class Refused(Exception):
    def __init__(self, kind, why, batch):
        super().__init__(why)
        self.kind, self.why, self.batch = kind, why, batch


def ac_call(g, rows, ok, list_, mp, budget=KS_BUDGET):
    """One call -> dict(L, wd, rows, batches, stats, error): rows take lanes in input order, L per batch.  A refusal is
    recorded with the batch it happens in, behind the record of the batches before it.  Per batch: its lanes, the
    listed lanes and their storing groups; per call the sizes a fresh workspace gives the walk offsets and elements."""
    p = len(rows)
    L = lanes_for(g.n, p)
    out = dict(L=L, wd=(L + 63) // 64, rows=[], batches=[], error=None,
               stats=dict(batches=0, push_levels=0, pull_levels=0), fresh=[])
    walks = elems = 0
    cap = dict(walk_off=0, elems=0)
    for b0 in range(0, p, L):
        cnt = min(L, p - b0)
        bi = len(out["batches"])
        try:
            res = [ac_row(g, s, t, ok[b0 + l], list_, mp) for l, (s, t) in enumerate(rows[b0:b0 + cnt])]
        except Unsupported as ex:
            out["error"] = Refused("unsupported", str(ex), bi)
            return out
        out["rows"] += res
        st = out["stats"]
        st["batches"] += 1
        st["push_levels"] += 1 + max([r["depth"] for r in res] + [0])
        st["pull_levels"] += max([r["stop"] for r in res] + [0])
        batch = dict(b0=b0, cnt=cnt, listed=[], groups=[])
        out["batches"].append(batch)
        if not list_:
            continue
        if mp == 0 and any(r["count"] == INT64_MAX for r in res):
            out["error"] = Refused("unsupported", "saturated", bi)
            return out
        nw, ne = walks + sum(r["npaths"] for r in res), elems + sum(r["elems"] for r in res)
        if ne > INT64_MAX // 8 or nw > INT64_MAX // 8 - 1:
            out["error"] = Refused("too_large", "elements", bi)
            return out
        fresh = {}
        for slot, count, keep in (("walk_off", nw + 1, walks), ("elems", ne, elems)):
            need = max(count * 8, 256)
            if cap[slot] < need:
                grow = keep > 0
                cap[slot] = max(2 * need, 4096) if grow else need + need // 8
                fresh[slot] = "grow" if grow else "reserve"
        out["fresh"].append(fresh)
        walks, elems = nw, ne
        batch["listed"] = [(l, r["last"]) for l, r in enumerate(res) if r["npaths"] > 0]
        try:
            batch["groups"] = store_groups(batch["listed"], L, budget, g.n_ab)
        except Unsupported:
            out["error"] = Refused("unsupported", "budget", bi)
            return out
    return out


# ---- the catalogue -----------------------------------------------------------------------------------------------------
class WBuilder(Builder):
    def __init__(self, n=0):
        super().__init__(n)
        self.w = []

    def edge(self, a, b, mult=1, w=1):
        super().edge(a, b, mult)
        self.w += [w] * mult

    def chain(self, a, length, b=None, w=1):
        cur = a
        for i in range(length):
            nxt = (self.new() if b is None else b) if i == length - 1 else self.new()
            self.edge(cur, nxt, w=w)
            cur = nxt
        return cur


def lane_graph():
    """Two sources into one target over different edges (row kind 'a': s1 -> p twice, p -> t: 2 walks; kind 'b':
    s2 -> q -> t, s2 -> p costs 9: 1 walk; for a lane of one kind the other's edges are not tight), a vertex x whose
    zero-weight edge into y is tight between two sentinel distances, a chain of 8 edges for a long row, a single edge
    and a diamonds(6) whose 64 walks of 12 edges cost the same"""
    b = WBuilder()
    s1, s2, p, q, t, x, y = (b.new() for _ in range(7))
    b.edge(s1, p, 2)
    b.edge(p, t)
    b.edge(s1, q)
    b.edge(q, t, w=5)
    b.edge(s2, q)
    b.edge(s2, p, w=9)
    b.edge(x, y, w=0)
    c0 = b.new()
    c8 = b.chain(c0, 8)
    e0 = b.new()
    e1 = b.chain(e0, 1)
    dn, ds, dd = diamonds(6)
    d0 = b.new(dn)[0]
    for u, v in zip(ds.tolist(), dd.tolist()):
        b.edge(d0 + u, d0 + v)
    kinds = {"a": ((s1, t), 1), "b": ((s2, t), 1), "null_id": ((s1, t), 0), "unreachable": ((t, s1), 1),
             "sentinel_only": ((s1, y), 1), "long": ((c0, c8), 1), "edge": ((e0, e1), 1),
             "diamonds": ((d0, d0 + dn - 1), 1)}
    return b, kinds


def lane_case(pattern, **kw):
    b, kinds = lane_graph()
    rows = [kinds[k][0] for k in pattern]
    ok = [kinds[k][1] for k in pattern]
    return dict(n=b.n, src=b.src, dst=b.dst, w=b.w, rows=rows, ok=ok, **kw)


SKIPS = ("null_id", "unreachable", "sentinel_only")


def lane_kind(l):
    """kinds a and b alternate; lanes 60-62, 124-126 and 188-190 (and l % 7 == 3) hold rows without walks"""
    if l % 256 in (63, 64, 127, 128, 191, 192):
        return "ab"[l % 2]
    if any(e - 4 < l % 256 < e - 1 for e in (64, 128, 192)) or l % 7 == 3:
        return SKIPS[l % 3]
    return "ab"[l % 2]


def case_lanes():
    """513 rows: three batches of 256 lanes (wd = 4), the last of one row; neighbouring listed lanes of different tight
    sets, lanes without walks between them; its prefixes give every lane width"""
    c = lane_case([lane_kind(l) for l in range(513)], widths=WIDTHS, budgets=GROUP_SIZES)
    c["named"] = {*{f"width_{p}" for p in WIDTHS}, *{f"L_{L}" for L in (32, 64, 96, 128, 160, 224, 256)},
                  *{f"wd_{k}" for k in (1, 2, 3, 4)}, "wd_partial_last_word",
                  *{f"tight_differs_{x}_{x + 1}" for x in (63, 127, 191)}, *{f"skip_{k}" for k in SKIPS},
                  "batches_1_2_list", "last_batch_cnt_1", *{f"group_close_{x}" for x in GROUP_SIZES},
                  "group_close_in_batch_2", "chunk_plain_store"}
    return c


def case_batch_1_empty():
    return dict(lane_case([SKIPS[l % 3] for l in range(256)] + ["ab"[l % 2] for l in range(256)]),
                named={"batch_1_empty_2_lists"})


def case_batch_2_empty():
    return dict(lane_case(["ab"[l % 2] for l in range(256)] + [SKIPS[l % 3] for l in range(256)] + ["b"]),
                named={"batches_1_3_list_2_empty", "last_batch_cnt_1"})


def case_grow():
    """batch 1: 256 walks of 1 edge; batch 2: 512 walks of 2 edges; batch 3: 40 rows of 64 walks of 12 edges -- on a
    fresh workspace batch 2 and batch 3 each outgrow what the batches before them placed"""
    return dict(lane_case(["edge"] * 256 + ["a"] * 256 + ["diamonds"] * 40), fresh=True,
                named={"grow_copy", "grow_twice"})


def case_budget_refusal():
    """a row of batch 2 whose 8-edge walk needs more layers than the budget, after batch 1 has stored its groups"""
    c = lane_case(["ab"[l % 2] for l in range(300)] + ["long"])
    g = Graph(c["n"], c["src"], c["dst"])
    c["refusal_budget"] = layer_bytes(2, 2, g.n_ab)
    c["named"] = {"budget_refused_in_batch_2"}
    return c


def case_hubs():
    """Hubs of HUB_DEGREES in-edges, each parent with one edge to its hub and edges from sources sa and sb: sa's
    edges cost 1 into the parents in even 128-position chunk parts of the hub's in-list and 2 into the others, sb's
    the other way round, so a part is zero for one of two neighbouring lanes and not for the other.  Sources s31, s32
    and s33 reach the first hub's parents at cost 2 but parent j at cost 1: the only tight entry of their hub row is
    step index j, behind non-tight ones."""
    b = WBuilder()
    sa, sb = b.new(), b.new()
    sj = {j: b.new() for j in (31, 32, 33)}
    hubs = []
    for d in HUB_DEGREES:
        hub = b.new()
        par = b.new(d)
        hubs.append((hub, par))
        for p in par:
            b.edge(p, hub)
    # the in-CSC offsets depend on the degrees only: place the weights by the parts they fall in
    pairs = [(sa, p) for _, par in hubs for p in par] + [(sb, p) for _, par in hubs for p in par]
    pairs += [(sj[j], p) for j in sj for p in hubs[0][1]]
    src = b.src + [x for x, _ in pairs]
    dst = b.dst + [y for _, y in pairs]
    lay = layout(b.n, src, dst)
    perm = np.empty(b.n, np.int64)
    perm[lay["inv"]] = np.arange(b.n)
    in_off = np.concatenate([[0], np.cumsum(lay["ind"][lay["inv"]])])
    w = list(b.w)
    for x, y in pairs:
        hub, par = next(h for h in hubs if h[1][0] <= y <= h[1][-1])
        i = y - par[0]
        start = int(in_off[perm[hub]])
        part = (start + i) // 128 - start // 128
        if x in (sa, sb):
            w.append(1 if (part % 2 == 0) == (x == sa) else 2)
        else:
            w.append(1 if i == next(j for j in sj if sj[j] == x) else 2)
    rows = [r for hub, _ in hubs for r in ((sa, hub), (sb, hub))] + [(sj[j], hubs[0][0]) for j in sj]
    return dict(n=b.n, src=src, dst=dst, w=w, rows=rows, ok=[1] * len(rows), chunks=True, threads=True,
                named={*{f"hub_{d}" for d in HUB_DEGREES}, "chunk_split_nonzero", "chunk_zero_next_to_nonzero_lane",
                       *{f"pick_step_{j}_after_nontight" for j in (31, 32, 33)}, "prefix_eq_rank_window_start"})


def case_lengths():
    """Zero-cost walks s -> t of 1 .. 20 edges (one chain each) and of 64 .. 80 edges (a 63-edge chain, then chains of
    1 .. 17): 37 lengths, none in 21 .. 63, so the lengths 32 .. 63 are a whole window without walks"""
    b = WBuilder()
    s, t = b.new(), b.new()
    for k in range(1, 21):
        b.chain(s, k, t, w=0)
    y = b.chain(s, 63, w=0)
    for k in range(1, 18):
        b.chain(y, k, t, w=0)
    return dict(n=b.n, src=b.src, dst=b.dst, w=b.w, rows=[(s, t), (y, t)], ok=[1, 1],
                named={"lengths_over_32", "length_window_empty"})


def case_infinite():
    """a 2-cycle s <-> a (t = a: infinite from h = 2 = |B(t)|); a zero-cost cycle at s2 ahead of 64 branches of 1 .. 64
    edges into t2 (|B(t2)| > 2000, infinite only after that many layers); a tight cycle that s3 reaches but that does
    not reach t3; a zero-cost cycle into t4 that s4 does not reach (its edges are tight between sentinels, outside
    B(t4)); a zero-cost self-loop at t5, and s == t on it"""
    b = WBuilder()
    s, a = b.new(), b.new()
    b.edge(s, a, w=0)
    b.edge(a, s, w=0)
    s2, c2, t2 = b.new(), b.new(), b.new()
    b.edge(s2, c2, w=0)
    b.edge(c2, s2, w=0)
    for k in range(1, 65):
        b.chain(s2, k, t2, w=0)
    s3, t3, c1, c3 = (b.new() for _ in range(4))
    b.edge(s3, t3)
    b.edge(s3, c1, w=0)
    b.edge(c1, c3, w=0)
    b.edge(c3, c1, w=0)
    s4, t4, z1, z2 = (b.new() for _ in range(4))
    b.edge(s4, t4, w=3)
    b.edge(z1, z2, w=0)
    b.edge(z2, z1, w=0)
    b.edge(z1, t4, w=0)
    s5, t5 = b.new(), b.new()
    b.edge(s5, t5, w=2)
    b.edge(t5, t5, w=0)
    rows = [(s, a), (s2, t2), (s3, t3), (s4, t4), (s5, t5), (t5, t5)]
    return dict(n=b.n, src=b.src, dst=b.dst, w=b.w, rows=rows, ok=[1] * len(rows), mps=(7,),
                named={"inf_at_h_eq_b", "inf_b_over_2000", "cycle_off_route_finite", "sentinel_cycle_outside_b",
                       "self_loop_at_t"})


def case_saturation():
    """64 zero-cost diamonds: 2^64 walks, a finite count that saturates; an infinite row in the same batch"""
    n, src, dst = diamonds(64)
    b = WBuilder(n)
    b.src, b.dst, b.w = src.tolist(), dst.tolist(), [0] * len(src)
    x = b.new()
    b.edge(0, x)
    b.edge(x, x, w=0)
    return dict(n=b.n, src=b.src, dst=b.dst, w=b.w, rows=[(0, n - 1), (0, x), (0, 11)], ok=[1, 1, 1], mps=(7,),
                named={"sat_refused", "sat_lists_1", "sat_lists_7", "sat_and_inf_one_batch"})


def case_specials_i64():
    """weights near -2^62: max/2 + w from an unreached vertex is a valid cost, so such an edge is tight (x -> s
    lowers d(s) to -1; u -> t2 gives t2 a cost its other edge cannot reach); every vertex starts dirty"""
    b = WBuilder()
    s, t, x, u, s2, t2 = (b.new() for _ in range(6))
    b.edge(x, s, w=-(1 << 62))
    b.edge(s, t, w=0)
    b.edge(s, t, w=1)
    b.edge(u, t2, w=-(1 << 62) + 5)
    b.edge(s2, t2, w=3)
    rows = [(s, t), (s2, t2), (x, t), (s, s)]
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=rows, ok=[1] * 4, small=True,
                named={"i64_sentinel_tight", "neg_weights_dirty"})


def case_specials_f64():
    """DOUBLE: an edge of -inf (d = -inf, and -inf + w stays tight after it), -0.0 next to 0.0, NaN (never tight)"""
    b = WBuilder()
    s, a, t, x, y, z = (b.new() for _ in range(6))
    b.edge(s, a, w=-0.0)
    b.edge(a, t, w=0.0)
    b.edge(s, t, w=0.0)
    b.edge(s, t, w=np.nan)
    b.edge(s, x, w=np.nan)
    b.edge(x, t, w=0.0)
    b.edge(t, y, w=-np.inf)
    b.edge(y, z, w=1.0)
    b.edge(t, z, w=2.0)
    rows = [(s, t), (s, y), (s, z), (a, z), (x, t)]
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.float64), rows=rows, ok=[1] * 5, small=True,
                named={"f64_neg_inf_tight", "f64_neg_zero", "f64_nan", "neg_weights_dirty"})


def case_layout():
    """s == t on a vertex without in-edges (internal id >= n_ab) and on one with them"""
    b = WBuilder()
    s, a, t = b.new(), b.new(), b.new()
    b.edge(s, a, w=2)
    b.edge(a, t, w=2)
    b.edge(s, t, w=4)
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=[(s, s), (t, t), (s, t)], ok=[1] * 3,
                small=True, named={"s_eq_t_source_only"})


def case_n1():
    return dict(n=1, src=[0], dst=[0], w=np.zeros(1, np.int64), rows=[(0, 0)], ok=[1], small=True, named={"n_1"})


def case_m0():
    return dict(n=3, src=[], dst=[], w=np.zeros(0, np.int64), rows=[(0, 0), (1, 1), (2, 0)], ok=[1] * 3, small=True,
                named={"m_0_s_eq_t"})


def case_walk_limit():
    """a zero-cost 2-cycle s <-> a: a walk s -> a every 2 edges, so 33000 of them take more than 65533 edges"""
    return dict(n=2, src=[0, 1], dst=[1, 0], w=np.zeros(2, np.int64), rows=[(0, 1)], ok=[1], mps=(33000,),
                named={"walk_limit_refused"})


CATALOGUE = {
    "lanes": case_lanes,
    "batch_1_empty": case_batch_1_empty,
    "batch_2_empty": case_batch_2_empty,
    "grow": case_grow,
    "budget_refusal": case_budget_refusal,
    "hubs": case_hubs,
    "lengths": case_lengths,
    "infinite": case_infinite,
    "saturation": case_saturation,
    "specials_i64": case_specials_i64,
    "specials_f64": case_specials_f64,
    "layout": case_layout,
    "n1": case_n1,
    "m0": case_m0,
    "walk_limit": case_walk_limit,
}

REQUIRED = (
    {f"width_{p}" for p in WIDTHS} | {f"L_{L}" for L in (32, 64, 96, 128, 160, 224, 256)}
    | {f"wd_{k}" for k in (1, 2, 3, 4)} | {"wd_partial_last_word"}
    | {f"tight_differs_{x}_{x + 1}" for x in (63, 127, 191)} | {f"skip_{k}" for k in SKIPS}
    | {"batches_1_2_list", "batch_1_empty_2_lists", "batches_1_3_list_2_empty", "last_batch_cnt_1"}
    | {"grow_copy", "grow_twice"}
    | {f"group_close_{x}" for x in GROUP_SIZES} | {"group_close_in_batch_2", "budget_refused_in_batch_2"}
    | {f"hub_{d}" for d in HUB_DEGREES} | {"chunk_plain_store", "chunk_split_nonzero", "chunk_zero_next_to_nonzero_lane"}
    | {f"pick_step_{j}_after_nontight" for j in (31, 32, 33)} | {"prefix_eq_rank_window_start"}
    | {"lengths_over_32", "length_window_empty"}
    | {"inf_at_h_eq_b", "inf_b_over_2000", "cycle_off_route_finite", "sentinel_cycle_outside_b", "self_loop_at_t"}
    | {"sat_refused", "sat_lists_1", "sat_lists_7", "sat_and_inf_one_batch"}
    | {"i64_sentinel_tight", "neg_weights_dirty", "f64_neg_inf_tight", "f64_neg_zero", "f64_nan"}
    | {"s_eq_t_source_only", "n_1", "m_0_s_eq_t", "walk_limit_refused"}
)


@lru_cache(maxsize=None)
def case(name):
    c = CATALOGUE[name]()
    c["w"] = np.asarray(c["w"], np.float64 if np.asarray(c["w"]).dtype.kind == "f" else np.int64)
    c["g"] = WGraph(c["n"], c["src"], c["dst"], c["w"])
    c["ps"] = np.array([s for s, _ in c["rows"]], np.int64)
    c["pd"] = np.array([t for _, t in c["rows"]], np.int64)
    c["sv"] = np.array(c["ok"], np.uint8)
    return c


def call(name, list_, mp, idx=None, budget=KS_BUDGET):
    c = case(name)
    idx = range(len(c["rows"])) if idx is None else idx
    return _call(name, list_, mp, tuple(idx), budget)


@lru_cache(maxsize=None)
def _call(name, list_, mp, idx, budget):
    c = case(name)
    return ac_call(c["g"], [c["rows"][i] for i in idx], [c["ok"][i] for i in idx], list_, mp, budget)


def max_paths_of(name):
    """0, 1, the largest finite count below INT64_MAX and one more, and the case's own"""
    counts = [r["count"] for r in call(name, False, 0)["rows"] if 0 < r["count"] < INT64_MAX]
    out = [0, 1] + ([max(counts), max(counts) + 1] if counts else []) + list(case(name).get("mps", ()))
    return tuple(dict.fromkeys(out))


def listed_budget(name, size):
    """the layer budget under which the first storing group of batch 1 closes at exactly `size` lanes"""
    res = call(name, True, 0)
    return layer_bytes(max(h for _, h in res["batches"][0]["listed"]), size, case(name)["g"].n_ab)


# ---- the work record's boundaries ---------------------------------------------------------------------------------------
def case_hits(name):
    c = case(name)
    g = c["g"]
    hits = set()
    full = call(name, True, 0)
    for p in c.get("widths", ()):
        res = call(name, True, 0, range(p))
        hits |= {f"width_{p}", f"L_{res['L']}", f"wd_{res['wd']}"}
        if res["L"] % 64 and any(b["cnt"] > 64 * (res["wd"] - 1) for b in res["batches"]):
            hits.add("wd_partial_last_word")
    for bi, batch in enumerate(full["batches"]):
        res = full["rows"][batch["b0"]:batch["b0"] + batch["cnt"]]
        lanes = [l for l, _ in batch["listed"]]
        for x in (63, 127, 191):
            if x in lanes and x + 1 in lanes and \
                    not np.array_equal(g.tight(res[x]["s"]), g.tight(res[x + 1]["s"])):
                hits.add(f"tight_differs_{x}_{x + 1}")
        for a_, b_ in zip(lanes, lanes[1:]):
            for l in range(a_ + 1, b_):
                hits.add(f"skip_{res[l]['kind']}")
        if batch["cnt"] == 1 and bi == len(full["batches"]) - 1 and bi > 0:
            hits.add("last_batch_cnt_1")
    listing = [bool(b["listed"]) for b in full["batches"]]
    if listing[:2] == [True, True]:
        hits.add("batches_1_2_list")
    if listing[:2] == [False, True]:
        hits.add("batch_1_empty_2_lists")
    if listing[:3] == [True, False, True]:
        hits.add("batches_1_3_list_2_empty")
    if c.get("fresh"):
        grows = [b.get("elems") == "grow" or b.get("walk_off") == "grow" for b in full["fresh"]]
        if len(grows) >= 3 and grows[1]:
            hits.add("grow_copy")
            if grows[2]:
                hits.add("grow_twice")
    for size in c.get("budgets", ()):
        res = call(name, True, 0, budget=listed_budget(name, size))
        if res["error"] is None and len(res["batches"][0]["groups"][0][0]) == size:
            hits.add(f"group_close_{size}")
            if len(res["batches"]) > 1 and len(res["batches"][1]["groups"]) > 1:
                hits.add("group_close_in_batch_2")
    if c.get("refusal_budget"):
        res = call(name, True, 0, budget=c["refusal_budget"])
        err = res["error"]
        if err is not None and err.why == "budget" and err.batch == 1 and res["batches"][0]["groups"]:
            hits.add("budget_refused_in_batch_2")
    # the rows: walks, chunks, windows, infinite rule, saturation, specials
    for mp in max_paths_of(name):
        res = call(name, True, mp)
        rows = res["rows"]
        if res["error"] is not None and res["error"].why == "saturated":
            if any(r["count"] == INT64_MAX and r["inf_at"] is None for r in rows):
                hits.add("sat_refused")
        if res["error"] is not None and res["error"].why == "too_long":
            hits.add("walk_limit_refused")
        for r in rows:
            if r["count"] == INT64_MAX and r["inf_at"] is None and r["npaths"] == mp and mp in (1, 7):
                hits.add(f"sat_lists_{mp}")
            for w in r["work"]:
                o = int(g.st_off[w["vertex"]])
                admit = g.tight(r["s"])[g.st_idx[o:o + w["j"]]]
                if w["j"] in (31, 32, 33) and not admit.any():
                    hits.add(f"pick_step_{w['j']}_after_nontight")
                if w["at_window_end"]:
                    hits.add("prefix_eq_rank_window_start")
            lens = [h for h, k in enumerate(r["takes"]) if k]
            if len(lens) > WINDOW:
                hits.add("lengths_over_32")
            if lens and any(not any(r["ct"][x * WINDOW:(x + 1) * WINDOW]) for x in range(lens[-1] // WINDOW)):
                hits.add("length_window_empty")
    counts = call(name, False, 0)
    for bi in range(len(counts["batches"])):
        b0, cnt = counts["batches"][bi]["b0"], counts["batches"][bi]["cnt"]
        rows = counts["rows"][b0:b0 + cnt]
        if any(r["inf_at"] for r in rows) and any(r["count"] == INT64_MAX and r["inf_at"] is None for r in rows):
            hits.add("sat_and_inf_one_batch")
    for r in counts["rows"]:
        s, t = r["s"], r["t"]
        if r["inf_at"] is not None and r["inf_at"] == r["bsize"] and r["inf_at"] > 1:
            hits.add("inf_at_h_eq_b")
        if r["inf_at"] is not None and r["bsize"] >= 2000 and r["inf_at"] == r["bsize"]:
            hits.add("inf_b_over_2000")
        if not r["open"]:
            continue
        T = g.tight(s)
        tight = [(a, 0, k, int(g.e[k])) for k, a in enumerate(g.row.tolist()) if T[k]]
        cyc = {a for a, _, k, b in tight if a == b} | {a for a, _, _, b in tight
                                                       if any(x == b and y == a for x, _, _, y in tight)}
        if r["kind"] == "counts" and r["count"] < INT64_MAX:
            d = g.dist(s)
            if any(d[x] != g.inf and x not in r["B"] for x in cyc):
                hits.add("cycle_off_route_finite")
            if any(d[x] == g.inf and x not in r["B"] and t in g.e[g.v[x]:g.v[x + 1]] for x in cyc):
                hits.add("sentinel_cycle_outside_b")
        if r["inf_at"] is not None and any(a == b == t for a, _, _, b in tight):
            hits.add("self_loop_at_t")
        if r["kind"] == "counts":
            d = g.dist(s)
            if not g.is_f and any(T[k] and d[int(g.row[k])] == g.inf and d[int(g.e[k])] != g.inf
                                  for k in range(len(g.e))):
                hits.add("i64_sentinel_tight")
            if g.is_f:
                if any(T[k] and g.w[k] == -np.inf for k in range(len(g.e))):
                    hits.add("f64_neg_inf_tight")
                if any(T[k] and g.w[k] == 0 and np.signbit(g.w[k]) for k in range(len(g.e))):
                    hits.add("f64_neg_zero")
            if s == t and g.perm[s] >= g.n_ab and r["count"] == 1:
                hits.add("s_eq_t_source_only")
    if g.is_f and np.isnan(g.w).any():
        hits.add("f64_nan")
    if (g.w < 0).any():
        hits.add("neg_weights_dirty")
    if g.n == 1 and len(g.e):
        hits.add("n_1")
    if len(g.e) == 0 and any(s == t for s, t in c["rows"]):
        hits.add("m_0_s_eq_t")
    if c.get("chunks"):
        hits |= chunk_hits(name)
    for r in full["rows"]:
        if r["lists"] and r["t"] < g.n and g.perm[r["t"]] < g.n_ab and 0 < g.in_deg[r["t"]] < 128:
            hits.add("chunk_plain_store")
    return hits


def chunk_hits(name):
    """k_ks_omega's parts of the hub rows, per lane, in the storing pass's step order (non-tight entries as zeros)"""
    c = case(name)
    g = c["g"]
    res = call(name, True, 0)
    hits = set()
    parts = {}
    for l, r in enumerate(res["rows"]):
        if not r["lists"]:
            continue
        admit = g.tight(r["s"])[g.step_csr]
        for w in chunk_work(g, r["lay"], {r["t"]}, r["last"], g.step_in, admit):
            if any(w["parts"]):
                if w["split"]:
                    hits.add("chunk_split_nonzero")
                if w["re"] - w["rs"] in HUB_DEGREES:
                    hits.add(f"hub_{w['re'] - w['rs']}")
            parts[(l, w["u"], w["h"])] = w["parts"]
    for (l, u, h), p in parts.items():
        q = parts.get((l + 1, u, h))
        if q and any(x == 0 and y > 0 for x, y in zip(p, q)):
            hits.add("chunk_zero_next_to_nonzero_lane")
    return hits


# ---- CPU: the hits, the coverage, the oracle against the restatement ------------------------------------------------
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_catalogue_hits_its_boundaries(name):
    missing = case(name)["named"] - case_hits(name)
    assert not missing, sorted(missing)


def test_catalogue_covers_every_boundary():
    named = set().union(*(CATALOGUE[x]()["named"] for x in CATALOGUE))
    assert REQUIRED <= named, sorted(REQUIRED - named)
    assert named <= REQUIRED, sorted(named - REQUIRED)


def oracle_call(name, list_, mp, idx=None, lanes=None):
    c = case(name)
    g = c["g"]
    idx = np.arange(len(c["rows"])) if idx is None else np.asarray(list(idx))
    L = lanes or lanes_for(g.n, len(idx))
    args = (g.n, g.v, g.e, g.ids, g.w, c["ps"][idx], c["pd"][idx])
    if not list_:
        return oac.cheapest_path_count(*args, c["sv"][idx], None, L)
    return oac.all_cheapest_paths(*args, mp, c["sv"][idx], None, L)


ORACLE_CODE = {"unsupported": oac.ERR_UNSUPPORTED, "too_large": oac.ERR_ALLOC}
DEVICE_CODE = {"unsupported": PGQ_ERR_UNSUPPORTED, "too_large": PGQ_ERR_OOM}


def restated_lists(res):
    return [r["lists"] if r["npaths"] else None for r in res["rows"]]


def check_oracle(name, list_, mp, idx=None):
    res = call(name, list_, mp, idx)
    if res["error"] is not None:
        with pytest.raises(orc.OracleError) as ex:
            oracle_call(name, list_, mp, idx)
        assert ex.value.code == ORACLE_CODE[res["error"].kind], (name, mp)
        return
    if not list_:
        cnt, valid, st = oracle_call(name, False, 0, idx)
        assert cnt.tolist() == [r["count"] for r in res["rows"]], name
        assert valid.tolist() == [int(r["count"] > 0) for r in res["rows"]], name
        assert st["pull_levels"] == res["stats"]["pull_levels"], name
    else:
        paths, cnt, st = oracle_call(name, True, mp, idx)
        assert cnt.tolist() == [r["count"] for r in res["rows"]], (name, mp)
        assert paths == restated_lists(res), (name, mp)
        assert st["pull_levels"] == res["stats"]["pull_levels"], (name, mp)
    for x in ("batches", "push_levels"):
        assert st[x] == res["stats"][x], (name, mp, x)


@pytest.mark.parametrize("name", list(CATALOGUE))
def test_oracle_equals_the_restatement(name):
    c = case(name)
    check_oracle(name, False, 0)
    for mp in max_paths_of(name):
        check_oracle(name, True, mp)
    for p in c.get("widths", ()):
        check_oracle(name, True, 0, range(p))


@pytest.mark.parametrize("name", [x for x in CATALOGUE if CATALOGUE[x]().get("small")])
def test_small_cases_are_the_brute_force_walks(name):
    c = case(name)
    g = c["g"]
    res = call(name, True, 40)
    for r in res["rows"]:
        s, t = r["s"], r["t"]
        tight = tight_edges(g.n, g.v, g.e, g.w, g.dist(s))
        if not r["open"]:
            assert r["count"] == 0
            continue
        inf = tight_cycle_on_route(g.n, tight, s, t)
        assert inf == (r["count"] == INT64_MAX), (s, t)
        walks = brute_walks(tight, g.ids, s, t, r["last"] if inf else g.n)
        assert (r["lists"] or []) == [x[2] for x in walks[:40]], (s, t)
        if not inf:
            assert r["count"] == len(walks), (s, t)


def test_refusals_of_the_restatement():
    """max_paths = 0 with a count of INT64_MAX (saturated and infinite), a row over the layer budget, a walk past
    65533 edges: each refused, as by the oracle"""
    assert call("saturation", True, 0)["error"].why == "saturated"
    assert call("n1", True, 0)["error"].why == "saturated"
    assert call("walk_limit", True, 33000)["error"].why == "too_long"
    assert call("walk_limit", True, 2)["error"] is None
    c = case("budget_refusal")
    assert call("budget_refusal", True, 0, budget=c["refusal_budget"])["error"].why == "budget"


# ---- GPU: the device against the oracle and the restatement -------------------------------------------------------------
def build(ctx, name):
    c = case(name)
    return pgq.DeviceCSR.build(ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64),
                               weight=c["w"])


def device_call(csr, name, list_, mp, idx=None):
    c = case(name)
    idx = np.arange(len(c["rows"])) if idx is None else np.asarray(list(idx))
    ps, pd, sv = c["ps"][idx], c["pd"][idx], c["sv"][idx]
    if not list_:
        return csr.cheapest_path_count(ps, pd, sv)
    return csr.all_cheapest_paths(ps, pd, mp, sv)


def compare(csr, name, list_, mp, idx=None, cheapest=None):
    """the device's answer equals the restatement's and the oracle's (a refusal: its status) -> stats or None"""
    res = call(name, list_, mp, idx)
    if res["error"] is not None:
        with pytest.raises(pgq.PgqError) as ex:
            device_call(csr, name, list_, mp, idx)
        assert ex.value.status == DEVICE_CODE[res["error"].kind], (name, mp)
        return None
    if not list_:
        cnt, valid, st = device_call(csr, name, False, 0, idx)
        assert cnt.tolist() == [r["count"] for r in res["rows"]], name
        assert valid.tolist() == [int(r["count"] > 0) for r in res["rows"]], name
        ocnt, ovalid, ost = oracle_call(name, False, 0, idx)
        assert np.array_equal(cnt, ocnt) and np.array_equal(valid, ovalid)
    else:
        paths, cnt, st = device_call(csr, name, True, mp, idx)
        assert cnt.tolist() == [r["count"] for r in res["rows"]], (name, mp)
        assert paths == restated_lists(res), (name, mp)
        opaths, ocnt, ost = oracle_call(name, True, mp, idx)
        assert paths == opaths and np.array_equal(cnt, ocnt)
        if cheapest is not None:
            assert [x[0] if x else None for x in paths] == [cheapest[i] if x else None
                                                            for i, x in enumerate(paths)], (name, mp)
    assert st["lanes"] == res["L"], name
    for x in ("batches", "push_levels", "pull_levels"):
        assert st[x] == res["stats"][x] == ost[x], (name, mp, x)
    return st


def cheapest_paths(csr, name):
    c = case(name)
    return csr.cheapest_path(c["ps"], c["pd"], c["sv"])[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    csr = build(gpu_ctx, name)
    try:
        cheapest = cheapest_paths(csr, name)
        compare(csr, name, False, 0)
        for mp in max_paths_of(name):
            compare(csr, name, True, mp, cheapest=cheapest)
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lanes", "hubs", "infinite", "saturation", "specials_f64"])
def test_device_widths_and_row_order(gpu_ctx, name):
    c = case(name)
    csr = build(gpu_ctx, name)
    try:
        for p in c.get("widths", ()):
            compare(csr, name, True, 0, range(p))
            compare(csr, name, False, 0, range(p))
        perm = np.random.default_rng(5).permutation(len(c["rows"]))
        for mp in max_paths_of(name):
            if call(name, True, mp)["error"] is not None:
                continue
            paths, cnt, _ = device_call(csr, name, True, mp, perm)
            opaths, ocnt, _ = oracle_call(name, True, mp, perm)
            assert paths == opaths and np.array_equal(cnt, ocnt), mp
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_layer_budgets(gpu_ctx, monkeypatch):
    """budgets that close the first storing group of each batch at exactly 1, 31, 32, 33, 64 and 65 lanes, and one
    byte below each; the storing pass's launches follow the restated groups"""
    name = "lanes"
    g = case(name)["g"]
    csr = build(gpu_ctx, name)
    try:
        base = compare(csr, name, True, 0)
        base_groups = [b["groups"] for b in call(name, True, 0)["batches"]]
        for size in GROUP_SIZES:
            for budget in (listed_budget(name, size), listed_budget(name, size) - 1):
                monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(budget))
                res = call(name, True, 0, budget=budget)
                if res["error"] is not None:
                    assert budget < layer_bytes(2, 1, g.n_ab)
                    with pytest.raises(pgq.PgqError) as ex:
                        device_call(csr, name, True, 0)
                    assert ex.value.status == PGQ_ERR_UNSUPPORTED
                    continue
                groups = [b["groups"] for b in res["batches"]]
                assert len(groups[0][0][0]) == (size if budget % 8 == 0 else size - 1), (size, budget)
                paths, cnt, st = device_call(csr, name, True, 0)
                assert paths == restated_lists(call(name, True, 0)), (size, budget)
                want = sum(store_launches(x) for x in groups) - sum(store_launches(x) for x in base_groups)
                assert (st["kernel_launches"] - st["levels"]) - (base["kernel_launches"] - base["levels"]) == want, \
                    (size, budget)
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_budget_refusal_in_batch_2(gpu_ctx, monkeypatch):
    """a row of batch 2 over the budget after batch 1 has stored: refused; then the same CSR answers in full"""
    name = "budget_refusal"
    csr = build(gpu_ctx, name)
    try:
        monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(case(name)["refusal_budget"]))
        with pytest.raises(pgq.PgqError) as ex:
            device_call(csr, name, True, 0)
        assert ex.value.status == PGQ_ERR_UNSUPPORTED
        monkeypatch.delenv("PGQ_B200_KSP_LAYER_BUDGET")
        compare(csr, name, True, 0)
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["chunked", "build", "build_device", "upload", "build_keys", "build_keys_device"])
@pytest.mark.parametrize("name", ["hubs", "specials_i64", "specials_f64", "lengths"])
def test_device_construction_routes(gpu_ctx, name, route):
    from test_gpu_csr_weighted_builds import graph_from_rows, make
    c = case(name)
    gr = graph_from_rows(c["n"], c["src"], c["dst"], c["w"])
    v, e, ids, w = orc.csr_build_weighted(gr.n, gr.src, gr.dst, gr.w, gr.eid)
    csr = make(gpu_ctx, gr, route)
    try:
        L = lanes_for(c["n"], len(c["ps"]))
        cnt, valid, _ = csr.cheapest_path_count(c["ps"], c["pd"], c["sv"])
        ocnt, ovalid, _ = oac.cheapest_path_count(c["n"], v, e, ids, w, c["ps"], c["pd"], c["sv"], None, L)
        assert np.array_equal(cnt, ocnt) and np.array_equal(valid, ovalid)
        for mp in max_paths_of(name):
            if call(name, True, mp)["error"] is not None:
                continue  # (the refusals: test_device_catalogue)
            paths, cnt, _ = csr.all_cheapest_paths(c["ps"], c["pd"], mp, c["sv"])
            opaths, ocnt, _ = oac.all_cheapest_paths(c["n"], v, e, ids, w, c["ps"], c["pd"], mp, c["sv"], None, L)
            assert paths == opaths and np.array_equal(cnt, ocnt), mp
    finally:
        csr.free()


def one_workspace_context(monkeypatch):
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    return pgq.Context(0)


@pytest.mark.gpu
def test_device_dirty_workspace(monkeypatch):
    """one workspace: a larger shortest_k_paths and shortest_k_groups on another CSR, then all_cheapest_paths; then a
    large all_cheapest_paths, then small calls of the other two -- every WS_KS_* slot starts out stale"""
    ctx = one_workspace_context(monkeypatch)
    try:
        for steps in ((("ks", "lanes", [("ks", 2), ("kg", 1, 0)]), ("ac", "lanes"), ("ac", "hubs")),
                      (("ac", "grow"), ("ac", "infinite"), ("ks", "n2", None), ("ks", "fan_in", None),
                       ("ac", "specials_f64"))):
            for step in steps:
                csr = ks_build(ctx, step[1]) if step[0] == "ks" else build(ctx, step[1])
                try:
                    if step[0] == "ks":
                        ks_compare_all(csr, step[1], keys=step[2])
                    else:
                        for mp in max_paths_of(step[1]):
                            compare(csr, step[1], True, mp)
                finally:
                    csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_fresh_workspace_grows(monkeypatch):
    """a new context with one workspace: batch 2 and batch 3 each grow the walk buffers, keeping what the batches
    before them placed"""
    ctx = one_workspace_context(monkeypatch)
    try:
        csr = build(ctx, "grow")
        try:
            assert [sorted(x.values()) for x in call("grow", True, 0)["fresh"]][1:] == [["grow", "grow"]] * 2
            compare(csr, "grow", True, 0)
        finally:
            csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_eight_threads(gpu_ctx):
    name = "hubs"
    c = case(name)
    csr = build(gpu_ctx, name)
    mp = max_paths_of(name)[2]
    exp = (restated_lists(call(name, True, mp)), [r["count"] for r in call(name, False, 0)["rows"]])
    out = [None] * 8

    def work(i):
        out[i] = (csr.all_cheapest_paths(c["ps"], c["pd"], mp, c["sv"])[0],
                  csr.cheapest_path_count(c["ps"], c["pd"], c["sv"])[0].tolist())

    ths = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(o == exp for o in out)
