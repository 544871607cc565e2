"""shortest_path_count, all_shortest_paths, shortest_k_paths and WALK's shortest_k_groups at the boundaries of their
path counts, chunks, warp scans and saturation, against two restatements.

The four functions share one piece of device machinery (csrc/pgq_allshortest.cu, csrc/pgq_kshortest.cu,
csrc/pgq_count.cuh): saturating 64-bit path counts (k_sigma_level, a warp per vertex, 32 lanes at a time; k_ks_omega,
128 in-CSC positions per warp, with a plain store for an in-list inside one chunk and atomic_sat_add for the parts of a
longer one), the step-ordered in-lists of build_step_lists (keys u * n + original parent id), and two warp-wide
saturating prefix-scan unrankers (k_as_unrank, k_ks_unrank; k_ks_unrank also scans a row's walk lengths 32 at a time).
Their answers are exact integers and exact lists, so a single wrong step is a wrong query result.  So:

- a restatement in Python integers written from the definitions: per-length walk counts by layered DP over the edge
  rows, and an unranker that walks back from t over each vertex's in-edges in step order with exact prefix sums.  It
  shows its work: per step the picked edge's step index, its 32-edge window and whether the prefix at that window's
  start equals the rank; per walk its 32-length window; per layer the in-lists that span more than one 128-position
  chunk and which of their parts are non-zero; per row its lane and 64-bit word; per call the storing groups of
  ks_run's greedy loop under a layer budget;
- a deterministic catalogue whose cases each name the boundaries they hit, proven on the CPU from the work record and
  layout(); a coverage test asks every boundary to be hit by some case;
- the C oracles (oracle/pgq_oracle_allshortest.c, pgq_oracle_kshortest.c, pgq_oracle_kgroups.c in WALK mode) equal to
  the restatement on every case, and to brute force on the small ones;
- on the GPU, the device equal to the oracle on every case, under lane widths and a row permutation, forced BFS
  schedules (checked in the level trace), layer budgets that close storing groups at chosen sizes (checked in the
  launch counts), other construction routes, one dirty workspace and eight threads on one CSR."""
import re
import threading
from collections import defaultdict
from functools import lru_cache

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_OOM, PGQ_ERR_UNSUPPORTED
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_allshortest as oas
from oracle import pgq_oracle_kgroups as okg
from oracle import pgq_oracle_kshortest as oks
from test_all_shortest_paths import diamonds
from test_csr_layout_shapes import Shape, layout, make
from test_shortest_k_paths import brute_walks, length_counts

INT64_MAX = (1 << 63) - 1
WALK_MAX = 65533
WINDOW = 32      # edges (unrankers) and walk lengths (k_ks_unrank's length scan) per warp step
CHUNK = 128      # KS_CHUNK: in-CSC positions per warp of k_ks_omega
KS_WIDTH = 512   # ks_lanes' widest batch
BFS_COUNTERS = ("batches", "levels", "edges_traversed", "frontier_vertices", "push_levels", "pull_levels", "lanes",
                "searches", "pruned", "search_rows")
KS_COUNTERS = ("batches", "lanes", "searches", "levels", "push_levels")


class Unsupported(Exception):
    pass


class TooLarge(Exception):
    pass


# ---- the restatement ---------------------------------------------------------------------------------------------------
class Graph:
    """The edge rows with the reference CSR (original ids), the device's internal order (layout()) and in-CSC, and
    every vertex's in-edges in step order: (parent's original id, the edge's position in the parent's adjacency)."""

    def __init__(self, n, src, dst):
        self.n = n
        self.src, self.dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
        self.v, self.e, self.ids = orc.csr_build(n, self.src, self.dst)
        self.lay = layout(n, self.src, self.dst)
        inv = self.lay["inv"]
        self.perm = np.empty(n, np.int64)
        self.perm[inv] = np.arange(n)
        self.n_ab = self.lay["n_ab"]
        self.in_off = np.concatenate([[0], np.cumsum(self.lay["ind"][inv])]).astype(np.int64)
        ti, pi = self.perm[self.dst], self.perm[self.src]
        self.in_adj = pi[np.lexsort((pi, ti))]  # internal parent ids, in-CSC order
        m = len(self.e)
        row = np.repeat(np.arange(n), np.diff(self.v[:n + 1]))
        order = np.lexsort((np.arange(m), row, self.e))  # by target, then parent, then adjacency position
        self.st_par, self.st_eid, self.st_idx = row[order], self.ids[order], order
        self.st_off = np.searchsorted(self.e[order], np.arange(n + 1))
        self.in_deg = self.lay["ind"]

    def steps(self, u):
        return self.st_par[self.st_off[u]:self.st_off[u + 1]], self.st_eid[self.st_off[u]:self.st_off[u + 1]]

    def back_reach(self, t):
        seen, q = {t}, [t]
        for u in q:
            for p in self.steps(u)[0].tolist():
                if p not in seen:
                    seen.add(p)
                    q.append(p)
        return seen

    def layer(self, prev):
        nxt = defaultdict(int)
        for u, c in prev.items():
            for w in self.e[self.v[u]:self.v[u + 1]].tolist():
                nxt[w] += c
        return dict(nxt)


def sat(x):
    return min(x, INT64_MAX)


def unrank(g, lay, s, t, h, r, rec, admit=None):
    """Walk r (exact rank) of the h-edge walks s -> t, whose w_j are lay[j] -> [s, e1, v1, ..., t].  Appends the work
    of every step to rec.  admit (optional): per step-list entry, whether the walk may take it; an entry it refuses
    stays in its in-list as a zero term."""
    out = [0] * (2 * h + 1)
    out[-1] = t
    if h == 0:
        out[0] = s
    cur = t
    for k in range(h, 0, -1):
        par, eid = g.steps(cur)
        o = int(g.st_off[cur])
        terms = [lay[k - 1].get(p, 0) if admit is None or admit[o + i] else 0 for i, p in enumerate(par.tolist())]
        pre, j = 0, None
        for i, x in enumerate(terms):
            if pre + x > r:
                j = i
                break
            pre += x
        assert j is not None, (cur, k, r)
        w = j // WINDOW
        wstart = sum(terms[:w * WINDOW])
        win = terms[w * WINDOW:(w + 1) * WINDOW]
        inclusive = np.cumsum([0] + [int(x) for x in win], dtype=object)[1:]
        rec.append(dict(
            vertex=cur, k=k, deg=len(terms), j=j, window=w, key=int(g.perm[cur]) * g.n + int(par[j]),
            at_window_end=w > 0 and wstart == r,
            sat_after_pick=any(int(x) >= INT64_MAX for x in inclusive[j - w * WINDOW + 1:])))
        r -= pre
        out[2 * k - 1] = int(eid[j])
        out[2 * k - 2] = int(par[j])
        cur = int(par[j])
    return out


def walk_layers(g, s, t, stop):
    """w_0 .. w_H from s, H the first layer where stop(h, count at t, w_h) holds -> (layers, counts at t)"""
    lay, counts, h = [{s: 1}], [1 if s == t else 0], 0
    if stop(0, counts[0], lay[0]):
        return lay, counts
    while True:
        h += 1
        lay.append(g.layer(lay[-1]))
        counts.append(lay[h].get(t, 0))
        if stop(h, counts[h], lay[h]):
            return lay, counts
        if h > WALK_MAX:
            raise Unsupported("walk past the limit")


def as_row(g, s, t, max_paths):
    """all_shortest_paths of one row -> dict(count (exact), h, lists, work)"""
    if s == t:
        return dict(count=1, h=0, lists=[[s]], work=[], lay=[{s: 1}])
    if s not in g.back_reach(t):
        return dict(count=0, h=-1, lists=None, work=[], lay=[{s: 1}])
    lay, counts = walk_layers(g, s, t, lambda h, c, w: c > 0 or not w)
    if counts[-1] == 0:
        return dict(count=0, h=-1, lists=None, work=[], lay=lay)
    h, c = len(counts) - 1, counts[-1]
    np_ = min(sat(c), max_paths) if max_paths else sat(c)
    if max_paths == 0 and c >= INT64_MAX:
        raise Unsupported("saturated count")
    if np_ * (2 * h + 1) > INT64_MAX // 8:
        raise TooLarge("elements")
    work = []
    return dict(count=c, h=h, lists=[unrank(g, lay, s, t, h, r, work) for r in range(np_)], work=work, lay=lay)


def kwalk_row(g, s, t, k, groups=False, max_paths=0):
    """shortest_k_paths (groups False) or WALK's shortest_k_groups of one row -> dict(lengths with their counts, walks,
    ranks' length work, the stop layer, groups outputs)"""
    B = g.back_reach(t)
    res = dict(valid=s in B, walks=None, counts=[], stop=0, count=0, ngroups=0, last=-1, npaths=0, work=[], lens=[],
               lay=[{s: 1}], B=B)
    if s not in B:
        res["complete"] = 1
        return res
    state = dict(total=0, groups=0)

    def stop(h, c, w):
        if groups:
            if c:
                state["groups"] += 1
            return state["groups"] >= k or (h > 0 and not any(u in B for u in w))
        state["total"] += min(c, k - state["total"])
        return state["total"] >= k or (h > 0 and not any(u in B for u in w))

    lay, counts = walk_layers(g, s, t, stop)
    res.update(lay=lay, counts=counts, stop=len(counts) - 1)
    # listed walks per length
    wants, listed = [], 0
    for h, c in enumerate(counts):
        if groups:
            want = min(c, max_paths - listed) if max_paths else c
        else:
            want = min(c, k - listed)
        wants.append(want)
        listed += want
    if groups:
        glen = [h for h, c in enumerate(counts) if c]
        res.update(count=sat(sum(counts)), ngroups=len(glen), last=glen[-1] if glen else -1)
        if max_paths == 0 and sum(counts) >= INT64_MAX:
            raise Unsupported("saturated count")
        if any(w * (2 * h + 1) > INT64_MAX // 8 for h, w in enumerate(wants)):
            raise TooLarge("elements")
        res["complete"] = int(listed == res["count"])
    res["npaths"] = listed
    walks, before = [], 0
    for h, want in enumerate(wants):
        for r in range(want):
            walks.append(unrank(g, lay, s, t, h, r, res["work"]))
            res["lens"].append(dict(h=h, rank=before + r, window=h // WINDOW,
                                    zero_window=any(not any(counts[x * WINDOW:(x + 1) * WINDOW])
                                                    for x in range(h // WINDOW)),
                                    starts_zero=h >= WINDOW and counts[h // WINDOW * WINDOW] == 0,
                                    carry_e=h >= WINDOW and any(wants[:h // WINDOW * WINDOW])))
        before += want
    res["walks"] = walks if walks else None
    if not walks:
        res["valid"] = False
    return res


def chunk_work(g, lay, B, H, in_adj=None, admit=None):
    """Per layer 1..H, the in-lists of the rows of B (internal ids) that span more than one chunk: their parts.
    in_adj (optional): the in-lists walked, internal parent ids by in-CSC position (g.in_adj by default); admit
    (optional): per position, whether its edge counts."""
    out = []
    inv = g.lay["inv"]
    if in_adj is None:
        in_adj = g.in_adj

    def part(a, b, prev):
        return sum(prev.get(int(inv[p]), 0) for i, p in enumerate(in_adj[a:b].tolist(), a)
                   if admit is None or admit[i])
    for u_int in range(g.n_ab):
        rs, re_ = int(g.in_off[u_int]), int(g.in_off[u_int + 1])
        u = int(inv[u_int])
        if u not in B:
            continue
        for h in range(1, H + 1):
            prev = lay[h - 1]
            if rs // CHUNK == (re_ - 1) // CHUNK:
                total = part(rs, re_, prev)
                out.append(dict(u=u_int, h=h, split=False, parts=[total], rs=rs, re=re_, middle=False))
                continue
            parts, middle = [], False
            for c0 in range(rs // CHUNK * CHUNK, re_, CHUNK):
                a, b = max(rs, c0), min(re_, c0 + CHUNK)
                parts.append(part(a, b, prev))
                middle |= rs < c0 and re_ > c0 + CHUNK
            out.append(dict(u=u_int, h=h, split=True, parts=parts, rs=rs, re=re_, middle=middle))
    return out


def layer_bytes(h, rows, n_ab):
    return (h + 1) * n_ab * rows * 8


def store_groups(rows, W, budget, n_ab):
    """ks_run's greedy packing: rows = [(lane, last length)] of the rows with walks in lane order -> [(lanes, H)]"""
    groups, grp, gh = [], [], 0
    for ln, h in rows:
        if layer_bytes(h, 1, n_ab) > budget:
            raise Unsupported("over the layer budget")
        if grp and (len(grp) == W or layer_bytes(max(gh, h), len(grp) + 1, n_ab) > budget):
            groups.append((grp, gh))
            grp, gh = [], 0
        grp.append(ln)
        gh = max(gh, h)
    if grp:
        groups.append((grp, gh))
    return groups


def store_launches(groups):
    return sum(2 + h for _, h in groups)


def ks_width(S, n_ab):
    w = KS_WIDTH
    while w > 64 and 2 * max(n_ab, 1) * w * 8 > (4 << 30):
        w >>= 1
    while w > 64 and S <= w // 2:
        w >>= 1
    return w


# ---- the catalogue -----------------------------------------------------------------------------------------------------
class Builder:
    def __init__(self, n=0):
        self.n, self.src, self.dst = n, [], []

    def new(self, k=1):
        self.n += k
        return self.n - k if k == 1 else list(range(self.n - k, self.n))

    def edge(self, a, b, mult=1):
        self.src += [a] * mult
        self.dst += [b] * mult

    def chain(self, a, length, b=None):
        """a -> ... -> b over `length` edges (new inner vertices; a new end when b is None) -> the end"""
        cur = a
        for i in range(length):
            nxt = (self.new() if b is None else b) if i == length - 1 else self.new()
            self.edge(cur, nxt)
            cur = nxt
        return cur


FAN_IN = (31, 32, 33, 63, 64, 65, 96, 97)


def case_fan_in():
    """One hub per in-degree of FAN_IN, each behind its own out-only source: s -> parent (sigma(parent) parallel
    edges, 1 to 3) -> hub, parent i with i + 1 more edges into a sink so that the device numbers the parents opposite
    to their original ids.  Every rank is listed, so some rank's prefix ends exactly at a window end."""
    b = Builder()
    rows = []
    for d in FAN_IN:
        s, hub, sink = b.new(), b.new(), b.new()
        for i in range(d):
            p = b.new()
            b.edge(s, p, 1 + (i * 7 + d) % 3)
            b.edge(p, hub)
            b.edge(p, sink, i + 1)
        rows.append((s, hub))
    return dict(n=b.n, src=b.src, dst=b.dst, rows=rows, mps=(0, 5), ks=(300,), kgs=((1, 0), (2, 7)),
                named={"as_pick_window_1", "as_pick_window_2", "as_pick_window_3", "as_prefix_eq_r_window_end",
                       "ks_pick_window_1", "ks_pick_window_2", "ks_pick_window_3", "ks_prefix_eq_r_window_end",
                       "source_out_only", "reach_list_crosses_warp_base", "chunk_plain_store",
                       *{f"fan_in_{d}" for d in FAN_IN}})


def binary_counter_parts(b, D=126):
    """diamonds(62) from x_0 = 0: x_i = 3i has 2^i paths of 2i edges.  -> tail(i, t): a disjoint chain of D - 2i edges
    from x_i to t, so that every path x_0 -> t has D edges"""
    n, src, dst = diamonds(62)
    b.n = n
    b.src, b.dst = src.tolist(), dst.tolist()
    return lambda i, t: b.chain(3 * i, D - 2 * i, t)


def case_binary_counter():
    """The count x_0 -> t is the sum of 2^i over the chosen x_i: 2^63 - 2 (i = 1 .. 62), 2^63 - 1 (i = 0 .. 62), and a
    saturated one: x_0's tail, then x_62 -> y twice (sigma(y) = 2^63) and y's tail, so that the prefix after the first
    in-edge of t3 (rank 0) saturates inside its window"""
    b = Builder()
    tail = binary_counter_parts(b)
    t1, t2, t3 = b.new(), b.new(), b.new()
    for i in range(1, 63):
        tail(i, t1)
    for i in range(63):
        tail(i, t2)
    tail(0, t3)
    y = b.new()
    b.edge(3 * 62, y, 2)
    b.edge(y, t3)  # (y is 125 edges from x_0)
    return dict(n=b.n, src=b.src, dst=b.dst, rows=[(0, t1), (0, t2), (0, t3), (0, 186)], mps=(5,), ks=(5,),
                kgs=((1, 5), (2, 3)), named={"count_int64_max_minus_1", "count_int64_max", "count_saturated",
                                             "as_sat_after_pick", "ks_sat_after_pick", "len_zero_window"})


CHUNK_HUBS = [(d, rho) for d in (127, 128, 129, 255, 256, 257, 385) for rho in (0, 1, 127)]


def case_chunks():
    """In-lists of 127 .. 385 edges starting at in-CSC offsets = 0, 1 and 127 (mod 128).  The hubs and the fillers
    before them (whose in-degrees set the offsets) lead the internal order through their out-degrees (edges into one
    sink); every hub parent has one in-edge, from the hub's source s for the parents in even chunk parts and from a
    second source s2 for the odd ones, so that a row meets zero parts next to non-zero ones.  A last hub of 256
    parents at 2^55 paths each (behind diamonds(55)) has two exact chunk parts of 2^62 whose sum saturates.  The first
    hub is internal row 0; a vertex with one in-edge from it is row n_ab - 1."""
    b = Builder()
    plan, off = [], 0
    for d, rho in CHUNK_HUBS + [(256, 0)]:
        a = (rho - off) % CHUNK
        if a:
            plan.append(("filler", a))
            off += a
        plan.append(("hub", d, off))
        off += d
    # the diamonds of the saturating hub first, so that their ids stay those of diamonds(55)
    dn, dsrc, dst_ = diamonds(55)
    b.n, b.src, b.dst = dn, dsrc.tolist(), dst_.tolist()
    rows, heads = [], []
    for j, item in enumerate(plan):
        if item[0] == "filler":
            v, g = b.new(), b.new()
            b.edge(g, v, item[1])
            heads.append(v)
            continue
        _, d, start = item
        hub = b.new()
        heads.append(hub)
        if j == len(plan) - 1:
            for _ in range(d):
                p = b.new()
                b.edge(3 * 55, p)
                b.edge(p, hub)
            rows.append((0, hub))
            continue
        s, s2 = b.new(), b.new()
        for i in range(d):
            p = b.new()
            b.edge(s if ((start + i) // CHUNK - start // CHUNK) % 2 == 0 else s2, p)
            b.edge(p, hub)
        rows.append((s, hub))
        if (start + d - 1) // CHUNK > start // CHUNK:
            rows.append((s2, hub))
    last = b.new()
    b.edge(heads[0], last)
    z = b.new()
    outd = np.bincount(np.asarray(b.src), minlength=b.n)
    base = int(outd.max()) + len(heads) + 1
    for j, v in enumerate(heads):  # descending out-degrees: the plan's order is the internal order
        b.edge(v, z, base - j - int(outd[v]))
    rows.append((rows[0][0], last))
    return dict(n=b.n, src=b.src, dst=b.dst, rows=rows, mps=(0, 3), ks=(3,), kgs=((1, 3),), plan=plan,
                named={"target_row_0", "target_row_last", "source_out_only", "chunk_plain_store", "chunk_split_nonzero",
                       "chunk_middle_inside", "chunk_parts_exact_sum_saturates", "chunk_zero_part_next_to_nonzero",
                       "reach_list_crosses_warp_base", "ks_pick_window_3",
                       *{f"chunk_len_{d}_at_{rho}" for d, rho in CHUNK_HUBS}})


def case_long_walks():
    """a chain of 30 edges into a self-loop at its end (walks of every length from 30 on); a chain of 33 edges into a
    2-cycle (walks of 33, 35, ...: the first window holds only zeros, the second starts with one); a chain of 31 edges
    into a 2-cycle (31, 33, ...: the walks cross 31/32 over a zero at 32); s == t on the self-loop and the 2-cycles"""
    b = Builder()
    a0 = b.new()
    a = b.chain(a0, 30)
    b.edge(a, a)
    b0 = b.new()
    bt = b.chain(b0, 33)
    bb = b.new()
    b.edge(bt, bb)
    b.edge(bb, bt)
    c0 = b.new()
    ct = b.chain(c0, 31)
    cc = b.new()
    b.edge(ct, cc)
    b.edge(cc, ct)
    return dict(n=b.n, src=b.src, dst=b.dst, rows=[(a0, a), (b0, bt), (c0, ct), (a, a), (ct, ct)], mps=(0,), ks=(40,),
                kgs=((2, 0), (3, 0), (40, 0), (40, 45)), small=True,
                named={"len_cross_31_32", "len_cross_63_64", "len_zero_window", "len_window_starts_zero", "len_carry_e",
                       "kg_s_eq_t_stop"})


LANE_ROWS = 520
GROUP_SIZES = (1, 31, 32, 33, 64, 65)


def case_lanes():
    """LANE_ROWS rows on private chains of 1, 2 or 3 edges (row l: 1 + l % 3), each from its own source: every vertex
    has one active lane, rows sit on every lane of a 512-lane batch, and with k = 1 a lane that stopped sits next to one
    that counts on in the same 64-bit word"""
    b = Builder()
    rows = []
    for lane in range(LANE_ROWS):
        s = b.new()
        rows.append((s, b.chain(s, 1 + lane % 3)))
    return dict(n=b.n, src=b.src, dst=b.dst, rows=rows, mps=(0,), ks=(1, 2), kgs=((1, 0),), as_lanes=(64, 128, 256, 512),
                budgets=GROUP_SIZES,
                named={"ks_stopped_next_to_counting", "store_group_W", *{f"ks_lane_{x}" for x in (0, 31, 32, 63, 64, 127, 511)},
                       "sigma_only_lane_32", *{f"sigma_only_lane_last_{w}" for w in (64, 128, 256, 512)},
                       *{f"store_group_{x}" for x in GROUP_SIZES}})


def case_two_batches():
    """64 rows on single edges, then 64 rows each behind its own diamonds(6) (64 paths of 12 edges): with 64 lanes the
    second BFS batch writes ~500x the elements of the first, so the walk buffer grows under the first batch's lists"""
    b = Builder()
    rows = []
    for _ in range(64):
        s = b.new()
        rows.append((s, b.chain(s, 1)))
    for _ in range(64):
        dn, ds, dd = diamonds(6)
        base = b.new(dn)[0]
        for x, y in zip(ds.tolist(), dd.tolist()):
            b.edge(base + x, base + y)
        rows.append((base, base + dn - 1))
    return dict(n=b.n, src=b.src, dst=b.dst, rows=rows, mps=(0,), ks=(3,), kgs=((1, 0),), as_options=64,
                named={"as_walk_grows"})


def case_wide_keys():
    """a cycle over n = 65537 vertices: every vertex has an in-edge and the internal order is the original one, so the
    step keys u * n + parent of the top rows need bit 32"""
    n = 65537
    return dict(n=n, src=list(range(n)), dst=[(i + 1) % n for i in range(n)],
                rows=[(65530, 65536), (65535, 1), (65536, 0)], mps=(0,), ks=(1,), kgs=((1, 0),),
                named={"step_key_bit_32"})


def case_n1():
    return dict(n=1, src=[0, 0], dst=[0, 0], rows=[(0, 0)], mps=(0, 2), ks=(1, 4), kgs=((2, 0), (3, 5)), small=True,
                named={"n_1", "kg_s_eq_t_stop"})


def case_n2():
    return dict(n=2, src=[0, 1, 1], dst=[1, 0, 1], rows=[(0, 1), (1, 0), (1, 1), (0, 0)], mps=(0, 1), ks=(1, 5),
                kgs=((2, 0), (3, 2)), small=True, named={"n_2"})


CATALOGUE = {
    "fan_in": case_fan_in,
    "binary_counter": case_binary_counter,
    "chunks": case_chunks,
    "long_walks": case_long_walks,
    "lanes": case_lanes,
    "two_batches": case_two_batches,
    "wide_keys": case_wide_keys,
    "n1": case_n1,
    "n2": case_n2,
}

REQUIRED = (
    {f"{f}_pick_window_{w}" for f in ("as", "ks") for w in (1, 2, 3)}
    | {"as_prefix_eq_r_window_end", "ks_prefix_eq_r_window_end", "as_sat_after_pick", "ks_sat_after_pick"}
    | {"len_cross_31_32", "len_cross_63_64", "len_zero_window", "len_window_starts_zero", "len_carry_e"}
    | {f"chunk_len_{d}_at_{rho}" for d, rho in CHUNK_HUBS}
    | {"chunk_plain_store", "chunk_split_nonzero", "chunk_middle_inside", "chunk_parts_exact_sum_saturates",
       "chunk_zero_part_next_to_nonzero", "reach_list_crosses_warp_base"}
    | {"sigma_only_lane_32"} | {f"sigma_only_lane_last_{w}" for w in (64, 128, 256, 512)}
    | {"source_out_only", "target_row_0", "target_row_last", "step_key_bit_32", "n_1", "n_2"}
    | {"count_int64_max_minus_1", "count_int64_max", "count_saturated"}
    | {f"store_group_{x}" for x in GROUP_SIZES} | {"store_group_W"}
    | {f"ks_lane_{x}" for x in (0, 31, 32, 63, 64, 127, 511)} | {"ks_stopped_next_to_counting", "kg_s_eq_t_stop"}
    | {"as_walk_grows"} | {f"fan_in_{d}" for d in FAN_IN}
)


@lru_cache(maxsize=None)
def case(name):
    c = CATALOGUE[name]()
    c["g"] = Graph(c["n"], c["src"], c["dst"])
    c["ps"] = np.array([s for s, _ in c["rows"]], np.int64)
    c["pd"] = np.array([t for _, t in c["rows"]], np.int64)
    return c


def _restate(fn, *args):
    try:
        return fn(*args)
    except Unsupported:
        return "unsupported"
    except TooLarge:
        return "too_large"


@lru_cache(maxsize=None)
def restated(name):
    """every query of the case, restated: ('as', mp) -> rows, ('ks', k) -> rows, ('kg', k, mp) -> rows"""
    c = case(name)
    g = c["g"]
    out = {}
    for mp in c["mps"]:
        out[("as", mp)] = [_restate(as_row, g, s, t, mp) for s, t in c["rows"]]
    for k in c["ks"]:
        out[("ks", k)] = [kwalk_row(g, s, t, k) for s, t in c["rows"]]
    for k, mp in c["kgs"]:
        out[("kg", k, mp)] = [_restate(kwalk_row, g, s, t, k, True, mp) for s, t in c["rows"]]
    return out


def as_lane_batches(c, L):
    """all_shortest_paths' lanes: one per distinct source in first-appearance order, L per batch"""
    srcs = list(dict.fromkeys(s for s, t in c["rows"] if s != t))
    return [srcs[i:i + L] for i in range(0, len(srcs), L)]


def case_hits(name):
    c, res = case(name), restated(name)
    g = c["g"]
    hits = set()
    for key, rows in res.items():
        fam = key[0]
        for (s, t), r in zip(c["rows"], rows):
            if isinstance(r, str):
                continue
            for w in r["work"]:
                if 1 <= w["window"] <= 3:
                    hits.add(f"{'as' if fam == 'as' else 'ks'}_pick_window_{w['window']}")
                if w["at_window_end"]:
                    hits.add(f"{'as' if fam == 'as' else 'ks'}_prefix_eq_r_window_end")
                if w["sat_after_pick"]:
                    hits.add(f"{'as' if fam == 'as' else 'ks'}_sat_after_pick")
                if w["key"] >= 1 << 32:
                    hits.add("step_key_bit_32")
            if fam == "as":
                if r["count"] == INT64_MAX - 1:
                    hits.add("count_int64_max_minus_1")
                if r["count"] == INT64_MAX:
                    hits.add("count_int64_max")
                if r["count"] > INT64_MAX:
                    hits.add("count_saturated")
                continue
            lens = [x["h"] for x in r["lens"]]
            if any(h <= 31 for h in lens) and any(h >= 32 for h in lens):
                hits.add("len_cross_31_32")
            if any(h <= 63 for h in lens) and any(h >= 64 for h in lens):
                hits.add("len_cross_63_64")
            for x in r["lens"]:
                for flag in ("zero_window", "starts_zero", "carry_e"):
                    if x[flag]:
                        hits.add({"zero_window": "len_zero_window", "starts_zero": "len_window_starts_zero",
                                  "carry_e": "len_carry_e"}[flag])
            if not r["valid"]:
                continue
            if g.in_deg[s] == 0 and s != t:
                hits.add("source_out_only")
            if g.perm[t] == 0:
                hits.add("target_row_0")
            if g.perm[t] == g.n_ab - 1:
                hits.add("target_row_last")
            if fam == "kg" and s == t and key[1] >= 2 and r["ngroups"] == key[1] and \
                    any(g.layer(r["lay"][-1]).get(u, 0) for u in r["B"]):
                hits.add("kg_s_eq_t_stop")  # it stops at its k-th group, counting h = 0, while longer walks exist
            for u in r["B"]:
                ui = int(g.perm[u])
                if ui < g.n_ab:
                    rs, re_ = int(g.in_off[ui]), int(g.in_off[ui + 1])
                    if rs % 32 and (re_ - 1) // 32 > rs // 32:
                        hits.add("reach_list_crosses_warp_base")
            for w in chunk_work(g, r["lay"], r["B"], r["stop"]):
                ln = w["re"] - w["rs"]
                if any(w["parts"]):
                    if ln in (127, 128, 129, 255, 256, 257, 385) and w["rs"] % CHUNK in (0, 1, 127):
                        hits.add(f"chunk_len_{ln}_at_{w['rs'] % CHUNK}")
                    hits.add("chunk_split_nonzero" if w["split"] else "chunk_plain_store")
                if w["split"]:
                    p = w["parts"]
                    if w["middle"]:
                        hits.add("chunk_middle_inside")
                    if all(x < INT64_MAX for x in p) and sum(p) >= INT64_MAX:
                        hits.add("chunk_parts_exact_sum_saturates")
                    if any(p[i] == 0 and (p[i - 1] if i else 0) + (p[i + 1] if i + 1 < len(p) else 0)
                           for i in range(len(p))):
                        hits.add("chunk_zero_part_next_to_nonzero")
    # ks lanes: rows in input order, one batch of ks_width lanes
    for k in c["ks"]:
        rows = res[("ks", k)]
        W = ks_width(len(rows), g.n_ab)
        if W == KS_WIDTH and len(rows) >= KS_WIDTH:
            hits |= {f"ks_lane_{x}" for x in (0, 31, 32, 63, 64, 127, 511)}
        stops = [r["stop"] if r["valid"] or r["counts"] else None for r in rows[:W]]
        for word in range(0, min(W, len(rows)), 64):
            st = [x for x in stops[word:word + 64] if x is not None]
            if st and min(st) >= 1 and max(st) > min(st):
                hits.add("ks_stopped_next_to_counting")
        with_walks = [(ln, max(x["h"] for x in r["lens"])) for ln, r in enumerate(rows) if r["walks"]]
        if with_walks:
            if any(len(gr) == W for gr, _ in store_groups(with_walks, W, 4 << 30, g.n_ab)):
                hits.add("store_group_W")
            for size in c.get("budgets", ()):
                groups = store_groups(with_walks, W, group_budget(with_walks, size, g.n_ab), g.n_ab)
                if len(groups[0][0]) == size:
                    hits.add(f"store_group_{size}")
    # sigma lanes: at some (vertex, level) only lane 32 or only lane L - 1 of the batch is active
    for L in c.get("as_lanes", ()):
        for batch in as_lane_batches(c, L):
            active = defaultdict(set)
            for lane, s in enumerate(batch):
                dist = {s: 0}
                q = [s]
                for u in q:
                    for w in g.e[g.v[u]:g.v[u + 1]].tolist():
                        if w not in dist:
                            dist[w] = dist[u] + 1
                            q.append(w)
                for u, d in dist.items():
                    if d >= 1:
                        active[(u, d)].add(lane)
            for lanes in active.values():
                if lanes == {32}:
                    hits.add("sigma_only_lane_32")
                if lanes == {L - 1}:
                    hits.add(f"sigma_only_lane_last_{L}")
    # the walk buffer: a later BFS batch writes many more elements than the first
    if c.get("as_options"):
        L = c["as_options"]
        rows = res[("as", c["mps"][0])]
        by_src = {s: i for i, s in enumerate(dict.fromkeys(s for s, t in c["rows"] if s != t))}
        tot = defaultdict(int)
        for (s, t), r in zip(c["rows"], rows):
            if not isinstance(r, str) and r["lists"] and s != t:
                tot[by_src[s] // L] += len(r["lists"]) * (2 * r["h"] + 1)
        if len(tot) >= 2 and tot[1] > 100 * tot[0]:
            hits.add("as_walk_grows")
    if name == "fan_in":
        for d in FAN_IN:
            if np.any(g.in_deg == d):
                hits.add(f"fan_in_{d}")
    if g.n in (1, 2) and len(g.e):
        hits.add(f"n_{g.n}")
    return hits


def group_budget(rows, size, n_ab):
    """the layer budget under which ks_run's first storing group closes at exactly `size` rows (when the rows' longest
    walk is among the first three)"""
    return layer_bytes(max(h for _, h in rows), size, n_ab)


# ---- CPU: the hits, the coverage, the oracles against the restatement ------------------------------------------------
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_catalogue_hits_its_boundaries(name):
    hits = case_hits(name)
    missing = case(name)["named"] - hits
    assert not missing, sorted(missing)


def test_catalogue_covers_every_boundary():
    named = set().union(*(case(x)["named"] for x in CATALOGUE))
    assert REQUIRED <= named, sorted(REQUIRED - named)
    assert named <= REQUIRED, sorted(named - REQUIRED)


def test_chunk_hubs_sit_where_planned():
    c = case("chunks")
    g = c["g"]
    hubs = [item for item in c["plan"] if item[0] == "hub"]
    starts = {int(g.in_off[u]): int(g.in_off[u + 1] - g.in_off[u]) for u in range(g.n_ab)}
    for _, d, start in hubs:
        assert starts.get(start) == d, (d, start)
    assert g.perm[c["rows"][0][1]] == 0 and g.perm[c["rows"][-1][1]] == g.n_ab - 1


def oracle_rows(name, key):
    c = case(name)
    g = c["g"]
    if key[0] == "as":
        return oas.all_shortest_paths(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], key[1])
    if key[0] == "ks":
        return oks.shortest_k_paths(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], key[1])
    return okg.shortest_k_groups(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], key[1], key[2], "WALK")


def expect_error(rows):
    """the error a call over these restated rows raises (the first row that fails), or None"""
    for r in rows:
        if isinstance(r, str):
            return r
    return None


ORACLE_CODE = {"unsupported": oas.ERR_UNSUPPORTED, "too_large": orc.ORC_ERR_ALLOC}
DEVICE_CODE = {"unsupported": PGQ_ERR_UNSUPPORTED, "too_large": PGQ_ERR_OOM}


@pytest.mark.parametrize("name", list(CATALOGUE))
def test_oracles_equal_the_restatement(name):
    c = case(name)
    for key, rows in restated(name).items():
        err = expect_error(rows)
        if err:
            with pytest.raises(orc.OracleError) as ex:
                oracle_rows(name, key)
            assert ex.value.code == ORACLE_CODE[err], key
            continue
        if key[0] == "as":
            paths, cnt = oracle_rows(name, key)
            assert cnt.tolist() == [sat(r["count"]) for r in rows], key
            assert paths == [r["lists"] for r in rows], key
            ccnt, cvalid = oas.shortest_path_count(c["n"], c["g"].v, c["g"].e, c["g"].ids, c["ps"], c["pd"])
            assert ccnt.tolist() == [sat(r["count"]) for r in rows]
            assert cvalid.tolist() == [int(r["count"] > 0) for r in rows]
        elif key[0] == "ks":
            paths, npaths, _ = oracle_rows(name, key)
            assert paths == [r["walks"] for r in rows], key
            assert npaths.tolist() == [r["npaths"] for r in rows], key
        else:
            paths, orows, _ = oracle_rows(name, key)
            assert paths == [r["walks"] for r in rows], key
            for field, mine in (("count", "count"), ("ngroups", "ngroups"), ("last_len", "last"),
                                ("complete", "complete"), ("npaths", "npaths")):
                assert orows[field].tolist() == [r[mine] for r in rows], (key, field)


@pytest.mark.parametrize("name", [x for x in CATALOGUE if CATALOGUE[x]().get("small")])
def test_small_cases_are_the_brute_force_walks(name):
    c = case(name)
    g = c["g"]
    for k in c["ks"]:
        for (s, t), r in zip(c["rows"], restated(name)[("ks", k)]):
            hmax = max((x["h"] for x in r["lens"]), default=0)
            exp = brute_walks(g.n, g.v, g.e, g.ids, s, t, hmax)[:k]
            assert (r["walks"] or []) == exp, (s, t, k)
            assert [sat(x) for x in r["counts"]] == length_counts(g.n, g.v, g.e, s, t, len(r["counts"]) - 1)


def test_saturation_error_codes():
    """max_paths = 0: 2^63 - 2 paths are exact but their elements cannot be held (refused for the total); 2^63 - 1 is
    taken as saturated (UNSUPPORTED); both oracles agree"""
    c = case("binary_counter")
    g = c["g"]
    for t, code in ((c["rows"][0][1], orc.ORC_ERR_ALLOC), (c["rows"][1][1], oas.ERR_UNSUPPORTED),
                    (c["rows"][2][1], oas.ERR_UNSUPPORTED)):
        with pytest.raises(orc.OracleError) as ex:
            oas.all_shortest_paths(g.n, g.v, g.e, g.ids, [0], [t], 0)
        assert ex.value.code == code
        with pytest.raises(orc.OracleError) as ex:
            okg.shortest_k_groups(g.n, g.v, g.e, g.ids, [0], [t], 1, 0, "WALK")
        assert ex.value.code == code
        assert expect_error([_restate(as_row, g, 0, t, 0)]) == {orc.ORC_ERR_ALLOC: "too_large"}.get(code, "unsupported")
    cnt, _ = oas.shortest_path_count(g.n, g.v, g.e, g.ids, [0] * 3, [t for _, t in c["rows"][:3]])
    assert cnt.tolist() == [INT64_MAX - 1, INT64_MAX, INT64_MAX]


# ---- GPU: the device against the oracle ------------------------------------------------------------------------------
def compare_all(csr, name, options=None, keys=None, as_options=None):
    """every query of the case on the device against the oracle; -> {key: stats}"""
    c = case(name)
    g = c["g"]
    stats = {}
    as_opt = as_options or options or (pgq.Options(c["as_options"]) if c.get("as_options") else None)
    for key, rows in restated(name).items():
        if keys is not None and key not in keys:
            continue
        err = expect_error(rows)
        if key[0] == "as":
            cnt, valid, sst = csr.shortest_path_count(c["ps"], c["pd"], None, None, as_opt)
            ocnt, ovalid = oas.shortest_path_count(g.n, g.v, g.e, g.ids, c["ps"], c["pd"])
            assert np.array_equal(cnt, ocnt) and np.array_equal(valid, ovalid), key
            if err:
                with pytest.raises(pgq.PgqError) as ex:
                    csr.all_shortest_paths(c["ps"], c["pd"], key[1], None, None, as_opt)
                assert ex.value.status == DEVICE_CODE[err], key
                continue
            paths, dcnt, st = csr.all_shortest_paths(c["ps"], c["pd"], key[1], None, None, as_opt)
            opaths, _ = oracle_rows(name, key)
            assert np.array_equal(dcnt, ocnt) and paths == opaths, key
            assert {x: st[x] for x in BFS_COUNTERS} == {x: sst[x] for x in BFS_COUNTERS}
            stats[key] = st
        elif key[0] == "ks":
            paths, npaths, st = csr.shortest_k_paths(c["ps"], c["pd"], key[1], None, None, options)
            opaths, onp, ost = oks.shortest_k_paths(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], key[1], None, None,
                                                    st["lanes"])
            assert np.array_equal(npaths, onp) and paths == opaths, key
            assert {x: st[x] for x in KS_COUNTERS} == {x: ost[x] for x in KS_COUNTERS}, key
            stats[key] = st
        else:
            k, mp = key[1], key[2]
            ccnt, cng, clast, cvalid, cst = csr.shortest_k_groups_count(c["ps"], c["pd"], k, None, None, options)
            _, orows, ost = okg.shortest_k_groups(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], k, 0, "WALK", None, None,
                                                  cst["lanes"], count_only=True)
            assert np.array_equal(ccnt, orows["count"]) and np.array_equal(cng, orows["ngroups"])
            assert np.array_equal(clast, orows["last_len"])
            if err:
                with pytest.raises(pgq.PgqError) as ex:
                    csr.shortest_k_groups(c["ps"], c["pd"], k, mp, None, None, options, "WALK")
                assert ex.value.status == DEVICE_CODE[err], key
                continue
            paths, cnt, ng, last, comp, st = csr.shortest_k_groups(c["ps"], c["pd"], k, mp, None, None, options, "WALK")
            opaths, orows, ost = okg.shortest_k_groups(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], k, mp, "WALK", None,
                                                       None, st["lanes"])
            assert paths == opaths, key
            for x, y in ((cnt, "count"), (ng, "ngroups"), (last, "last_len"), (comp, "complete")):
                assert np.array_equal(x, orows[y]), (key, y)
            assert {x: st[x] for x in KS_COUNTERS} == {x: ost[x] for x in KS_COUNTERS}, key
            stats[key] = st
    return stats


def build(ctx, name):
    c = case(name)
    return pgq.DeviceCSR.build(ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_device_catalogue(gpu_ctx, name):
    csr = build(gpu_ctx, name)
    try:
        compare_all(csr, name)
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_saturation_errors(gpu_ctx):
    c = case("binary_counter")
    csr = build(gpu_ctx, "binary_counter")
    try:
        for t, status in ((c["rows"][0][1], PGQ_ERR_OOM), (c["rows"][1][1], PGQ_ERR_UNSUPPORTED),
                          (c["rows"][2][1], PGQ_ERR_UNSUPPORTED)):
            for call in (lambda: csr.all_shortest_paths([0], [t], 0), lambda: csr.shortest_k_groups([0], [t], 1, 0)):
                with pytest.raises(pgq.PgqError) as ex:
                    call()
                assert ex.value.status == status
        cnt, _, _ = csr.shortest_path_count([0] * 3, [t for _, t in c["rows"][:3]])
        assert cnt.tolist() == [INT64_MAX - 1, INT64_MAX, INT64_MAX]
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fan_in", "chunks", "lanes", "long_walks"])
def test_device_lane_widths_and_row_order(gpu_ctx, name):
    c = case(name)
    csr = build(gpu_ctx, name)
    try:
        for lanes in (64, 128, 256, 512):
            opt = pgq.Options(lanes)
            stats = compare_all(csr, name, options=opt, as_options=pgq.Options(lanes, no_prune=True))
            assert all(st["lanes"] == lanes for st in stats.values())
        perm = np.random.default_rng(7).permutation(len(c["ps"]))
        k = c["ks"][0]
        base = oks.shortest_k_paths(c["n"], c["g"].v, c["g"].e, c["g"].ids, c["ps"], c["pd"], k)[0]
        paths, _, _ = csr.shortest_k_paths(c["ps"][perm], c["pd"][perm], k)
        assert paths == [base[i] for i in perm]
        mp = c["mps"][-1]
        base, _ = oas.all_shortest_paths(c["n"], c["g"].v, c["g"].e, c["g"].ids, c["ps"], c["pd"], mp)
        paths, _, _ = csr.all_shortest_paths(c["ps"][perm], c["pd"][perm], mp)
        assert paths == [base[i] for i in perm]
    finally:
        csr.free()


LEVEL = re.compile(r"\[pgq\] batch (\d+) level (\d+) (push|pull|tail) ")


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["b", "p", "t", "bp", "pb", "tb"])
@pytest.mark.parametrize("name", ["fan_in", "chunks", "lanes", "two_batches"])
def test_device_forced_schedules(gpu_ctx, monkeypatch, capfd, name, schedule):
    """sigma needs every vertex at a level <= K recorded: forced bottom-up levels over the fan-in hubs must keep it"""
    csr = build(gpu_ctx, name)
    keys = [k for k in restated(name) if k[0] == "as"]
    try:
        monkeypatch.setenv("PGQ_B200_TRACE", "1")
        monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
        capfd.readouterr()
        compare_all(csr, name, keys=keys)
        lines = [LEVEL.match(x) for x in capfd.readouterr().err.splitlines()]
        kinds = [(int(x.group(2)), x.group(3)) for x in lines if x]
        assert kinds
        for level, kind in kinds:
            want = schedule[(level - 1) % len(schedule)]
            assert kind == {"b": "pull", "p": "push"}.get(want, kind) and (want == "t" or kind != "tail"), (level, kind)
            if want == "t":
                assert kind in ("tail", "push")
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("env", [("PGQ_B200_PULL_SKIP", "0"), ("PGQ_B200_NO_TAIL", "1")])
def test_device_bfs_switches(gpu_ctx, monkeypatch, env):
    csr = build(gpu_ctx, "fan_in")
    try:
        monkeypatch.setenv(*env)
        for schedule in ("b", "t", "tb"):
            monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
            compare_all(csr, "fan_in", keys=[k for k in restated("fan_in") if k[0] == "as"])
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_layer_budgets(gpu_ctx, monkeypatch):
    """budgets that close the first storing group at exactly 1, 31, 32, 33, 64 and 65 rows, and one byte below each;
    the launches of the storing pass follow the restated groups"""
    c = case("lanes")
    g = c["g"]
    csr = build(gpu_ctx, "lanes")
    try:
        k = 1
        key = ("ks", k)
        rows = restated("lanes")[key]
        with_walks = [(ln, max(x["h"] for x in r["lens"])) for ln, r in enumerate(rows) if r["walks"]]
        W = ks_width(len(rows), g.n_ab)
        base = compare_all(csr, "lanes", keys=[key])[key]
        base_groups = store_groups(with_walks, W, 4 << 30, g.n_ab)
        assert [len(x) for x, _ in base_groups] == [W, len(rows) - W]
        for size in GROUP_SIZES:
            for budget in (group_budget(with_walks, size, g.n_ab), group_budget(with_walks, size, g.n_ab) - 1):
                hmax = max(h for _, h in with_walks)
                if budget < layer_bytes(hmax, 1, g.n_ab):
                    monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(budget))
                    with pytest.raises(pgq.PgqError) as ex:
                        csr.shortest_k_paths(c["ps"], c["pd"], k)
                    assert ex.value.status == PGQ_ERR_UNSUPPORTED
                    continue
                groups = store_groups(with_walks, W, budget, g.n_ab)
                assert len(groups[0][0]) == (size if budget % 8 == 0 else size - 1), (size, budget)
                monkeypatch.setenv("PGQ_B200_KSP_LAYER_BUDGET", str(budget))
                st = compare_all(csr, "lanes", keys=[key])[key]
                assert st["kernel_launches"] - base["kernel_launches"] == \
                    store_launches(groups) - store_launches(base_groups), (size, budget)
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["device", "upload_noids", "chunked8", "i64_1"])
@pytest.mark.parametrize("name", ["fan_in", "chunks", "long_walks"])
def test_device_construction_routes(gpu_ctx, name, route):
    c = case(name)
    sh = Shape(c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64))
    csr, (v, e, ids, _), _ = make(gpu_ctx, sh, route)
    res = restated(name)
    try:
        ps, pd = c["ps"], c["pd"]
        cnt, valid, _ = csr.shortest_path_count(ps, pd)
        ocnt, ovalid = oas.shortest_path_count(c["n"], v, e, ids, ps, pd)
        assert np.array_equal(cnt, ocnt) and np.array_equal(valid, ovalid)
        for mp in c["mps"]:
            if expect_error(res[("as", mp)]):
                continue  # (the refusals: test_device_catalogue)
            paths, cnt, _ = csr.all_shortest_paths(ps, pd, mp)
            opaths, ocnt = oas.all_shortest_paths(c["n"], v, e, ids, ps, pd, mp)
            assert paths == opaths and np.array_equal(cnt, ocnt), mp
        for k in c["ks"]:
            paths, _, _ = csr.shortest_k_paths(ps, pd, k)
            assert paths == oks.shortest_k_paths(c["n"], v, e, ids, ps, pd, k)[0], k
        for k, mp in c["kgs"]:
            if expect_error(res[("kg", k, mp)]):
                continue
            paths, cnt, ng, last, comp, _ = csr.shortest_k_groups(ps, pd, k, mp)
            opaths, orows, _ = okg.shortest_k_groups(c["n"], v, e, ids, ps, pd, k, mp, "WALK")
            assert paths == opaths and np.array_equal(cnt, orows["count"]) and np.array_equal(ng, orows["ngroups"])
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_dirty_workspace(monkeypatch):
    """a context with one workspace: a larger call on another CSR first, then the three functions in turn, so that
    WS_AS_SIGMA, WS_WALK and WS_KS_* start out holding stale data"""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        for name, rounds in (("two_batches", 1), ("fan_in", 2), ("long_walks", 2), ("n2", 2), ("chunks", 2)):
            csr = build(ctx, name)
            try:  # (every CSR is freed before its context closes, whatever fails)
                for _ in range(rounds):
                    compare_all(csr, name)
            finally:
                csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_eight_threads(gpu_ctx):
    c = case("fan_in")
    g = c["g"]
    csr = build(gpu_ctx, "fan_in")
    exp = (oas.all_shortest_paths(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], 0)[0],
           oks.shortest_k_paths(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], 300)[0],
           okg.shortest_k_groups(g.n, g.v, g.e, g.ids, c["ps"], c["pd"], 2, 7, "WALK")[0])
    out = [None] * 8

    def work(i):
        out[i] = (csr.all_shortest_paths(c["ps"], c["pd"], 0)[0], csr.shortest_k_paths(c["ps"], c["pd"], 300)[0],
                  csr.shortest_k_groups(c["ps"], c["pd"], 2, 7)[0])

    ths = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert all(o == exp for o in out)
