"""cheapest_k_paths at the boundaries of its lane batches, bans, tight walk back and sentinels, against a restatement and
the oracle.

cheapest_k_paths (csrc/pgq_cheapest_k.cu) runs the k-path rounds of km_run (csrc/pgq_kpaths_modes.cu) over one
Bellman-Ford lane per spur search.  Its lanes are 32 .. 256 wide, addressed in 64-bit ban words (l >> 6) and walked in
32-lane groups; TRAIL's banned positions sit in a (position * 512 + lane) table filtered by word (km_ban_mask); the seed
test, the level-1 walk back and the in-list walk back are loops over 32-entry chunks; and every sum is tested against
the sentinel (BIGINT before the add, DOUBLE after its rounding).  So:

- a restatement in Python written from the header's construction and DESIGN.md section 3: Yen's rounds with Lawler's
  rule, each mode's spur range, the D lists and the vertex and edge bans, the admissible seeds, the Bellman-Ford fixed
  point in the weight type's arithmetic (Python floats are IEEE doubles; BIGINT is tested before the add), the tight
  BFS levels, the walk back over the step-ordered in-lists, and the pool keyed by (cost, h, steps).  It plans the
  batches (the lane cap from n, W per round, lanes in (row, j) order) and records its work: per spur its round, row, j,
  seed index, lane, word and group, tight depth and each walk-back pick; per batch W, cnt and the TRAIL key table.  It
  refuses what the device refuses: a tight depth past 65534, an accepted path past 65533 edges, a weight below zero;
- a catalogue whose cases each name the boundaries they hit, proven on the CPU from that record; a coverage test asks
  every boundary in REQUIRED to be hit, and no other;
- on the CPU, the C oracle (oracle/pgq_oracle_cheapest_k.c) equal to the restatement on every case, the small cases
  equal to the brute-force paths of test_cheapest_k_paths, costs non-decreasing and each the left-to-right fold of its
  weights (which holds under rounding too: a child's Lawler class is a subset of its parent's);
- on the GPU, the device equal to both on every case and mode, bit for bit in the costs, with the same batches,
  lanes, searches and push_levels; then forced widths and a row permutation, the lane cap at n = 2^20 and 2^20 + 1,
  the weighted construction routes, the identities with shortest_k_paths and cheapest_path, the refusals by status
  and message, a one-workspace context shared with shortest_k_paths, and eight threads on one CSR.

The number of Bellman-Ford sweeps of a call (stats levels) depends on the order of the parallel relaxations, so only
levels >= batches is asserted of it."""
import sys
import threading
from collections import deque
from fractions import Fraction
from functools import lru_cache

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from duckpgq_extension_b200.pgq import PGQ_ERR_UNSUPPORTED
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_cheapest as ocp
from oracle import pgq_oracle_cheapest_k as ock
from oracle.pgq_oracle import OracleError
from test_all_cheapest_boundaries import WBuilder, WGraph
from test_cheapest_k_paths import brute_paths

INT64_MAX = (1 << 63) - 1
S_I = INT64_MAX // 2                     # BF_INF_I64: the BIGINT sentinel
S_F = sys.float_info.max / 2             # BF_INF_F64: the DOUBLE sentinel
ULP_S_F = 2.0 ** 970                     # the spacing of the doubles at S_F
LEVEL_MAX = 65534                        # CK_LEVEL_MAX: the deepest tight level
PATH_MAX = 65533                         # KM_PATH_MAX: the longest accepted path
CK_BUDGET = 2 << 30                      # the distance array n x W x 8 bytes stays within this
MODES = ("WALK", "TRAIL", "ACYCLIC", "SIMPLE")
REFUSAL_TEXT = {"tight": "went beyond 65534 tight levels", "long": "needs a path longer than 65533 edges",
                "negative": "needs weights >= 0"}


# ---- the restatement ---------------------------------------------------------------------------------------------------
class Refused(Exception):
    def __init__(self, kind):
        super().__init__(REFUSAL_TEXT[kind])
        self.kind = kind


class Lists:
    """The CSR as Python lists: out-adjacency (v, e, ids, w in CSR order) and the step-ordered in-lists (by parent's
    original id, then position), which is the order the device's walk back reads its in-lists in"""

    def __init__(self, g):
        self.g, self.n, self.is_f = g, g.n, g.is_f
        self.v, self.e, self.ids, self.w = g.v.tolist(), g.e.tolist(), g.ids.tolist(), g.w.tolist()
        self.st_off, self.st_par, self.st_idx = g.st_off.tolist(), g.st_par.tolist(), g.st_idx.tolist()

    def add(self, c, w):
        """c + w in the weight type's arithmetic, None when it is NaN or reaches the sentinel (BIGINT: tested before
        the addition, as ck_sum does)"""
        if self.is_f:
            r = c + w
            return r if r < S_F else None
        return c + w if w < S_I - c else None


def skipped_kind(G, idx, x, dset, vban, eban, rc):
    """why entry idx (to x) of u's adjacency is not an admissible seed from the root cost rc"""
    if idx in dset:
        return "d"
    if idx in eban:
        return "eban"
    if x in vban:
        return "vban"
    w = G.w[idx]
    if G.is_f and w != w:
        return "nan"
    return "sentinel"


def spur_search(G, u, t, rc, dset, vban, eban, rec):
    """One spur search from u to t with root cost rc: the seeds, the Bellman-Ford fixed point, the tight BFS and the
    walk back.  -> [(parent, position)] of the spur, or None.  Fills rec (seed, skipped, depth, picks)."""
    v, e, w, add = G.v, G.e, G.w, G.add
    d = {}
    rec.update(seed=None, skipped=[], depth=0, picks=[], h=0)
    for idx in range(v[u], v[u + 1]):
        x = e[idx]
        c = add(rc, w[idx]) if idx not in dset and idx not in eban and x not in vban else None
        if c is None:
            if rec["seed"] is None:
                rec["skipped"].append(skipped_kind(G, idx, x, dset, vban, eban, rc))
            continue
        if rec["seed"] is None:
            rec["seed"] = idx - v[u]
        if x not in d or c < d[x]:
            d[x] = c
    if rec["seed"] is None:
        return None
    queue, queued = deque(d), set(d)
    while queue:  # the fixed point does not depend on the order of the relaxations
        x = queue.popleft()
        queued.discard(x)
        dx = d[x]
        for idx in range(v[x], v[x + 1]):
            y = e[idx]
            if idx in eban or y in vban:
                continue
            c = add(dx, w[idx])
            if c is not None and (y not in d or c < d[y]):
                d[y] = c
                if y not in queued:
                    queued.add(y)
                    queue.append(y)
    rec["dist_t"], rec["dist"] = d.get(t), d
    lvl, front = {}, []
    for idx in range(v[u], v[u + 1]):
        x = e[idx]
        if idx in dset or idx in eban or x in vban or x in lvl:
            continue
        c = add(rc, w[idx])
        if c is not None and c == d[x]:
            lvl[x] = 1
            front.append(x)
    lv = 1
    while t not in lvl and front:
        if lv + 1 > LEVEL_MAX:
            raise Refused("tight")
        rec["depth"] += 1
        nxt = []
        for x in front:
            dx = d[x]
            for idx in range(v[x], v[x + 1]):
                y = e[idx]
                if y in lvl or idx in eban or y in vban:
                    continue
                c = add(dx, w[idx])
                if c is not None and c == d.get(y):
                    lvl[y] = lv + 1
                    nxt.append(y)
        lv += 1
        front = nxt
    if t not in lvl:
        return None
    H = lvl[t]
    rec["h"] = H
    steps = [None] * H
    cur = t
    for l in range(H, 1, -1):
        dc, before = d[cur], []
        for i in range(G.st_off[cur], G.st_off[cur + 1]):
            par, idx = G.st_par[i], G.st_idx[i]
            c = add(d[par], w[idx]) if par in d else None
            tight = c is not None and c == dc
            if lvl.get(par) == l - 1 and idx not in eban and tight:
                break
            before.append("trail_banned" if tight and lvl.get(par) == l - 1 else
                          "wrong_level" if tight else "nontight")
        else:
            raise AssertionError("a vertex at level lv has a tight admissible parent at level lv - 1")
        rec["picks"].append(dict(kind="in", index=i - G.st_off[cur], before=set(before), vertex=cur, parent=par))
        steps[l - 1] = (par, idx)
        cur = par
    dc, before = d[cur], []
    for idx in range(v[u], v[u + 1]):
        if e[idx] != cur:
            continue
        c = add(rc, w[idx]) if idx not in dset and idx not in eban and cur not in vban else None
        if c is not None and c == dc:
            break
        before.append("nontight" if c is not None else "inadmissible")
    rec["picks"].append(dict(kind="adj", index=idx - v[u], before=set(before), vertex=cur, parent=u))
    steps[0] = (u, idx)
    return steps


def lane_cap(n, lanes):
    """CkSearch's cap: opts->lanes, or the widest of 256 .. 32 whose distance array n x W x 8 bytes fits 2 GiB"""
    if lanes:
        return lanes
    cap = 256
    while cap > 32 and max(n, 1) * cap * 8 > CK_BUDGET:
        cap >>= 1
    return cap


def round_width(cap, lanes, searches):
    """km_lanes: the cap, halved while the round's searches are at most half of it (not with forced lanes)"""
    W = cap
    while not lanes and W > 32 and searches <= W // 2:
        W >>= 1
    return W


def path_key(q):
    """the pool's and the result's order: cost, h, then (parent's original id, position) from t back to s"""
    h = len(q["pos"])
    return (q["cost"][-1], h, tuple((q["v"][i], q["pos"][i]) for i in range(h - 1, -1, -1)))


def ck_call(G, rows, ok, k, mode, lanes=0):
    """One call -> dict(paths, costs, npaths, stats, spurs, batches, rounds); raises Refused."""
    if (np.asarray(G.g.w) < 0).any():
        raise Refused("negative")
    walk, trail = mode == "WALK", mode == "TRAIL"
    bans_vertices = mode in ("ACYCLIC", "SIMPLE")
    zero = 0.0 if G.is_f else 0
    cap = lane_cap(G.n, lanes)
    R = []
    for (s, t), good in zip(rows, ok):
        if not good:
            R.append(None)
            continue
        r = dict(s=s, t=t, acc=[], pool={}, known=set(), live=True, closed=s == t)
        if s == t:  # A[0] = [s], no search
            q = dict(v=[s], pos=[], cost=[zero], dev=0)
            r["known"].add(path_key(q))
            r["acc"].append(q)
            r["live"] = k > 1
        R.append(r)
    stats = dict(batches=0, lanes=lanes or 32, searches=0, push_levels=0)
    spurs_rec, batches_rec, rounds = [], [], []
    for rnd in range(1 << 30):
        spurs = []
        for ri, r in enumerate(R):
            if r is None or not r["live"]:
                continue
            if rnd == 0:
                if not r["closed"]:
                    spurs.append(dict(row=ri, j=0, u=r["s"], rc=zero, dset=set(), vban=set(), eban=set()))
                continue
            P = r["acc"][-1]
            L = len(P["pos"])
            j0, j1 = P["dev"], L if trail or walk else L - 1
            if mode == "SIMPLE" and r["closed"] and L == 0:
                j0 = j1 = 0
            for j in range(j0, j1 + 1):
                vban = {x for x in P["v"][:j + 1] if not (r["closed"] and x == r["t"])} if bans_vertices else set()
                dset = {Q["pos"][j] for Q in r["acc"] if len(Q["pos"]) > j and Q["pos"][:j] == P["pos"][:j]}
                eban = set(P["pos"][:j]) if trail else set()
                spurs.append(dict(row=ri, j=j, u=P["v"][j], rc=P["cost"][j], dset=dset, vban=vban, eban=eban))
        for x, sp in enumerate(spurs):
            sp.update(round=rnd, index=x)
            sp["steps"] = spur_search(G, sp["u"], R[sp["row"]]["t"], sp["rc"], sp["dset"], sp["vban"], sp["eban"], sp)
        lane_of = [sp for sp in spurs if sp["seed"] is not None]
        W = round_width(cap, lanes, len(lane_of))
        stats["lanes"] = max(stats["lanes"], W)
        stats["searches"] += len(lane_of)
        rounds.append(dict(searches=len(lane_of), W=W, spurs=len(spurs)))
        for b0 in range(0, len(lane_of), W):
            lanes_b = lane_of[b0:b0 + W]
            keys = sorted((p, l) for l, sp in enumerate(lanes_b) for p in sp["eban"]) if trail else []
            batches_rec.append(dict(round=rnd, W=W, cnt=len(lanes_b), keys=keys, spurs=lanes_b))
            for l, sp in enumerate(lanes_b):
                sp.update(lane=l, word=l >> 6, group=l >> 5, batch=len(batches_rec) - 1)
            stats["batches"] += 1
            stats["push_levels"] += max(sp["depth"] for sp in lanes_b)
        spurs_rec += spurs
        for sp in lane_of:  # R + spur into the row's pool unless known
            if sp["steps"] is None:
                continue
            r = R[sp["row"]]
            if rnd == 0:
                q = dict(v=[r["s"]], pos=[], cost=[zero], dev=0)
            else:
                P, j = r["acc"][-1], sp["j"]
                q = dict(v=P["v"][:j + 1], pos=P["pos"][:j], cost=P["cost"][:j + 1], dev=j)
            for i, (par, idx) in enumerate(sp["steps"]):
                q["pos"].append(idx)
                q["v"].append(sp["steps"][i + 1][0] if i + 1 < len(sp["steps"]) else r["t"])
                q["cost"].append(q["cost"][-1] + G.w[idx])
            key = path_key(q)
            if key not in r["known"]:
                r["known"].add(key)
                r["pool"][key] = q
        any_live = False
        for r in R:
            if r is None or not r["live"]:
                continue
            if rnd == 0 and r["closed"]:
                any_live = True
                continue
            if not r["pool"]:
                r["live"] = False
                continue
            key = min(r["pool"])
            if key[1] > PATH_MAX:
                raise Refused("long")
            r["acc"].append(r["pool"].pop(key))
            r["live"] = len(r["acc"]) < k
            any_live |= r["live"]
        if not any_live:
            break
    paths, costs = [], []
    for r in R:
        if r is None or not r["acc"]:
            paths.append(None)
            costs.append(None)
            continue
        paths.append([[q["v"][0]] + [x for i in range(len(q["pos"])) for x in (G.ids[q["pos"][i]], q["v"][i + 1])]
                      for q in r["acc"]])
        costs.append([q["cost"][-1] for q in r["acc"]])
    return dict(paths=paths, costs=costs, npaths=[0 if p is None else len(p) for p in paths], stats=stats,
                spurs=spurs_rec, batches=batches_rec, rounds=rounds, rows=R)


# ---- the catalogue -----------------------------------------------------------------------------------------------------
ROUND_SIZES = (32, 33, 64, 65, 128, 129, 256, 257)
FORCED = (32, 64, 128, 256)
LADDER_DISTINCT = 250
LADDER_DUPS = 7


def ladder(w_scale=1):
    """257 rows into one target t over a ladder: row r has s_r -> t (its cheapest path) and s_r -> y_r -> s_(r-64) ->
    t (the next one; y_r -> q_r -> t below 64), so row r's spurs run through the source of the row 64 lanes before it.
    ACYCLIC and SIMPLE ban s_(r-64) in that row's lane and not in row r's; TRAIL's third round bans in row r - 64's lane
    the positions row r's route takes.  Sources without out-edges (a row each, no seed, no lane) sit between the rows,
    and the last 7 rows repeat rows 64 .. 70, so their TRAIL bans are the same positions in another word."""
    b = WBuilder()
    t = b.new()
    s = [b.new() for _ in range(LADDER_DISTINCT)]
    for r in range(LADDER_DISTINCT):
        b.edge(s[r], t, w=w_scale * (1 + r % 3))
        y = b.new()
        b.edge(s[r], y, w=w_scale)
        if r >= 64:
            b.edge(y, s[r - 64], w=w_scale)
        else:
            q = b.chain(y, 1, w=w_scale)
            b.edge(q, t, w=w_scale)
    rows, real = [], []
    for r in list(range(LADDER_DISTINCT)) + list(range(64, 64 + LADDER_DUPS)):
        if r % 5 == 2:
            rows.append((b.new(), t))  # a source with no out-edge: no seed
        real.append(len(rows))
        rows.append((s[r], t))
    return b, rows, real


def case_ladder():
    b, rows, real = ladder()
    return dict(n=b.n, src=b.src, dst=b.dst, w=b.w, rows=rows, ok=[1] * len(rows), ks=(3,), real=real,
                named={*{f"round_{x}" for x in ROUND_SIZES}, *{f"forced_{x}" for x in FORCED}, "last_batch_cnt_1",
                       "lane_ne_spur", *{f"vban_differs_{x}_{x + 1}" for x in (63, 127, 191)}, "vban_cross_word",
                       "dist_differs_31_32", "trail_pos_two_words", "trail_pos_ge_32", "trail_cross_word",
                       "duplicate_rows", "words_4"})


def case_cap(n_total):
    def make():
        b = WBuilder()
        t = b.new()
        for r in range(129):
            b.edge(b.new(), t, w=1 + r % 5)
        rows = [(x, t) for x in range(1, 130)]
        return dict(n=n_total, src=b.src, dst=b.dst, w=b.w, rows=rows, ok=[1] * len(rows), modes=("WALK",), ks=(1,),
                    named={f"cap_{lane_cap(n_total, 0)}_n_{n_total}"})
    return make


def chunk_graph(is_f):
    """For j = 31, 32, 33: u_j's adjacency holds its first path's edge (D in round 1), a self-loop (banned by ACYCLIC
    and SIMPLE), then sentinel entries (BIGINT weights S and INT64_MAX; DOUBLE NaN, +inf and S_F), then at index j
    the only admissible seed of round 1.  t_j's in-list holds 34 parents in step order whose edges are not tight from
    s_j (one is tight at the wrong level) but for parent j.  v_j has j parallel non-tight edges to x_j ahead of the
    tight one at index j."""
    b = WBuilder()
    t = b.new()
    bad = [S_I, INT64_MAX] if not is_f else [np.nan, np.inf, S_F]
    one = 1.0 if is_f else 1
    rows = []
    for j in (31, 32, 33):
        u, a = b.new(), b.new()
        b.edge(u, t, w=one)
        b.edge(u, u, w=one)
        for i in range(2, j):
            b.edge(u, t, w=bad[i % len(bad)])
        b.edge(u, a, w=one)
        b.edge(a, t, w=one)
        rows.append((u, t))
    for j in (31, 32, 33):
        s, tt, q = b.new(), b.new(), b.new()
        par = b.new(34)
        b.edge(s, q, w=one)
        for i, p in enumerate(par):
            b.edge(s, p, w=one if i == j else 2 * one)
            b.edge(p, tt, w=one)
        b.edge(q, par[1], w=0 * one)  # par[1]: cost 1 at level 2, its edge to tt tight at the wrong level
        rows.append((s, tt))
    for j in (31, 32, 33):
        s, x = b.new(), b.new()
        for _ in range(j):
            b.edge(s, x, w=5 * one)
        b.edge(s, x, w=one)
        b.edge(x, t, w=one)
        rows.append((s, t))
    return b, rows


def case_chunks(is_f):
    def make():
        b, rows = chunk_graph(is_f)
        names = {*{f"seed_at_{j}" for j in (31, 32, 33)}, *{f"pick_in_{j}" for j in (31, 32, 33)},
                 *{f"pick_adj_{j}" for j in (31, 32, 33)}, "seed_behind_d", "seed_behind_vban", "seed_behind_sentinel",
                 "pick_in_behind_nontight", "pick_in_behind_wrong_level", "pick_adj_behind_nontight",
                 "parallel_one_tight"}
        names |= {"seed_behind_nan", "f64_inf", "f64_nan"} if is_f else {"i64_weight_S", "i64_weight_max"}
        return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.float64 if is_f else np.int64), rows=rows,
                    ok=[1] * len(rows), ks=(3,), named=names)
    return make


def case_trail_detour():
    """TRAIL: s -> a -> b -> c -> t, and c -> a, a -> m -> b, b -> d -> t at zero cost around it.  The spur at c (root
    s, a, b, c) returns to a, where the banned root edge a -> b is tight: the tight route detours over m.  A second
    edge a -> b beside the first: a walk back that meets the banned parallel edge first must skip it."""
    b = WBuilder()
    s, a, bb, c, t, m, d = (b.new() for _ in range(7))
    b.edge(s, a, w=1)
    b.edge(a, bb, w=0)
    b.edge(a, m, w=0)
    b.edge(m, bb, w=0)
    b.edge(bb, c, w=1)
    b.edge(c, t, w=1)
    b.edge(c, a, w=0)
    b.edge(bb, d, w=1)
    b.edge(d, t, w=1)
    s2, a2, b2, t2 = (b.new() for _ in range(4))
    b.edge(s2, a2, w=1)
    b.edge(a2, b2, w=1, mult=2)
    b.edge(b2, t2, w=1)
    b.edge(b2, a2, w=0)
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=[(s, t), (s2, t2)], ok=[1, 1],
                ks=(6,), small=True, named={"trail_detour", "pick_in_behind_trail_banned"})


def case_modes():
    """closed rows in every mode (SIMPLE exempts t), a zero-cost cycle that fills WALK, NULL ids, a duplicate row and
    k above a row's total"""
    b = WBuilder()
    s, a, c, t = (b.new() for _ in range(4))
    b.edge(s, a, w=1)
    b.edge(a, c, w=0)
    b.edge(c, a, w=0)
    b.edge(a, t, w=1)
    b.edge(t, s, w=2)
    b.edge(s, t, w=3)
    rows = [(s, t), (s, s), (a, a), (s, t), (t, t), (c, s)]
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=rows, ok=[1, 1, 1, 0, 1, 1],
                dv=[1, 1, 1, 1, 1, 0], ks=(8,), small=True,
                named={*{f"closed_{m}" for m in MODES}, "simple_closed_exempt_t", "zero_cycle_fills_walk",
                       "null_ids", "k_above_total"})


def case_specials_i64():
    """BIGINT prefix sums at S - 1 (found) and S (refused: the edge closing it is not admissible); finding 2: 0 -> 1
    -> 2 over [S - 1, INT64_MAX] and [1, INT64_MAX], which the reference's wrapping sum still costs"""
    b = WBuilder()
    s, a, t1, t2 = (b.new() for _ in range(4))
    b.edge(s, a, w=S_I - 2)
    b.edge(a, t1, w=1)
    b.edge(a, t2, w=2)
    f = [b.new() for _ in range(6)]
    b.edge(f[0], f[1], w=S_I - 1)
    b.edge(f[1], f[2], w=INT64_MAX)
    b.edge(f[3], f[4], w=1)
    b.edge(f[4], f[5], w=INT64_MAX)
    rows = [(s, t1), (s, t2), (f[0], f[2]), (f[3], f[5]), (f[0], f[1])]
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=rows, ok=[1] * len(rows), ks=(3,),
                small=True, finding2=[2, 3],
                named={"i64_prefix_S_minus_1", "i64_prefix_S_refused", "i64_weight_max", "finding_2"})


def case_specials_f64():
    """DOUBLE: sums that round to exactly S_F (refused) and just below it; +inf, NaN, -0.0 and 5e-324 weights; the
    non-dyadic finding 1 graph verbatim (0 -> 3 is not tight: 1.0000000000000002 != d(3) = 1.0)"""
    b = WBuilder()
    s, x, t1, t2, t3, z, t4, t5, y = (b.new() for _ in range(9))
    b.edge(s, x, w=S_F - ULP_S_F)
    b.edge(x, t1, w=1.25 * ULP_S_F)
    b.edge(x, t2, w=0.25 * ULP_S_F)
    b.edge(s, t3, w=np.inf)
    b.edge(s, t3, w=np.nan)
    b.edge(s, t3, w=1.0)
    b.edge(s, z, w=-0.0)
    b.edge(z, t4, w=-0.0)
    b.edge(s, t5, w=5e-324)
    b.edge(s, y, w=0.0)
    b.edge(y, t5, w=5e-324)
    f = b.new(5)
    b.edge(f[0], f[3], w=1.0000000000000002)
    b.edge(f[0], f[1], w=0.5)
    b.edge(f[1], f[2], w=0.25)
    b.edge(f[2], f[3], w=0.25)
    b.edge(f[3], f[4], w=2.0)
    rows = [(s, t1), (s, t2), (s, t3), (s, t4), (s, t5), (f[0], f[4])]
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.float64), rows=rows, ok=[1] * len(rows), ks=(3,),
                small=True, finding1=5,
                named={"f64_sum_rounds_to_S_refused", "f64_sum_just_below_S", "f64_inf", "f64_nan",
                       "f64_neg_zero_cost", "f64_subnormal", "nondyadic", "finding_1"})


def case_perm():
    """two cheapest routes s -> p -> t and s -> q -> t of one cost; q (the higher original id) has more out-edges, so
    the internal order puts it before p: the tie goes to p, by original id"""
    b = WBuilder()
    s, p, q, t, z = (b.new() for _ in range(5))
    b.edge(s, p, w=1)
    b.edge(s, q, w=1)
    b.edge(p, t, w=1)
    b.edge(q, t, w=1)
    b.edge(q, z, w=5, mult=3)
    return dict(n=b.n, src=b.src, dst=b.dst, w=np.array(b.w, np.int64), rows=[(s, t)], ok=[1], ks=(3,), small=True,
                named={"tie_by_original_id"})


CHAIN = 65536


def case_chain():
    """a zero-cost chain 0 -> 1 -> ... -> 65536 with ascending ids and an isolated 65537: rows of 65533 edges (found),
    65534 (refused at acceptance), 65535 (refused: tight depth) and the isolated target (refused: the tight BFS runs
    on along the chain although no path exists)"""
    n = CHAIN + 2
    src = list(range(CHAIN))
    return dict(n=n, src=src, dst=[x + 1 for x in src], w=np.zeros(CHAIN, np.int64),
                rows=[(0, 65533), (0, 65534), (0, 65535), (0, CHAIN + 1)], ok=[1] * 4, modes=("WALK",), ks=(1,),
                single_rows=True,
                named={"chain_65533", "chain_65534_refused_long", "chain_65535_refused_tight",
                       "unreachable_refused_tight"})


CATALOGUE = {
    "ladder": case_ladder,
    "cap_2p20": case_cap(1 << 20),
    "cap_2p20_1": case_cap((1 << 20) + 1),
    "chunks_i64": case_chunks(False),
    "chunks_f64": case_chunks(True),
    "trail_detour": case_trail_detour,
    "modes": case_modes,
    "specials_i64": case_specials_i64,
    "specials_f64": case_specials_f64,
    "perm": case_perm,
    "chain": case_chain,
}

REQUIRED = (
    {f"round_{x}" for x in ROUND_SIZES} | {f"forced_{x}" for x in FORCED} | {"last_batch_cnt_1", "lane_ne_spur"}
    | {f"vban_differs_{x}_{x + 1}" for x in (63, 127, 191)} | {"vban_cross_word", "dist_differs_31_32", "words_4"}
    | {"trail_pos_two_words", "trail_pos_ge_32", "trail_cross_word", "trail_detour", "duplicate_rows"}
    | {f"cap_256_n_{1 << 20}", f"cap_128_n_{(1 << 20) + 1}"}
    | {f"seed_at_{j}" for j in (31, 32, 33)} | {f"pick_in_{j}" for j in (31, 32, 33)}
    | {f"pick_adj_{j}" for j in (31, 32, 33)}
    | {"seed_behind_d", "seed_behind_vban", "seed_behind_sentinel", "seed_behind_nan"}
    | {"pick_in_behind_nontight", "pick_in_behind_wrong_level", "pick_in_behind_trail_banned",
       "pick_adj_behind_nontight", "parallel_one_tight"}
    | {f"closed_{m}" for m in MODES} | {"simple_closed_exempt_t", "zero_cycle_fills_walk", "null_ids", "k_above_total"}
    | {"i64_prefix_S_minus_1", "i64_prefix_S_refused", "i64_weight_S", "i64_weight_max", "finding_2"}
    | {"f64_sum_rounds_to_S_refused", "f64_sum_just_below_S", "f64_inf", "f64_nan", "f64_neg_zero_cost",
       "f64_subnormal", "nondyadic", "finding_1"}
    | {"tie_by_original_id"}
    | {"chain_65533", "chain_65534_refused_long", "chain_65535_refused_tight", "unreachable_refused_tight"}
)


@lru_cache(maxsize=None)
def case(name):
    c = CATALOGUE[name]()
    c["w"] = np.asarray(c["w"], np.float64 if np.asarray(c["w"]).dtype.kind == "f" else np.int64)
    c["g"] = WGraph(c["n"], c["src"], c["dst"], c["w"])
    c["G"] = Lists(c["g"])
    c["ps"] = np.array([s for s, _ in c["rows"]], np.int64)
    c["pd"] = np.array([t for _, t in c["rows"]], np.int64)
    c["sv"] = np.array(c["ok"], np.uint8)
    c["dv"] = np.array(c.get("dv", [1] * len(c["rows"])), np.uint8)
    c.setdefault("modes", MODES)
    return c


def ks_of(name):
    return tuple(dict.fromkeys((1, 3) + case(name).get("ks", ())))


def row_sets(name):
    """the row subsets a case is called with: every row at once, or (single_rows) one row per call"""
    c = case(name)
    if c.get("single_rows"):
        return [(i,) for i in range(len(c["rows"]))]
    return [tuple(range(len(c["rows"])))]


def prefix(name, count):
    """the rows up to the count-th row that takes a lane in round 0"""
    return tuple(range(case(name)["real"][count - 1] + 1))


def call(name, k, mode, idx=None, lanes=0):
    c = case(name)
    idx = tuple(range(len(c["rows"]))) if idx is None else tuple(idx)
    return _call(name, k, mode, idx, lanes)


@lru_cache(maxsize=None)
def _call(name, k, mode, idx, lanes):
    c = case(name)
    ok = [bool(c["sv"][i] and c["dv"][i]) for i in idx]
    try:
        return ck_call(c["G"], [c["rows"][i] for i in idx], ok, k, mode, lanes)
    except Refused as ex:
        return dict(error=ex)


def calls(name):
    """(k, mode, idx, lanes) of every call a case is checked with"""
    c = case(name)
    out = [(k, m, idx, 0) for m in c["modes"] for k in ks_of(name) for idx in row_sets(name)]
    if "real" in c:
        out += [(1, "WALK", prefix(name, x), 0) for x in ROUND_SIZES]
        out += [(3, m, None, x) for m in ("TRAIL", "ACYCLIC") for x in FORCED]
    return out


# ---- the work record's boundaries ---------------------------------------------------------------------------------------
def case_hits(name):
    c = case(name)
    g, G = c["g"], c["G"]
    hits = set()
    for k, mode, idx, lanes in calls(name):
        res = call(name, k, mode, idx, lanes)
        if "error" in res:
            continue
        for rd in res["rounds"]:
            if rd["searches"] in ROUND_SIZES:
                hits.add(f"round_{rd['searches']}")
        if lanes and any(b["cnt"] == lanes for b in res["batches"]) and res["stats"]["batches"] > 1:
            hits.add(f"forced_{lanes}")
        if len(res["batches"]) > 1 and res["batches"][-1]["cnt"] == 1 and res["batches"][-2]["round"] == \
                res["batches"][-1]["round"]:
            hits.add("last_batch_cnt_1")
        for b in res["batches"]:
            sp = b["spurs"]
            if any(x["lane"] != x["index"] for x in sp):
                hits.add("lane_ne_spur")
            if b["W"] == 256 and b["cnt"] > 192:
                hits.add("words_4")
            for x in (63, 127, 191):
                if b["cnt"] > x + 1 and sp[x]["vban"] and sp[x + 1]["vban"] and sp[x]["vban"] != sp[x + 1]["vban"]:
                    hits.add(f"vban_differs_{x}_{x + 1}")
            if b["cnt"] > 32 and sp[31].get("dist_t") != sp[32].get("dist_t"):
                hits.add("dist_differs_31_32")
            for l, x in enumerate(sp):  # a lane's route through a vertex or a position that a lane of another word,
                if x["steps"] is None:   # at the same bit, bans
                    continue
                route_v = {par for par, _ in x["steps"][1:]}
                route_e = {idx for _, idx in x["steps"]}
                for o in range(l & 63, b["cnt"], 64):
                    if o != l and route_v & sp[o]["vban"] and not route_v & x["vban"]:
                        hits.add("vban_cross_word")
                    if o != l and route_e & sp[o]["eban"] and not route_e & x["eban"]:
                        hits.add("trail_cross_word")
            words = {}
            for p, l in b["keys"]:
                words.setdefault(p, set()).add(l >> 6)
                if p >= 32:
                    hits.add("trail_pos_ge_32")
            if any(len(x) > 1 for x in words.values()):
                hits.add("trail_pos_two_words")
        for sp in res["spurs"]:
            if sp["seed"] in (31, 32, 33) and sp["seed"] == len(sp["skipped"]):
                hits.add(f"seed_at_{sp['seed']}")
                hits |= {f"seed_behind_{x}" for x in sp["skipped"] if x != "eban"}
            for pk in sp["picks"]:
                if pk["index"] in (31, 32, 33):
                    hits.add(f"pick_{pk['kind']}_{pk['index']}")
                    hits |= {f"pick_{pk['kind']}_behind_{x}" for x in pk["before"] if x != "inadmissible"}
                if pk["kind"] == "in" and "trail_banned" in pk["before"]:
                    hits.add("pick_in_behind_trail_banned")
                if pk["kind"] == "in" and g.perm[pk["parent"]] > min(
                        (g.perm[G.st_par[i]] for i in range(G.st_off[pk["vertex"]], G.st_off[pk["vertex"] + 1])
                         if G.st_par[i] != pk["parent"]), default=g.n):
                    hits.add("tie_by_original_id")
                if pk["kind"] == "adj" and "nontight" in pk["before"]:
                    hits.add("parallel_one_tight")
            if mode == "TRAIL" and sp["steps"] is not None and sp["eban"]:
                route_v = [par for par, _ in sp["steps"]]
                banned_tight = [p for p in sp["eban"] if G.e[p] in route_v and g.row[p] in route_v]
                if banned_tight and sp["h"] > 1 + len(banned_tight):
                    hits.add("trail_detour")
        rows = [c["rows"][i] for i in (range(len(c["rows"])) if idx is None else idx)]
        for (s, t), p, cs in zip(rows, res["paths"], res["costs"]):
            if p and s == t and k >= 3 and (len(p) > 1) == (mode != "ACYCLIC"):  # (ACYCLIC: [s] alone)
                hits.add(f"closed_{mode}")
                if mode == "SIMPLE" and all(q[-1] == t and t not in q[2:-1:2] for q in p[1:]):
                    hits.add("simple_closed_exempt_t")
            if p and mode == "WALK" and len(p) == k == 8 and len(set(cs)) == 1 and len({len(q) for q in p}) == 8:
                hits.add("zero_cycle_fills_walk")
            if p and len(p) < k and mode == "ACYCLIC":
                hits.add("k_above_total")
        if len(set(rows)) < len(rows):
            hits.add("duplicate_rows")
        if any(p is None for p, i in zip(res["paths"], range(len(rows)))) and not all(c["sv"] & c["dv"]):
            hits.add("null_ids")
        for sp in res["spurs"]:
            if not G.is_f and sp.get("dist_t") == S_I - 1:
                hits.add("i64_prefix_S_minus_1")
            if G.is_f and sp.get("dist_t") is not None and S_F - ULP_S_F <= sp["dist_t"] < S_F:
                hits.add("f64_sum_just_below_S")
    w = c["w"]
    if not G.is_f:
        if (w == S_I).any():
            hits.add("i64_weight_S")
        if (w == INT64_MAX).any():
            hits.add("i64_weight_max")
        refused = [r for r in case_refused_sums(name) if r == S_I]
        if refused:
            hits.add("i64_prefix_S_refused")
    else:
        if np.isinf(w).any():
            hits.add("f64_inf")
        if np.isnan(w).any():
            hits.add("f64_nan")
        if (w == 5e-324).any():
            hits.add("f64_subnormal")
        if any(x == S_F for x in case_refused_sums(name)):
            hits.add("f64_sum_rounds_to_S_refused")
        res = call(name, 3, "WALK")
        for p, cs in zip(res["paths"], res["costs"]):
            for q, x in zip(p or [], cs or []):
                ws = [g.w[int(np.flatnonzero(g.ids == eid)[0])] for eid in q[1::2]]
                if ws and all(y == 0 and np.signbit(y) for y in ws) and not np.signbit(x):
                    hits.add("f64_neg_zero_cost")
                if sum(Fraction(float(y)) for y in ws) != Fraction(x):  # the cost rounded
                    hits.add("nondyadic")
    if "finding1" in c and finding_1_holds(name):
        hits.add("finding_1")
    if "finding2" in c and finding_2_holds(name):
        hits.add("finding_2")
    if name == "chain":
        for i, hit in enumerate(("chain_65533", "chain_65534_refused_long", "chain_65535_refused_tight",
                                 "unreachable_refused_tight")):
            res = call(name, 1, "WALK", (i,))
            want = (None, "long", "tight", "tight")[i]
            if (res.get("error") and res["error"].kind) == want and (want or len(res["paths"][0][0]) == 2 * 65533 + 1):
                hits.add(hit)
    if name.startswith("cap"):
        res = call(name, 1, "WALK")
        hits.add(f"cap_{res['stats']['lanes']}_n_{c['n']}")
    return hits


def case_refused_sums(name):
    """the sums a WALK search of the case refused from a reached vertex's distance over an out-edge: at or above the
    sentinel (as values, rounded for DOUBLE; NaN left out)"""
    G = case(name)["G"]
    res = call(name, 1, "WALK")
    out = []
    for sp in res.get("spurs", ()):
        for x, dx in sp.get("dist", {}).items():
            for idx in range(G.v[x], G.v[x + 1]):
                if G.add(dx, G.w[idx]) is None and dx + G.w[idx] == dx + G.w[idx]:
                    out.append(dx + G.w[idx])
    return out


def finding_1_paths():
    """finding 1's two paths (0 -> 1 -> 2 -> 3 -> 4 and 0 -> 3 -> 4) as element lists"""
    c = case("specials_f64")
    g = c["g"]
    s = c["rows"][c["finding1"]][0]
    eid = {(int(g.row[k]), int(g.e[k])): int(g.ids[k]) for k in range(len(g.e))}
    four = [s, eid[s, s + 1], s + 1, eid[s + 1, s + 2], s + 2, eid[s + 2, s + 3], s + 3, eid[s + 3, s + 4], s + 4]
    two = [s, eid[s, s + 3], s + 3, eid[s + 3, s + 4], s + 4]
    return four, two


def finding_1_holds(name):
    """finding 1: the 4-edge path of cost 3.0 leads the 2-edge one of the same cost in every mode"""
    i = case(name)["finding1"]
    return all(call(name, 3, m)["paths"][i] == list(finding_1_paths()) and call(name, 3, m)["costs"][i] == [3.0, 3.0]
               for m in MODES)


def finding_2_holds(name):
    """finding 2: cheapest_k_paths has no path on the rows whose BIGINT sum would pass INT64_MAX"""
    c = case(name)
    return all(call(name, k, m)["paths"][i] is None for i in c["finding2"] for m in MODES for k in (1, 3))


# ---- CPU: the hits, the coverage, the oracle against the restatement ------------------------------------------------
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_catalogue_hits_its_boundaries(name):
    hits = case_hits(name)
    missing = case(name)["named"] - hits
    assert not missing, sorted(missing)


def test_catalogue_covers_every_boundary():
    named = set().union(*(CATALOGUE[x]()["named"] for x in CATALOGUE))
    assert REQUIRED <= named, sorted(REQUIRED - named)
    assert named <= REQUIRED, sorted(named - REQUIRED)


def oracle_call(name, k, mode, idx=None, lanes=0):
    c = case(name)
    g = c["g"]
    idx = np.arange(len(c["rows"])) if idx is None else np.asarray(list(idx))
    return ock.cheapest_k_paths(g.n, g.v, g.e, g.ids, g.w, c["ps"][idx], c["pd"][idx], k, mode, c["sv"][idx],
                                c["dv"][idx], lanes)


def bits(costs):
    """per-row cost lists as raw bits (ints stay ints): -0.0 apart from 0.0"""
    return [None if r is None else [np.float64(x).tobytes() if isinstance(x, float) else x for x in r] for r in costs]


STATS = ("batches", "lanes", "searches", "push_levels")


def check_oracle(name, k, mode, idx, lanes):
    res = call(name, k, mode, idx, lanes)
    if "error" in res:
        with pytest.raises(OracleError) as ex:
            oracle_call(name, k, mode, idx, lanes)
        assert ex.value.code == ock.ERR_UNSUPPORTED, (name, k, mode)
        return
    paths, costs, npaths, st = oracle_call(name, k, mode, idx, lanes)
    assert paths == res["paths"], (name, k, mode, lanes)
    assert bits(costs) == bits(res["costs"]), (name, k, mode, lanes)
    assert npaths.tolist() == res["npaths"], (name, k, mode, lanes)
    for x in STATS:
        assert st[x] == res["stats"][x], (name, k, mode, lanes, x)


@pytest.mark.parametrize("name", list(CATALOGUE))
def test_oracle_equals_the_restatement(name):
    for k, mode, idx, lanes in calls(name):
        check_oracle(name, k, mode, idx, lanes)


@pytest.mark.parametrize("name", [x for x in CATALOGUE if CATALOGUE[x]().get("small")])
def test_small_cases_are_the_brute_force_paths(name):
    """the TRAIL, ACYCLIC and SIMPLE paths of the small cases by enumeration, in (cost, h, steps) order; not on finding
    1's row, where a sum rounds and the construction orders the paths"""
    c = case(name)
    g = c["g"]
    sentinel = S_F if g.is_f else S_I
    for mode in ("TRAIL", "ACYCLIC", "SIMPLE"):
        res = call(name, 8, mode)
        for i, (s, t) in enumerate(c["rows"]):
            if not (c["sv"][i] and c["dv"][i]) or i == c.get("finding1"):
                continue
            exp = [(p, x) for p, x in brute_paths(g.n, g.v, g.e, g.ids, g.w, s, t, mode) if x < sentinel]
            assert list(zip(res["paths"][i] or [], res["costs"][i] or [])) == exp[:8], (name, mode, s, t)


def fold(c, path):
    """the path's weights summed left to right from 0 in the weight type's arithmetic"""
    g = c["g"]
    pos = {int(x): k for k, x in enumerate(g.ids)}
    x = 0.0 if g.is_f else 0
    for eid in path[1::2]:
        x = x + g.w[pos[eid]].item()
    return x


@pytest.mark.parametrize("name", list(CATALOGUE))
def test_costs_are_sorted_folds(name):
    c = case(name)
    for k, mode, idx, lanes in calls(name):
        res = call(name, k, mode, idx, lanes)
        if "error" in res:
            continue
        for p, cs in zip(res["paths"], res["costs"]):
            if p is None:
                continue
            assert cs == sorted(cs), (name, mode, k)
            for q, x in zip(p, cs):
                f = fold(c, q)
                assert np.float64(f).tobytes() == np.float64(x).tobytes() if c["g"].is_f else f == x


def test_finding_1_rounding_order_is_the_construction():
    """0 -> 3 costs 1.0000000000000002 != d(3) = 1.0, so it is not tight: the 4-edge path of cost 3.0 comes first, the
    2-edge path of the same rounded cost second -- not (cost, h) order"""
    i = case("specials_f64")["finding1"]
    four, two = finding_1_paths()
    for mode in MODES:
        res = call("specials_f64", 3, mode, (i,))
        assert res["paths"][0] == [four, two], mode
        assert res["costs"][0] == [3.0, 3.0], mode
        paths, costs, _, st = oracle_call("specials_f64", 3, mode, (i,))
        assert paths[0] == [four, two] and costs[0] == [3.0, 3.0], mode
        assert (st["batches"], st["lanes"], st["searches"], st["push_levels"]) == (2, 32, 2, 4), mode


def test_finding_2_bigint_sum_past_int64_max():
    """cheapest_path_length wraps (the reference's sum, kept for parity) and cheapest_path lists the route, while
    cheapest_k_paths refuses the sum before it is added: no path"""
    c = case("specials_i64")
    g = c["g"]
    for i in c["finding2"]:
        s, t = c["rows"][i]
        cost, valid = orc.cheapest_path_length(g.n, g.v, g.e, g.w, [s], [t])
        assert valid[0] == 1 and cost[0] < 0
        for mode in MODES:
            assert call("specials_i64", 1, mode)["paths"][i] is None
            assert oracle_call("specials_i64", 1, mode)[0][i] is None


W_COVERED = 1 << 62  # the largest BIGINT weight whose sums cheapest_path_length defines (max/2 + w does not overflow)


def covered(w):
    """the case's weights with BIGINT weights above 2^62 lowered to 2^62: still at or past the sentinel for
    cheapest_k_paths, and within what cheapest_path_length's reference sum covers"""
    w = np.asarray(w)
    return w if w.dtype.kind == "f" else np.minimum(w, W_COVERED)


def test_k1_identity_where_cheapest_path_length_is_defined():
    """k = 1 gives the oracle's cheapest_path and cheapest_path_length on every case once no BIGINT weight is above
    2^62; above it the reference's sum from a vertex s does not reach (max/2 + INT64_MAX) wraps into t, and the two
    part: the chunk rows' target keeps a cost-1 path here and gets a wrapped negative cost there"""
    for name in CATALOGUE:
        if name == "chain":
            continue  # (refused rows: test_refusals_of_the_restatement)
        c = case(name)
        ok = (c["sv"] & c["dv"]) == 1
        ps, pd = c["ps"][ok], c["pd"][ok]
        v, e, ids, w = orc.csr_build_weighted(c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64),
                                              covered(c["w"]))
        cost, valid = orc.cheapest_path_length(c["n"], v, e, w, ps, pd)
        cpaths, _ = ocp.cheapest_path(c["n"], v, e, ids, w, ps, pd)
        for mode in MODES:
            one, one_c, _, _ = ock.cheapest_k_paths(c["n"], v, e, ids, w, ps, pd, 1, mode)
            assert [r[0] if r else None for r in one] == cpaths, (name, mode)
            assert bits([r[:1] if r else None for r in one_c]) == \
                bits([[cost[i].item()] if valid[i] else None for i in range(len(ps))]), (name, mode)
    c = case("chunks_i64")
    g = c["g"]
    rows = [0, 1, 2]
    cost, valid = orc.cheapest_path_length(g.n, g.v, g.e, g.w, c["ps"][rows], c["pd"][rows])
    assert valid.tolist() == [1, 1, 1] and all(x < 0 for x in cost.tolist())
    for mode in MODES:
        assert [r[0] for r in call("chunks_i64", 1, mode)["costs"][:3]] == [1, 1, 1]


def test_refusals_of_the_restatement():
    for i, kind in ((1, "long"), (2, "tight"), (3, "tight")):
        assert call("chain", 1, "WALK", (i,))["error"].kind == kind
    assert len(call("chain", 1, "WALK", (0,))["paths"][0][0]) == 2 * PATH_MAX + 1
    g = WGraph(2, [0], [1], np.array([-1], np.int64))
    with pytest.raises(Refused) as ex:
        ck_call(Lists(g), [(0, 1)], [True], 1, "WALK")
    assert ex.value.kind == "negative"


# ---- GPU: the device against the restatement and the oracle ------------------------------------------------------------
def build(ctx, name):
    c = case(name)
    return pgq.DeviceCSR.build(ctx, c["n"], np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64),
                               weight=c["w"])


def device_call(csr, name, k, mode, idx=None, lanes=0):
    c = case(name)
    idx = np.arange(len(c["rows"])) if idx is None else np.asarray(list(idx))
    return csr.cheapest_k_paths(c["ps"][idx], c["pd"][idx], k, c["sv"][idx], c["dv"][idx], pgq.Options(lanes), mode)


def compare(csr, name, k, mode, idx=None, lanes=0):
    """the device's answer equals the restatement's and the oracle's (a refusal: its status and message)"""
    res = call(name, k, mode, idx, lanes)
    if "error" in res:
        with pytest.raises(pgq.PgqError) as ex:
            device_call(csr, name, k, mode, idx, lanes)
        assert ex.value.status == PGQ_ERR_UNSUPPORTED, (name, k, mode)
        assert REFUSAL_TEXT[res["error"].kind] in str(ex.value), (name, k, mode, str(ex.value))
        return None
    paths, costs, npaths, st = device_call(csr, name, k, mode, idx, lanes)
    assert paths == res["paths"], (name, k, mode, lanes)
    assert bits(costs) == bits(res["costs"]), (name, k, mode, lanes)
    assert npaths.tolist() == res["npaths"], (name, k, mode, lanes)
    opaths, ocosts, _, ost = oracle_call(name, k, mode, idx, lanes)
    assert paths == opaths and bits(costs) == bits(ocosts)
    for x in STATS:
        assert st[x] == res["stats"][x] == ost[x], (name, k, mode, lanes, x)
    assert st["levels"] >= st["batches"]
    return paths, costs


@pytest.mark.gpu
@pytest.mark.parametrize("name", [x for x in CATALOGUE if x != "chain"])
def test_device_catalogue(gpu_ctx, name):
    csr = build(gpu_ctx, name)
    try:
        for k, mode, idx, lanes in calls(name):
            compare(csr, name, k, mode, idx, lanes)
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_chain_refusals(gpu_ctx):
    """65533 edges found; 65534 refused at acceptance; 65535 and an unreachable target refused at tight depth 65534 --
    each by status and message"""
    csr = build(gpu_ctx, "chain")
    try:
        for i in range(4):
            compare(csr, "chain", 1, "WALK", (i,))
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_findings(gpu_ctx):
    """finding 1's order on the device, bit for bit; finding 2's divergence from cheapest_path_length and
    cheapest_path on the device"""
    csr = build(gpu_ctx, "specials_f64")
    try:
        c = case("specials_f64")
        i = c["finding1"]
        for mode in MODES:
            paths, costs, _, st = device_call(csr, "specials_f64", 3, mode, (i,))
            assert paths[0] == list(finding_1_paths()) and costs[0] == [3.0, 3.0], mode
            assert (st["batches"], st["lanes"], st["searches"], st["push_levels"]) == (2, 32, 2, 4)
    finally:
        csr.free()
    csr = build(gpu_ctx, "specials_i64")
    try:
        c = case("specials_i64")
        rows = c["finding2"]
        ps, pd = c["ps"][rows], c["pd"][rows]
        cost, valid, _ = csr.cheapest_path_length(ps, pd)
        cpaths, _ = csr.cheapest_path(ps, pd)
        assert valid.tolist() == [1, 1] and all(x < 0 for x in cost.tolist())
        assert all(p is not None and len(p) == 5 for p in cpaths)
        for mode in MODES:
            paths, costs, npaths, _ = csr.cheapest_k_paths(ps, pd, 1, mode=mode)
            assert paths == [None, None] and costs == [None, None] and npaths.tolist() == [0, 0]
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_row_permutation(gpu_ctx):
    """the ladder's rows shuffled: each row's paths and costs are its own, whatever lane it lands in"""
    name = "ladder"
    c = case(name)
    csr = build(gpu_ctx, name)
    try:
        perm = np.random.default_rng(7).permutation(len(c["rows"]))
        for mode in MODES:
            exp = call(name, 3, mode)
            paths, costs, _, _ = device_call(csr, name, 3, mode, perm)
            assert paths == [exp["paths"][i] for i in perm], mode
            assert bits(costs) == bits([exp["costs"][i] for i in perm]), mode
            opaths, _, _, ost = oracle_call(name, 3, mode, perm)
            assert opaths == paths
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["chunked", "build", "build_device", "upload", "build_keys", "build_keys_device"])
@pytest.mark.parametrize("name", ["chunks_i64", "chunks_f64", "specials_f64", "perm", "modes"])
def test_device_construction_routes(gpu_ctx, name, route):
    from test_gpu_csr_weighted_builds import graph_from_rows, make
    c = case(name)
    gr = graph_from_rows(c["n"], c["src"], c["dst"], c["w"])
    v, e, ids, w = orc.csr_build_weighted(gr.n, gr.src, gr.dst, gr.w, gr.eid)
    csr = make(gpu_ctx, gr, route)
    try:
        for mode in MODES:
            for k in ks_of(name):
                paths, costs, _, _ = csr.cheapest_k_paths(c["ps"], c["pd"], k, c["sv"], c["dv"], mode=mode)
                opaths, ocosts, _, _ = ock.cheapest_k_paths(gr.n, v, e, ids, w, c["ps"], c["pd"], k, mode, c["sv"],
                                                            c["dv"])
                assert paths == opaths and bits(costs) == bits(ocosts), (mode, k)
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ladder", "modes", "perm", "chunks_i64"])
def test_device_identities(gpu_ctx, name):
    """all-0 and all-1 BIGINT weights give shortest_k_paths(mode) at 64 .. 256 lanes; k = 1 gives cheapest_path and
    cheapest_path_length where the latter is defined, with no BIGINT weight above 2^62 (covered(); the finding 2 rows
    are in test_device_findings)"""
    c = case(name)
    src, dst = np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64)
    ok = c["sv"] & c["dv"]
    ps, pd = c["ps"][ok == 1], c["pd"][ok == 1]
    plain = pgq.DeviceCSR.build(gpu_ctx, c["n"], src, dst)
    try:
        for unit in (0, 1):
            csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], src, dst, weight=np.full(len(src), unit, np.int64))
            try:
                for mode in MODES:
                    for lanes in (64, 128, 256):
                        paths, costs, _, _ = csr.cheapest_k_paths(ps, pd, 3, options=pgq.Options(lanes), mode=mode)
                        assert paths == plain.shortest_k_paths(ps, pd, 3, options=pgq.Options(lanes), mode=mode)[0]
                        assert costs == [None if r is None else [unit * (len(q) // 2) for q in r] for r in paths]
            finally:
                csr.free()
    finally:
        plain.free()
    csr = pgq.DeviceCSR.build(gpu_ctx, c["n"], src, dst, weight=covered(c["w"]))
    try:
        cost, cvalid, _ = csr.cheapest_path_length(ps, pd)
        cpaths, _ = csr.cheapest_path(ps, pd)
        for mode in MODES:
            one, one_c, _, _ = csr.cheapest_k_paths(ps, pd, 1, mode=mode)
            assert [r[0] if r else None for r in one] == cpaths, mode
            assert [r[0] if r else None for r in one_c] == [cost[i] if cvalid[i] else None for i in range(len(ps))]
    finally:
        csr.free()


@pytest.mark.gpu
def test_device_lane_cap_at_2p20(gpu_ctx):
    """129 searches in one round: n = 2^20 keeps 256 lanes (one batch), n = 2^20 + 1 gets 128 (two batches)"""
    for name, lanes, batches in (("cap_2p20", 256, 1), ("cap_2p20_1", 128, 2)):
        csr = build(gpu_ctx, name)
        try:
            compare(csr, name, 1, "WALK")
            st = device_call(csr, name, 1, "WALK")[3]
            assert (st["lanes"], st["batches"]) == (lanes, batches), name
        finally:
            csr.free()


@pytest.mark.gpu
def test_device_one_workspace(monkeypatch):
    """one workspace: a 512-lane TRAIL shortest_k_paths on a larger CSR, then a small TRAIL cheapest_k_paths; then the
    other way round -- every WS_KM_* and WS_CK_* slot starts stale"""
    from duckpgq_extension_b200 import datagen
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        n, src, dst = datagen.rmat_edges(12)
        ps, pd = datagen.hashed_pairs(600, n)
        big = pgq.DeviceCSR.build(ctx, n, src, dst)
        ladder_csr = build(ctx, "ladder")
        small = build(ctx, "trail_detour")
        try:
            v, e, ids = orc.csr_build(n, src, dst)
            from oracle import pgq_oracle_kpaths_modes as okm
            exp_big = okm.shortest_k_paths_mode(n, v, e, ids, ps, pd, 2, "TRAIL")[0]
            for order in (("big", "small", "ladder"), ("ladder", "small", "big", "small")):
                for step in order:
                    if step == "big":
                        paths, _, st = big.shortest_k_paths(ps, pd, 2, options=pgq.Options(512), mode="TRAIL")
                        assert paths == exp_big and st["lanes"] == 512
                    elif step == "small":
                        compare(small, "trail_detour", 6, "TRAIL")
                    else:
                        compare(ladder_csr, "ladder", 3, "TRAIL")
        finally:
            for x in (big, ladder_csr, small):
                x.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_device_eight_threads(gpu_ctx):
    name = "ladder"
    csr = build(gpu_ctx, name)
    modes = MODES * 2
    exp = [call(name, 3, m)["paths"] for m in modes]
    out = [None] * 8

    def work(i):
        out[i] = device_call(csr, name, 3, modes[i])[0]

    ths = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    csr.free()
    assert out == exp
