"""iterativelengthbidirectional at the boundaries of the CSR layout and of its meet test, against two restatements.

The bidirectional driver (run_bidir_batch in csrc/pgq_bfs.cu) runs two BFS sides per 512-lane batch, each with its own
mask set, item lists, finished-rows bitmap with snapshots and direction state, and answers rows through k_meet: after a
bottom-up level it scans rows [0, n_ab), after a top-down or tail level the new frontier's item list, both in a
grid-stride loop, and its last block answers the rows that met.  So:

- bidir_run, a numpy restatement of the reference's loop (512 lanes, rows in input order) that shows its work: the
  side, the frontier expanded, the lanes that met with their meet vertices and the stop reason of every batch.  It
  equals oracle/pgq_oracle_bidir.c on every case here (CPU);
- a catalogue of bidirectional boundaries (meet vertex at internal row 0 / n_ab - 1 / on a long row over three ranges /
  on a short row of the last padded slice, seeds without in-edges, meets on either side, last-batch lane counts, met
  lanes 0 / 63 / 64 / 511 next to open ones, every stop reason, coupling across lanes, side frontiers at k_tail's
  limits, and a `wide` shape whose n_ab and item lists exceed k_meet's grid), each proven hit on the CPU;
- on the GPU, every case under forced schedules with the per-iteration trace checked against the restatement, routes,
  the PGQ_B200_PULL_SKIP / PGQ_B200_NO_TAIL switches, one dirty workspace and eight threads on one CSR."""
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_bidir as orb
from test_csr_layout_shapes import CATALOGUE, ROUTES, _oracle, check_download, layout, make, shape

LANES = 512              # LANE_LIMIT of the reference: the lanes of one bidirectional batch
ITEM_EDGES = 256         # PGQ_ITEM_EDGES
TAIL_ITEMS, TAIL_EDGES = 256, 1024  # PGQ_TAIL_ITEMS / PGQ_TAIL_EDGES
H100_SMS = 132           # the H100 SXM; the GPU tests read the device's own count
MEET_BLOCKS_PER_SM = 8   # k_meet's grid: at most SMs x 8 blocks of 256 threads


def meet_grid(sms):
    """Rows or items k_meet covers in one pass of its grid-stride loop."""
    return sms * MEET_BLOCKS_PER_SM * 256


# ---- the restatement that shows its work ----------------------------------------------------------------------------
def bidir_run(n, v, e, src, dst, sv=None, dv=None):
    """The reference's IterativeLengthBidirectionalFunction over the CSR (v, e) as oracle/pgq_oracle_bidir.c reads it:
    rows take lanes in input order, 512 per batch (NULL rows and src == dst take none), iteration i expands side i & 1
    (0 from the sources, 1 from the destinations, both along out-edges), and a lane is answered i + 1 by the first
    iteration after which its two seen sets share a vertex.  -> dict(out, valid, batches, iterations, edges, runs,
    trace): runs[b] = dict(rows, stop, met_at) per batch, trace = one dict per iteration (batch, it, side, fv, fe,
    items, new_items, met = {lane: meet vertices})."""
    v = np.asarray(v, dtype=np.int64)
    e = np.asarray(e, dtype=np.int64)
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    p = len(src)
    ok = np.ones(p, bool)
    if sv is not None:
        ok &= np.asarray(sv) != 0
    if dv is not None:
        ok &= np.asarray(dv) != 0
    lane_rows = np.flatnonzero(ok & (src != dst))
    if len(lane_rows) and (np.any((src[lane_rows] < 0) | (src[lane_rows] >= n)) or
                           np.any((dst[lane_rows] < 0) | (dst[lane_rows] >= n))):
        raise ValueError("source or destination outside [0, n)")
    out = np.full(p, -1, dtype=np.int64)
    valid = np.zeros(p, dtype=np.uint8)
    trivial = ok & (src == dst)
    out[trivial], valid[trivial] = 0, 1
    od = np.diff(v[:n + 1]) if n else np.zeros(0, np.int64)
    items_of = np.maximum(1, -(-od // ITEM_EDGES))
    row = np.repeat(np.arange(n), od)
    order = np.argsort(e, kind="stable")
    pull_src = row[order]                        # the edges by head: tails of each head's in-edges
    heads, starts = np.unique(e[order], return_index=True)
    nl = len(lane_rows)
    # the lane loop stops right behind a batch's 512th lane, so rows behind a full last batch start one more
    n_batches = -(-nl // LANES) + (1 if p and nl % LANES == 0 and (nl == 0 or lane_rows[-1] < p - 1) else 0)
    res = dict(out=out, valid=valid, batches=n_batches, iterations=0, edges=0, runs=[], trace=[])
    for b in range(n_batches):
        rows = lane_rows[b * LANES:(b + 1) * LANES]
        cnt = len(rows)
        run = dict(rows=rows, stop=("no_lanes", -1, -1), met_at=np.full(cnt, -1, np.int64))
        res["runs"].append(run)
        if cnt == 0:
            continue
        words = (cnt + 63) // 64
        lane = np.arange(cnt)
        bit = np.left_shift(np.uint64(1), (lane & 63).astype(np.uint64))
        seen = [np.zeros((n, words), np.uint64) for _ in range(2)]
        visit = [np.zeros((n, words), np.uint64) for _ in range(2)]
        for s, seeds in ((0, src[rows]), (1, dst[rows])):
            np.bitwise_or.at(visit[s], (seeds, lane >> 6), bit)
            np.bitwise_or.at(seen[s], (seeds, lane >> 6), bit)
        open_ = np.ones(cnt, bool)
        it = 0
        while open_.any():
            s = it & 1
            fr = visit[s].any(axis=1)
            rec = dict(batch=b, it=it, side=s, fv=int(fr.sum()), fe=int(od[fr].sum()), items=int(items_of[fr].sum()),
                       new_items=0, met={})
            res["trace"].append(rec)
            res["iterations"] += 1
            res["edges"] += rec["fe"]
            nxt = np.zeros((n, words), np.uint64)
            if len(heads):
                nxt[heads] = np.bitwise_or.reduceat(visit[s][pull_src], starts, axis=0)
            nxt &= ~seen[s]
            seen[s] |= nxt
            visit[s] = nxt
            new = nxt.any(axis=1)
            rec["new_items"] = int(items_of[new].sum())
            if not new.any():  # no lane gained a bit on this side (l.120-127)
                run["stop"] = ("empty", it, s)
                break
            inter = nxt & seen[1 - s]
            hit = np.flatnonzero(inter.any(axis=1))
            if len(hit):
                sub = inter[hit]
                for l in np.flatnonzero(open_):
                    at = (sub[:, l >> 6] >> np.uint64(l & 63)) & np.uint64(1)
                    if at.any():
                        rec["met"][int(l)] = hit[at != 0]
                        r = rows[l]
                        out[r], valid[r] = it + 1, 1
                        open_[l] = False
                        run["met_at"][l] = it
            if not open_.any():
                run["stop"] = ("all_met", it, s)
            it += 1
    return res


def restated(n, v, e, call):
    """bidir_run on the CSR (v, e) for call = (src, dst, sv, dv), once per content (the answer depends on neither the
    schedule nor the route)."""
    src, dst, sv, dv = call
    row = np.repeat(np.arange(n), np.diff(np.asarray(v[:n + 1], dtype=np.int64)))
    canon = np.asarray(e)[np.lexsort((e, row))]  # nothing here depends on the order inside a row
    return _oracle("bidir", lambda: bidir_run(n, v, canon, src, dst, sv, dv), v, canon, src, dst, sv, dv)


# ---- shapes the layout catalogue cannot give ------------------------------------------------------------------------
@dataclass
class BShape:
    n: int
    src: np.ndarray
    dst: np.ndarray
    focus: list = field(default_factory=list)


def _shuffle(rng, n, src, dst):
    p = rng.permutation(n)
    return p, p[np.asarray(src)], p[np.asarray(dst)]


def meet_rows_shape():
    """A sparse graph with every vertex class: 1800 vertices with 1 .. 4 out-edges, 200 sinks (in-edges only), 200
    sources without in-edges and 200 isolated vertices, ids shuffled.  Lengths 1 .. ~12."""
    rng = np.random.default_rng(90)
    body, sinks, outs, n = 1800, 200, 200, 2400
    od = rng.integers(1, 5, body)
    s = np.repeat(np.arange(body), od)
    d = rng.integers(0, body + sinks, len(s))
    s2 = np.repeat(np.arange(body + sinks, body + sinks + outs), 2)
    d2 = rng.integers(0, body, len(s2))
    _, src, dst = _shuffle(rng, n, np.concatenate([s, s2]), np.concatenate([d, d2]))
    return BShape(n, src, dst)


def chain_shape():
    """A path of 600 vertices (ids shuffled) with a few branches off it: lengths up to ~120."""
    rng = np.random.default_rng(91)
    k, n = 600, 700
    s = np.concatenate([np.arange(k - 1), rng.integers(0, k, 100)])
    d = np.concatenate([np.arange(1, k), np.arange(k, n)])
    perm, src, dst = _shuffle(rng, n, s, d)
    return BShape(n, src, dst, focus=[int(x) for x in perm[:k]])  # focus: the path in order


def wide_shape(sms):
    """One hub (no in-edges) over 1.25 x meet_grid(sms) leaves, each leaf with one out-edge into a chain of 64
    vertices.  n_ab > meet_grid: a bottom-up level's meet test takes a second grid-stride pass; the hub's level-1
    frontier is an item list that long, both as the new frontier of the hub's level (the meet test's item scan) and
    as the frontier of the side's next top-down level."""
    rng = np.random.default_rng(92)
    k = meet_grid(sms) + meet_grid(sms) // 4
    zc = 64
    leaves = np.arange(1, k + 1)
    chain = np.arange(k + 1, k + 1 + zc)
    s = np.concatenate([np.zeros(k, np.int64), leaves, chain[:-1]])
    d = np.concatenate([leaves, chain[leaves % zc], chain[1:]])
    n = k + 1 + zc
    perm, src, dst = _shuffle(rng, n, s, d)
    return BShape(n, src, dst, focus=[int(perm[0])] + [int(x) for x in perm[chain]])


# ---- pair sets ------------------------------------------------------------------------------------------------------
class Graph:
    """Out- and in-lists of a shape (original ids)."""

    def __init__(self, sh):
        self.n = sh.n
        self.v, self.e, _ = orc.csr_build(sh.n, sh.src, sh.dst)
        self.lay = layout(sh.n, sh.src, sh.dst)
        order = np.argsort(self.e, kind="stable")
        self.row = np.repeat(np.arange(sh.n), np.diff(self.v[:sh.n + 1]))
        self.in_src = self.row[order]
        self.in_off = np.concatenate([[0], np.cumsum(np.bincount(self.e, minlength=sh.n)[:sh.n])])

    def outs(self, x):
        return self.e[self.v[x]:self.v[x + 1]]

    def ins(self, x):
        return self.in_src[self.in_off[x]:self.in_off[x + 1]]


def _meet_at(g, x):
    """Pairs whose lane meets at x alone: (u, x) with u -> x meets on the source side at iteration 0; (x, w) with
    w -> x, x -/-> w and no other common out-neighbour meets on the destination side at iteration 1."""
    out = []
    preds = [int(u) for u in g.ins(x) if u != x]
    if preds:
        out.append((preds[0], x))
    ox = set(g.outs(x).tolist())
    for w in preds[:64]:
        if w not in ox and not (ox & set(g.outs(w).tolist())) - {x, w}:
            out.append((x, w))
            break
    return out


def targeted(g):
    """Pairs aimed at the boundaries: meets at internal row 0, n_ab - 1, a long row over three ranges and a short row
    of the last slice; seeds without in-edges (class 2) on either side; a sink source next to growing lanes."""
    lay, cls = g.lay, g.lay["cls"]
    inv, n_ab = lay["inv"], lay["n_ab"]
    xs = []
    if n_ab:
        xs += [int(inv[0]), int(inv[n_ab - 1])]
    span = ((lay["ends"] - 1) >> 10) - (lay["starts"] >> 10) >= 2
    xs += [int(x) for x in lay["long_orig"][span][:1]]
    if lay["n_short"]:
        xs.append(int(lay["short_orig"][-1]))
    pairs = []
    for x in xs:
        pairs += _meet_at(g, x)
    for c in np.flatnonzero(cls == 2)[:2]:
        t = int(g.outs(c)[0])
        z = [int(u) for u in g.ins(t) if u != c][:1]
        if z:
            pairs += [(int(c), z[0]), (z[0], int(c))]
    sinks = np.flatnonzero((g.lay["od"] == 0) & (g.lay["ind"] > 0))
    for a in sinks[:2]:
        b = [int(u) for u in g.ins(a) if u != a][:1]
        if b:
            pairs.append((int(a), b[0]))  # alone: NULL (the source side dies at iteration 0)
    return pairs


def never_meet(g, k, rng):
    """k pairs whose lanes can never meet: both seeds without out-edges, or one of them isolated."""
    dead = np.flatnonzero(g.lay["od"] == 0)
    if len(dead) < 2:
        return []
    a = rng.choice(dead, k)
    b = rng.choice(dead, k)
    b = np.where(a == b, dead[(np.searchsorted(dead, a) + 1) % len(dead)], b)
    return list(zip(a.tolist(), b.tolist()))


def random_pairs(g, k, rng):
    n = g.n
    if n < 2:
        return []
    has_out = np.flatnonzero(g.lay["od"] > 0)
    has_in = np.flatnonzero(g.lay["ind"] > 0)
    s = rng.choice(has_out, k) if len(has_out) else rng.integers(0, n, k)
    d = np.where(rng.random(k) < 0.7, rng.choice(has_in, k) if len(has_in) else rng.integers(0, n, k),
                 rng.integers(0, n, k))
    d = np.where(d == s, (d + 1) % n, d)
    return list(zip(s.tolist(), d.tolist()))


def with_lanes(pairs, lanes, rng, extra=True):
    """A call of exactly `lanes` lane rows (pairs first, in order; random pairs make up the rest) with NULL-source,
    NULL-destination and src == dst rows inserted among them -> (src, dst, sv, dv)."""
    pairs = list(pairs)[:lanes]
    src = [p[0] for p in pairs]
    dst = [p[1] for p in pairs]
    sv = [1] * len(src)
    dv = [1] * len(src)
    if extra:
        for kind in (0, 0, 1, 1, 2, 2):
            i = int(rng.integers(0, len(src) + 1))
            x = int(src[i % len(src)]) if src else 0
            src.insert(i, x)
            dst.insert(i, x if kind == 2 else int(dst[i % len(dst)]) if dst else 0)
            sv.insert(i, 0 if kind == 0 else 1)
            dv.insert(i, 0 if kind == 1 else 1)
    return (np.array(src, np.int64), np.array(dst, np.int64), np.array(sv, np.uint8), np.array(dv, np.uint8))


LAST_BATCH = [1, 63, 64, 65, 511, 512]


def main_call(g, idx):
    """Targeted pairs, then random ones, 512 + LAST_BATCH[idx % 6] lanes (64 on the big shapes)."""
    rng = np.random.default_rng(700 + idx)
    lanes = LANES + LAST_BATCH[idx % len(LAST_BATCH)] if g.n <= 40000 else 64
    pairs = targeted(g)
    pairs += random_pairs(g, lanes - len(pairs), rng)
    if len(pairs) < lanes:  # (a graph of one vertex has no lane at all)
        return with_lanes(pairs, len(pairs), rng)
    return with_lanes(pairs, lanes, rng)


def lane_pattern_call(g, rng):
    """Two full batches: lanes 0, 63 and 511 of the first and lane 64 of the second meet (length 1) while their
    neighbours can never meet."""
    meet = [pr for x in rng.permutation(np.flatnonzero(g.lay["ind"] > 0))[:64] for pr in _meet_at(g, int(x))[:1]]
    pairs = random_pairs(g, 2 * LANES, rng)
    dead = never_meet(g, 8, rng)
    for lane, pr in zip((0, 63, 511, LANES + 64), meet):
        pairs[lane] = pr
    for lane, pr in zip((1, 62, 64, 510, LANES + 63, LANES + 65), dead):
        pairs[lane] = pr
    return with_lanes(pairs, 2 * LANES, rng)


def stop_calls(g, rng):
    """A batch whose source side is empty at iteration 0 (every source a sink: no lane meets), and one lane whose
    destination side is empty at iteration 1 (a sink destination the source does not reach in one step)."""
    out = []
    dead = never_meet(g, 5, rng)
    if dead:
        out.append(with_lanes(dead, len(dead), rng, extra=False))
    sinks = np.flatnonzero((g.lay["od"] == 0) & (g.lay["ind"] > 0))
    for u in np.flatnonzero(g.lay["od"] > 0)[:50]:
        a = [int(x) for x in sinks if x not in set(g.outs(u).tolist())][:1]
        if a:
            out.append(with_lanes([(int(u), a[0])], 1, rng, extra=False))
            break
    return out


def tail_hub_calls(sh, g):
    """outdeg_tail: per tail hub one call whose lanes all start at the hub and one whose lanes all end there, so that
    the side's second level expands exactly the hub's leaves (256 / 257 items, 1024 / 1025 edges)."""
    out = []
    rng = np.random.default_rng(95)
    far = np.array([x for x in range(2000) if g.lay["od"][x] > 0])  # the body graph, away from the hubs
    for h in sh.tail:
        others = rng.choice(far, 12, replace=False)
        out.append(with_lanes([(h, int(x)) for x in others], 12, rng, extra=False))
        out.append(with_lanes([(int(x), h) for x in others], 12, rng, extra=False))
    return out


def chain_calls(sh, g):
    path = sh.focus
    pairs = [(path[i], path[i + d]) for i, d in ((0, 25), (3, 60), (100, 1), (200, 7))]
    pairs += [(path[i + d], path[i]) for i, d in ((10, 30), (300, 2))]
    rng = np.random.default_rng(96)
    return [with_lanes(pairs + random_pairs(g, 40, rng), 46, rng)]


def wide_calls(sh, g, sms):
    """64 lanes from the hub: to leaves at internal rows beyond one grid pass and below it, and into the chain."""
    lay = g.lay
    pos = np.empty(sh.n, np.int64)
    pos[lay["inv"]] = np.arange(sh.n)
    hub, chain = sh.focus[0], sh.focus[1:]
    leaves = g.outs(hub)
    rng = np.random.default_rng(97)
    beyond = rng.choice(leaves[pos[leaves] >= meet_grid(sms)], 24, replace=False)
    below = rng.choice(leaves[pos[leaves] < meet_grid(sms)], 8, replace=False)
    pairs = [(hub, int(x)) for x in np.concatenate([beyond, below])]
    pairs += [(hub, int(chain[i])) for i in range(32, 64, 4)]
    pairs += [(int(x), int(chain[-1])) for x in rng.choice(leaves, 12, replace=False)]
    pairs += [(int(chain[0]), int(x)) for x in beyond[:10]]
    return [with_lanes(pairs, len(pairs), rng)]


# ---- the catalogue --------------------------------------------------------------------------------------------------
NEW_SHAPES = {"meet_rows": meet_rows_shape, "chain": chain_shape}
CASES = list(CATALOGUE) + list(NEW_SHAPES) + ["wide"]


@dataclass
class Case:
    sh: object
    g: Graph
    calls: list
    sms: int = 0


_cases = {}


def case(name, sms=H100_SMS):
    key = (name, sms if name == "wide" else 0)
    if key not in _cases:
        if name == "wide":
            sh = wide_shape(sms)
        elif name in NEW_SHAPES:
            sh = NEW_SHAPES[name]()
        else:
            sh = shape(name)
        g = Graph(sh)
        rng = np.random.default_rng(800 + CASES.index(name))
        if name == "wide":
            calls = wide_calls(sh, g, sms)
        elif name == "chain":
            calls = chain_calls(sh, g)
        else:
            calls = [main_call(g, CASES.index(name))]
        if name == "outdeg_tail":
            calls += tail_hub_calls(sh, g)
        if name == "meet_rows":
            calls += [lane_pattern_call(g, rng), with_lanes(random_pairs(g, 8, rng), 8, rng)] + stop_calls(g, rng)
        _cases[key] = Case(sh, g, calls, sms if name == "wide" else 0)
    return _cases[key]


def bidir_hits(c, results):
    """Every bidirectional boundary the calls of case c hit, by name (results: bidir_run's answer per call)."""
    lay = c.g.lay
    n, n_ab, cls, inv = lay["n"], lay["n_ab"], lay["cls"], lay["inv"]
    pos = np.empty(n, np.int64)
    pos[inv] = np.arange(n)
    span = ((lay["ends"] - 1) >> 10) - (lay["starts"] >> 10) >= 2
    long3 = set(lay["long_orig"][span].tolist())
    last_slice = set()
    if lay["n_short"]:
        first = (lay["n_short"] - 1) // 32 * 32
        rows = lay["short_orig"][first:]
        if len(rows) < 32 or np.any(lay["ind"][rows] < lay["widths"][-1]):
            last_slice = set(rows.tolist())
    grid = meet_grid(c.sms) if c.sms else None
    out = set()
    if grid and n_ab > grid:
        out.add("wide_nab_beyond_grid")
    for (src, dst, _, _), res in zip(c.calls, results):
        runs = res["runs"]
        full = [r for r in runs if len(r["rows"])]
        if full and len(full[-1]["rows"]) in LAST_BATCH:
            out.add(f"last_batch_lanes_{len(full[-1]['rows'])}")
        for r in full:
            met_at = r["met_at"]
            cnt = len(met_at)
            if not np.any(met_at >= 0):
                out.add("no_meet_batch")
            for lane in (0, 63, 64, 511):
                nb = [x for x in (lane - 1, lane + 1) if 0 <= x < cnt]
                if lane < cnt and met_at[lane] >= 0 and nb and all(met_at[x] < 0 for x in nb):
                    out.add(f"met_lane_{lane}_neighbours_open")
            reason, it, side = r["stop"]
            if reason == "all_met":
                out.add("stop_all_met")
            elif reason == "empty":
                if it == 0 and side == 0:
                    out.add("stop_src_empty_it0")
                if it == 1 and side == 1:
                    out.add("stop_dst_empty_it1")
                if it >= 3 and np.any(met_at < 0):
                    out.add("stop_empty_open_depth3")
        for rec in res["trace"]:
            rows = runs[rec["batch"]]["rows"]
            for kind, val, lim in (("items", rec["items"], TAIL_ITEMS), ("edges", rec["fe"], TAIL_EDGES)):
                if val in (lim, lim + 1):
                    out.add(f"tail_{kind}_{val}_{'dst' if rec['side'] else 'src'}")
            if grid and rec["new_items"] > grid:
                out.add("wide_new_items_beyond_grid")
            if grid and rec["items"] > grid:
                out.add("wide_frontier_items_beyond_grid")
            for lane, verts in rec["met"].items():
                s, d = src[rows[lane]], dst[rows[lane]]
                out.add("meet_dst_side" if rec["side"] else "meet_src_side")
                if rec["it"] == 0:
                    out.add("len_1")
                if rec["it"] + 1 >= 40:
                    out.add("len_ge_40")
                if pos[d] >= n_ab:
                    out.add("dst_seed_beyond_nab_meets")
                if pos[s] >= n_ab:
                    out.add("src_seed_beyond_nab_meets")
                if len(verts) != 1:
                    continue
                x = int(verts[0])
                if pos[x] == 0:
                    out.add("meet_row_0")
                if pos[x] == n_ab - 1:
                    out.add("meet_row_last_in_only" if cls[x] == 1 else "meet_row_last")
                if x in long3:
                    out.add("meet_long_3_ranges")
                if x in last_slice:
                    out.add("meet_short_last_slice")
                if grid and pos[x] >= grid:
                    out.add("wide_meet_row_beyond_grid")
    return out


def coupled_rows(c, results):
    """Rows whose answer differs from their answer when run alone (among the rows with a sink source, at most 4)."""
    out = []
    v, e = c.g.v, c.g.e
    for (src, dst, sv, dv), res in zip(c.calls, results):
        for r in np.flatnonzero((sv == 1) & (dv == 1) & (src != dst)):
            if c.g.lay["od"][src[r]] == 0 and c.g.lay["ind"][src[r]] > 0 and len(out) < 4:
                alone = bidir_run(c.sh.n, v, e, src[r:r + 1], dst[r:r + 1])
                if (alone["out"][0], alone["valid"][0]) != (res["out"][r], res["valid"][r]):
                    out.append(r)
    return out


# the boundaries each case is named for (test_bidir_catalogue_hits_its_boundaries proves them hit)
NAMED = {
    "split_m0": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_1", "len_1", "meet_dst_side", "meet_row_0",
                 "meet_row_last_in_only", "meet_src_side", "src_seed_beyond_nab_meets", "stop_all_met"},
    "split_m1": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_63", "len_1", "meet_dst_side",
                 "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                 "src_seed_beyond_nab_meets", "stop_all_met"},
    "split_m31": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_64", "len_1", "meet_dst_side",
                  "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                  "src_seed_beyond_nab_meets", "stop_all_met"},
    "long_m1": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_65", "len_1", "meet_dst_side",
                "meet_long_3_ranges", "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                "src_seed_beyond_nab_meets", "stop_all_met", "stop_empty_open_depth3"},
    "long_0": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_511", "len_1", "meet_dst_side",
               "meet_long_3_ranges", "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
               "src_seed_beyond_nab_meets", "stop_all_met", "stop_empty_open_depth3"},
    "long_p1": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_512", "len_1", "meet_dst_side",
                "meet_long_3_ranges", "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                "src_seed_beyond_nab_meets", "stop_empty_open_depth3"},
    "outdeg_tail": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_1", "len_1", "meet_dst_side",
                    "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                    "src_seed_beyond_nab_meets", "stop_all_met", "stop_empty_open_depth3", "tail_edges_1024_dst",
                    "tail_edges_1024_src", "tail_edges_1025_dst", "tail_edges_1025_src", "tail_items_256_dst",
                    "tail_items_256_src", "tail_items_257_dst", "tail_items_257_src"},
    "bipartite": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_63", "len_1", "meet_dst_side",
                  "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                  "src_seed_beyond_nab_meets"},
    "selfloops": {"last_batch_lanes_64", "no_meet_batch", "stop_src_empty_it0"},
    "inonly_isolated": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_65", "len_1", "meet_dst_side",
                        "meet_long_3_ranges", "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice",
                        "meet_src_side", "src_seed_beyond_nab_meets", "stop_empty_open_depth3"},
    "n1": set(),
    "n2": {"last_batch_lanes_512", "len_1", "meet_row_0", "meet_row_last", "meet_short_last_slice", "meet_src_side",
           "stop_all_met"},
    "n32": {"last_batch_lanes_1", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_short_last_slice",
            "meet_src_side", "stop_all_met"},
    "n33": {"last_batch_lanes_63", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_short_last_slice",
            "meet_src_side", "stop_all_met"},
    "n1024": {"last_batch_lanes_64", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_src_side",
              "stop_all_met", "tail_edges_1024_dst"},
    "n1025": {"last_batch_lanes_65", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_short_last_slice",
              "meet_src_side", "stop_all_met"},
    "n2047": {"last_batch_lanes_511", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_short_last_slice",
              "meet_src_side", "stop_all_met"},
    "n2048": {"last_batch_lanes_512", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_src_side",
              "stop_all_met"},
    "n32768": {"last_batch_lanes_1", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_src_side",
               "stop_all_met"},
    "n32769": {"last_batch_lanes_63", "len_1", "meet_dst_side", "meet_row_0", "meet_row_last", "meet_short_last_slice",
               "meet_src_side", "stop_all_met"},
    "multigraph": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_64", "len_1", "meet_dst_side",
                   "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                   "src_seed_beyond_nab_meets", "stop_all_met"},
    "lcc": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_65", "len_1", "meet_dst_side", "meet_row_0",
            "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side", "src_seed_beyond_nab_meets",
            "stop_all_met"},
    "empty_n1": set(),
    "empty_n5": {"last_batch_lanes_512", "no_meet_batch", "stop_src_empty_it0"},
    "meet_rows": {"coupling", "dst_seed_beyond_nab_meets", "last_batch_lanes_1", "last_batch_lanes_512", "len_1",
                  "meet_dst_side", "meet_row_0", "meet_row_last_in_only", "meet_short_last_slice", "meet_src_side",
                  "met_lane_0_neighbours_open", "met_lane_511_neighbours_open", "met_lane_63_neighbours_open",
                  "met_lane_64_neighbours_open", "no_meet_batch", "src_seed_beyond_nab_meets", "stop_all_met",
                  "stop_dst_empty_it1", "stop_empty_open_depth3", "stop_src_empty_it0"},
    "chain": {"len_1", "len_ge_40", "meet_dst_side", "meet_short_last_slice", "meet_src_side",
              "src_seed_beyond_nab_meets", "stop_empty_open_depth3"},
    "wide": {"len_1", "len_ge_40", "meet_long_3_ranges", "meet_row_last_in_only", "meet_src_side",
             "src_seed_beyond_nab_meets", "stop_all_met", "wide_frontier_items_beyond_grid",
             "wide_meet_row_beyond_grid", "wide_nab_beyond_grid", "wide_new_items_beyond_grid"},
}

REQUIRED = (
    {"meet_row_0", "meet_row_last", "meet_row_last_in_only", "meet_long_3_ranges", "meet_short_last_slice",
     "dst_seed_beyond_nab_meets", "src_seed_beyond_nab_meets", "meet_src_side", "meet_dst_side", "len_1",
     "len_ge_40", "no_meet_batch", "stop_all_met", "stop_src_empty_it0", "stop_dst_empty_it1",
     "stop_empty_open_depth3", "coupling", "wide_nab_beyond_grid", "wide_new_items_beyond_grid",
     "wide_frontier_items_beyond_grid", "wide_meet_row_beyond_grid"}
    | {f"last_batch_lanes_{k}" for k in LAST_BATCH}
    | {f"met_lane_{k}_neighbours_open" for k in (0, 63, 64, 511)}
    | {f"tail_{kind}_{val}_{side}" for kind, vals in (("items", (256, 257)), ("edges", (1024, 1025)))
       for val in vals for side in ("src", "dst")}
)


def case_results(c):
    return [restated(c.sh.n, c.g.v, c.g.e, call) for call in c.calls]


# ---- CPU: the two restatements agree; the catalogue hits what it names ------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_restatements_agree(name):
    c = case(name)
    for call, res in zip(c.calls, case_results(c)):
        o, ov, st = orb.iterativelengthbidirectional(c.sh.n, c.g.v, c.g.e, *call)
        assert np.array_equal(res["valid"], ov) and np.array_equal(res["out"], o)
        assert (res["batches"], res["iterations"], res["edges"]) == (st.batches, st.iterations, st.edges_traversed)
        assert len(res["trace"]) == res["iterations"]


@pytest.mark.parametrize("name", CASES)
def test_bidir_catalogue_hits_its_boundaries(name):
    c = case(name)
    results = case_results(c)
    got = bidir_hits(c, results)
    if coupled_rows(c, results):
        got.add("coupling")
    want = NAMED.get(name, set())
    print(f"{name}: n={c.sh.n} n_ab={c.g.lay['n_ab']} calls={len(c.calls)} hits {sorted(got)}")
    assert want <= got, sorted(want - got)


def test_bidir_catalogue_covers_every_boundary():
    named = set().union(*NAMED.values())
    assert REQUIRED <= named, sorted(REQUIRED - named)


# ---- GPU ------------------------------------------------------------------------------------------------------------
TRACE = re.compile(r"\[pgq\] batch (\d+) iteration (\d+) (src|dst) side (push|pull|tail) frontier_v=(\d+) "
                   r"frontier_e=(\d+) items=(-?\d+)")
# (bbbbbbp: each side runs three bottom-up levels before a top-down one)
SCHEDULES = ["a", "b", "p", "t", "bp", "pb", "tp", "pt", "tb", "bt", "bbp", "ppb", "tpb", "bbbbbbp"]


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_and_check(csr, n, v, e, call, options=None):
    """One call on the device against the restatement: results, counters and lanes."""
    res = restated(n, v, e, call)
    out, valid, st = csr.iterativelengthbidirectional(*call, options)
    assert np.array_equal(valid, res["valid"]), np.flatnonzero(valid != res["valid"])[:10]
    assert np.array_equal(out, res["out"]), np.flatnonzero(out != res["out"])[:10]
    assert (st["batches"], st["levels"], st["edges_traversed"]) == (res["batches"], res["iterations"], res["edges"])
    assert st["lanes"] == LANES
    return res


def check_trace(err, res, schedule, m, use_tail=True):
    """Every iteration's trace line: batch and iteration in the restatement's order, the side of the iteration's
    parity, the forced kind where it is eligible, and the frontier the restatement expanded: its vertices, out-edges
    and work items -> [(kind, side, it, batch)].  The items are exact except on a bottom-up level that follows
    another one, which has no item list and shows the bound fv + fe / 256; a top-down or tail level behind a
    bottom-up one lists its frontier from the masks first, so stale bits of a finished row would show there."""
    lines = [TRACE.match(x) for x in err.splitlines()]
    lines = [x for x in lines if x]
    assert len(lines) == len(res["trace"])
    prev = {}  # side -> (kind, fv, fe) of the side's last level in this batch
    kinds = []
    for mt, rec in zip(lines, res["trace"]):
        batch, it, side, kind = int(mt.group(1)), int(mt.group(2)), mt.group(3), mt.group(4)
        fv, fe, items = int(mt.group(5)), int(mt.group(6)), int(mt.group(7))
        assert (batch, it) == (rec["batch"] + 1, rec["it"])
        assert side == ("dst" if it & 1 else "src")
        assert (fv, fe) == (rec["fv"], rec["fe"]), (it, side, fv, fe, rec["fv"], rec["fe"])
        if it == 0:
            prev = {}
        # after a bottom-up level the side has no item list: k_tail is judged on the bound fv + fe / 256
        last = prev.get(side)
        n_items = fv + fe // ITEM_EDGES if last == "pull" else rec["items"]
        assert items == (n_items if kind == "pull" else rec["items"]), (it, side, kind, items, n_items, rec["items"])
        want = schedule[it % len(schedule)]
        if want == "p":
            assert kind == "push", (it, kind)
        elif want == "b":
            assert kind == ("pull" if m else "push"), (it, kind)
        elif want == "t":
            eligible = use_tail and n_items <= TAIL_ITEMS and fe <= TAIL_EDGES
            assert kind == ("tail" if eligible else "push"), (it, kind, n_items, fe)
        if not use_tail:
            assert kind != "tail"
        prev[side] = kind
        kinds.append((kind, side, it, rec["batch"]))
    return kinds


@pytest.fixture(scope="module")
def sms():
    return device_sms()


def _case_gpu(name, sms):
    c = case(name, sms)
    if name == "wide":
        assert c.g.lay["n_ab"] > meet_grid(sms)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_bidir_shape_schedules(gpu_ctx, monkeypatch, capfd, sms, name):
    """Every case built by pgq_csr_build, under every schedule: answers and counters equal the restatement's, and
    each iteration's trace line shows the side, the forced kind and the frontier the restatement expanded."""
    c = _case_gpu(name, sms)
    csr = pgq.DeviceCSR.build(gpu_ctx, c.sh.n, c.sh.src, c.sh.dst)
    try:
        v, e, _ = csr.download()
        assert np.array_equal(v, c.g.v)
        monkeypatch.setenv("PGQ_B200_TRACE", "1")
        for schedule in SCHEDULES:
            monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
            for call in c.calls:
                capfd.readouterr()
                res = run_and_check(csr, c.sh.n, v, e, call)
                check_trace(capfd.readouterr().err, res, schedule, len(e))
    finally:
        csr.free()


@pytest.mark.gpu
def test_mixed_schedules_meet_in_every_kind(gpu_ctx, monkeypatch, capfd):
    """meet_rows under the six two-character mixed schedules: between them, meets are found in push, pull and tail
    levels of both sides (the restatement says which iteration met, the trace which kind of level ran it)."""
    c = case("meet_rows")
    csr = pgq.DeviceCSR.build(gpu_ctx, c.sh.n, c.sh.src, c.sh.dst)
    found = set()
    try:
        v, e, _ = csr.download()
        monkeypatch.setenv("PGQ_B200_TRACE", "1")
        for schedule in ["bp", "pb", "tp", "pt", "tb", "bt"]:
            monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
            for call in c.calls:
                capfd.readouterr()
                res = run_and_check(csr, c.sh.n, v, e, call)
                kinds = check_trace(capfd.readouterr().err, res, schedule, len(e))
                for (kind, side, _, _), rec in zip(kinds, res["trace"]):
                    if rec["met"]:
                        found.add((kind, side))
    finally:
        csr.free()
    assert found == {(k, s) for k in ("push", "pull", "tail") for s in ("src", "dst")}, sorted(found)


def _relabel(sh, k):
    if k == 0:
        return sh
    rng = np.random.default_rng(600 + k)
    p = rng.permutation(sh.n)
    return BShape(sh.n, p[sh.src], p[sh.dst])


def _relabel_calls(calls, perm):
    return [(perm[s], perm[d], sv, dv) for s, d, sv, dv in calls]


ROUTE_CASES = ["split_m1", "long_0", "bipartite", "inonly_isolated", "meet_rows"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["device", "chunked8", "upload_noids", "keys", "clone"])
@pytest.mark.parametrize("name", ROUTE_CASES)
def test_bidir_routes(gpu_ctx, monkeypatch, name, route):
    """The same answers from a CSR built on the device, fed in chunks by eight threads, uploaded without edge ids,
    built from signed sparse key columns, and from a clone called after its primary was freed and a CSR of the same
    sizes took the primary's buffers."""
    c = case(name)
    sh = c.sh
    live, ctxs = [], []
    try:
        if route in ROUTES:
            csr, exp, exact = make(gpu_ctx, sh, route)
            live.append(csr)
            v, e, _, _ = check_download(csr, sh, exp, exact)
        elif route == "keys":
            keys = np.random.default_rng(31).choice(1 << 40, sh.n, replace=False).astype(np.int64) - (1 << 39)
            csr = pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys[sh.src], keys[sh.dst])
            live.append(csr)
            v, e, _ = csr.download()
            assert np.array_equal(v, c.g.v)
        else:
            ctx_a, ctx_b = pgq.Context(0), pgq.Context(0)
            ctxs += [ctx_a, ctx_b]
            prim = pgq.DeviceCSR.build(ctx_a, sh.n, sh.src, sh.dst)
            csr = prim.clone(ctx_b)
            live.append(csr)
            prim.free()
            other_sh = _relabel(sh, 1)
            other = pgq.DeviceCSR.build(ctx_a, other_sh.n, other_sh.src, other_sh.dst)
            live.append(other)
            for call in c.calls[:1]:  # the freed primary's buffers are busy with other contents
                ov, oe, _ = other.download()
                run_and_check(other, sh.n, ov, oe, call)
            v, e, _ = csr.download()
            assert np.array_equal(v, c.g.v)
        for schedule in ("a", "b", "pt"):
            monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
            for call in c.calls:
                run_and_check(csr, sh.n, v, e, call)
    finally:
        for x in live:
            x.free()
        for x in ctxs:
            x.close()


@pytest.mark.gpu
@pytest.mark.parametrize("env", [("PGQ_B200_PULL_SKIP", "0"), ("PGQ_B200_NO_TAIL", "1")])
@pytest.mark.parametrize("name", ["split_m0", "long_p1", "outdeg_tail", "meet_rows", "chain"])
def test_bidir_switches(gpu_ctx, monkeypatch, capfd, name, env):
    """The same answers with finished rows never skipped, and with k_tail switched off (then no level is a tail)."""
    c = case(name)
    monkeypatch.setenv(*env)
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    csr = pgq.DeviceCSR.build(gpu_ctx, c.sh.n, c.sh.src, c.sh.dst)
    try:
        v, e, _ = csr.download()
        for schedule in ("a", "b", "t", "bt"):
            monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
            for call in c.calls:
                capfd.readouterr()
                res = run_and_check(csr, c.sh.n, v, e, call)
                check_trace(capfd.readouterr().err, res, schedule, len(e), use_tail=env[0] != "PGQ_B200_NO_TAIL")
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["meet_rows", "bipartite", "split_m31"])
def test_bidir_one_workspace(monkeypatch, name):
    """A context with one workspace: CSRs of equal sizes (relabelled) in a row, each taking the freed buffers of the
    one before, and on each bidirectional, iterativelength (default and reference batching), shortestpath and
    bidirectional again on the same dirty buffers.  The first bidirectional call is one batch whose seeds include
    vertices beyond n_ab, and iterativelength runs right behind it."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    base = case(name)
    try:
        size = None
        for k in range(3):
            rng = np.random.default_rng(900 + k)
            perm = np.arange(base.sh.n) if k == 0 else np.random.default_rng(600 + k).permutation(base.sh.n)
            sh = _relabel(base.sh, k)
            calls = _relabel_calls(base.calls, perm)
            lay = layout(sh.n, sh.src, sh.dst)
            beyond = np.flatnonzero(lay["cls"] >= 2)
            g_pairs = [(int(perm[a]), int(perm[b])) for a, b in targeted(base.g)]
            g_pairs = [pr for pr in g_pairs if lay["cls"][pr[0]] >= 2 or lay["cls"][pr[1]] >= 2] or \
                [(int(beyond[0]), int(beyond[1]))]
            first = with_lanes(g_pairs + [(int(a), int(b)) for a, b in zip(rng.choice(sh.n, 40), rng.choice(sh.n, 40))
                                          if a != b], 40, rng, extra=False)
            assert np.any(lay["cls"][np.concatenate(first[:2])] >= 2)  # seeds beyond n_ab
            csr = pgq.DeviceCSR.build(ctx, sh.n, sh.src, sh.dst)
            try:
                if size is None:
                    size = csr.info()[2]
                assert csr.info()[2] == size
                v, e, ids = csr.download()
                run_and_check(csr, sh.n, v, e, first)
                ps, pd = calls[0][0], calls[0][1]
                sv = (calls[0][2] & calls[0][3]).astype(np.uint8)
                o, ov, ost = _oracle("il", lambda: orc.iterativelength(sh.n, v, e, ps, pd, sv, 512), v, e, ps, pd, sv, 512)
                out, valid, _ = csr.iterativelength(ps, pd, sv)
                assert np.array_equal(valid, ov) and np.array_equal(out, o)
                out, valid, st = csr.iterativelength(ps, pd, sv, pgq.Options(512, reference_batching=True))
                assert np.array_equal(valid, ov) and np.array_equal(out, o)
                assert (st["batches"], st["levels"], st["edges_traversed"]) == (ost.batches, ost.levels,
                                                                                ost.edges_traversed)
                q = slice(0, 100)
                paths, _ = csr.shortestpath(ps[q], pd[q], sv[q])
                assert paths == _oracle("sp", lambda: orc.shortestpath(sh.n, v, e, ids, ps[q], pd[q], sv[q], 512)[0],
                                        v, e, ids, ps[q], pd[q], sv[q])
                for call in calls:
                    run_and_check(csr, sh.n, v, e, call)
                out, valid, _ = csr.iterativelength(ps, pd, sv)
                assert np.array_equal(valid, ov) and np.array_equal(out, o)
            finally:
                csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_bidir_eight_threads_one_csr(gpu_ctx):
    """Eight threads on one CSR, each with its own pairs, alternating bidirectional and iterativelength calls."""
    c = case("meet_rows")
    n = c.sh.n
    csr = pgq.DeviceCSR.build(gpu_ctx, n, c.sh.src, c.sh.dst)
    try:
        v, e, _ = csr.download()
        work = []
        for t in range(8):
            rng = np.random.default_rng(1000 + t)
            call = with_lanes(random_pairs(c.g, 300 + 100 * t, rng), 300 + 100 * t, rng)
            ps, pd = call[0], call[1]
            sv = (call[2] & call[3]).astype(np.uint8)
            work.append((call, restated(n, v, e, call), orc.iterativelength(n, v, e, ps, pd, sv, 512)))

        def body(t):
            call, res, (o, ov, _) = work[t]
            ps, pd = call[0], call[1]
            sv = (call[2] & call[3]).astype(np.uint8)
            for _ in range(3):
                out, valid, st = csr.iterativelengthbidirectional(*call)
                assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"])
                assert (st["batches"], st["levels"], st["edges_traversed"]) == (res["batches"], res["iterations"],
                                                                                res["edges"])
                out, valid, _ = csr.iterativelength(ps, pd, sv)
                assert np.array_equal(valid, ov) and np.array_equal(out, o)
            return t

        with ThreadPoolExecutor(max_workers=8) as pool:
            assert sorted(pool.map(body, range(8))) == list(range(8))
    finally:
        csr.free()
