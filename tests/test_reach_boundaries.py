"""reachability at the boundaries of its reference batches, its reach-mode switches and the stale rows it clears,
against a restatement that shows its batches.

pgq_reachability with PGQ_OPT_REFERENCE_BATCHING (csrc/pgq_api.cu, pgq_bfs_reachability_device in csrc/pgq_bfs.cu)
adds three things to the shared call driver, and a fault in any of them changes no answer on the R-MAT pairs of
tests/test_gpu_reachability.py -- only searches / levels / edges_traversed, or an answer on a shape R-MAT rarely makes:

- the host cut: the API replaces a NULL destination by its source, then a scan cuts the rows into chunks (a new valid
  source opens the next lane, the chunk ends behind the row that opened lane 512), each chunk its own run_call;
- CallCtx::reach: src == dst rows search on their source's lane (AssignArgs::trivial_lanes), sources are seen from the
  start (mark_seen), and a batch runs until a level adds no bit (stop_answered = 0, on the host and in k_tail);
- the cleanup of seen rows from n_ab on: a source without in-edges is seen on its lane, and a later batch on the same
  workspace clears only the rows below n_ab, where a BFS level can write.

So:
- reach_run, a numpy restatement that shows its work: the API step (valid rows, the NULL-destination rewrite); per
  chunk its rows, every row's lane, the lane sources and why the cut ended; per chunk and level the frontier, its
  out-edges and work items and the rows answered; per call the summed counters.  It equals oracle/pgq_oracle_reach.c
  (defined batch start) and scipy's reachability on every case; the default mode is driver_run's iterativelength;
- a catalogue of cases that each name what they hit, proven on the CPU from reach_run and layout();
- on the GPU every case in both modes with answers, counters and every PGQ_B200_TRACE line, forced schedules and the
  level-loop switches, every construction route, one workspace shared with every BFS consumer, and eight threads."""
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np
import pytest
from scipy.sparse.csgraph import shortest_path as sp_shortest_path

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle_bidir as orb
from oracle import pgq_oracle_reach as orr
from test_call_driver_boundaries import (CALL, COUNTERS, LEVEL, NO_PRUNE, REF, Graph, RangeError, check_trace,
                                         counters, driver_run, options)
from test_csr_layout_shapes import CATALOGUE, ROUTES, Shape, _oracle, layout, make
from test_csr_layout_shapes import shape as layout_shape

L = 512                     # LANE_LIMIT: lanes of a reference batch
ITEM_EDGES = 256            # PGQ_ITEM_EDGES
TAIL_MAX = 32               # PGQ_TAIL_MAX: levels one k_tail launch may run
TAIL_ITEMS, TAIL_EDGES = 256, 1024  # k_tail takes a level with at most this many work items and out-edges
SCHEDULES = ["b", "p", "t", "bp", "pb", "tbp", "ppbb", "bbbt"]  # (from tests/test_bfs_schedules.py's FIXED)
GARBAGE = (-1, 1 << 40, -(1 << 33))  # ids under a NULL: never read


def graph(n, src_e, dst_e):
    return _oracle("reach_graph", lambda: Graph(n, src_e, dst_e), n, np.asarray(src_e), np.asarray(dst_e))


# ---- the restatement that shows its work ------------------------------------------------------------------------------
def reach_run(n, src_e, dst_e, ps, pd, sv=None, dv=None, ref=True, lanes=0):
    """pgq_reachability restated from the edge rows -> dict.
    API step  valid (both ids valid), sdst (the searched destination: a NULL one replaced by the source); a valid id
              outside [0, n) raises RangeError, in either position, whatever the other id is;
    default   (ref=False) driver_run's iterativelength with flags 0 over the valid rows: its dict, with out = reached
              and valid, valid = both ids valid;
    per chunk chunks[c] = dict(b0, end, rows, lane (per row, -1 = NULL source), lane_src, cut ("lane_512_opened" or
              "end_of_rows"), searches, search_rows, answered_at (per row: the level that found it, 0 = at the
              start, -1 = never), levels = [dict(level, fv, fe, items, answered rows)], stop);
    per call  out, valid, searches, pruned (0), search_rows, lanes (512), batches, levels, edges, fv."""
    ps, pd = np.asarray(ps, dtype=np.int64), np.asarray(pd, dtype=np.int64)
    p = len(ps)
    sok = np.ones(p, bool) if sv is None else np.asarray(sv) != 0
    dok = np.ones(p, bool) if dv is None else np.asarray(dv) != 0
    if np.any(sok & ((ps < 0) | (ps >= n))) or np.any(dok & ((pd < 0) | (pd >= n))):
        raise RangeError("source or destination outside [0, n)")
    valid = sok & dok
    if not ref:
        both = None if sv is None and dv is None else valid.astype(np.uint8)
        res = dict(driver_run(n, src_e, dst_e, ps, pd, both, lanes, 0))
        res.update(mode="default", lengths=(res["out"], res["valid"]), valid=valid.astype(np.uint8),
                   out=((res["valid"] != 0) & valid).astype(np.uint8))
        return res
    g = graph(n, src_e, dst_e)
    sdst = np.where(dok, pd, ps)
    out = np.zeros(p, np.uint8)
    one = np.uint64(1)
    chunks, b0 = [], 0
    while b0 < p:
        lane_of, end = {}, b0
        while end < p and len(lane_of) < L:
            if sok[end]:
                lane_of.setdefault(int(ps[end]), len(lane_of))
            end += 1
        rows = np.arange(b0, end)
        lane = np.array([lane_of[int(ps[r])] if sok[r] else -1 for r in rows], np.int64)
        lane_src = np.array(list(lane_of), np.int64)
        ch = dict(b0=b0, end=end, rows=rows, lane=lane, lane_src=lane_src,
                  cut="lane_512_opened" if len(lane_of) == L else "end_of_rows", searches=len(lane_src),
                  search_rows=int(np.count_nonzero(lane >= 0)), answered_at=np.full(len(rows), -1), levels=[],
                  stop=None)
        chunks.append(ch)
        b0 = end
        if not len(lane_src):
            continue
        k = len(lane_src)
        words = (k + 63) // 64
        lk = np.arange(k)
        visit = np.zeros((n, words), np.uint64)
        np.bitwise_or.at(visit, (lane_src, lk >> 6), np.left_shift(one, (lk & 63).astype(np.uint64)))
        seen = visit.copy()  # sources are seen from the start
        on = lane >= 0
        srows, sl, sd = rows[on], lane[on], sdst[rows[on]]

        def found():
            return ((seen[sd, sl >> 6] >> (sl & 63).astype(np.uint64)) & one) != 0

        at = np.where(found(), 0, -1)
        it = 1
        while True:
            fr = visit.any(axis=1)
            nxt = np.zeros((n, words), np.uint64)
            if len(g.heads):
                nxt[g.heads] = np.bitwise_or.reduceat(visit[g.pull_src], g.starts, axis=0)
            nxt &= ~seen
            seen |= nxt
            visit = nxt
            new = found() & (at < 0)
            at[new] = it
            ch["levels"].append(dict(level=it, fv=int(fr.sum()), fe=int(g.od[fr].sum()),
                                     items=int(np.maximum(1, -(-g.od[fr] // ITEM_EDGES)).sum()), answered=srows[new]))
            if not nxt.any():  # the only stop: a level that adds no bit
                ch["stop"] = "frontier_empty"
                break
            it += 1
        ch["answered_at"][on] = at
        out[srows] = (at >= 0) & valid[srows]
    return dict(mode="reference", sdst=sdst, chunks=chunks, out=out, valid=valid.astype(np.uint8),
                searches=sum(c["searches"] for c in chunks), pruned=0,
                search_rows=sum(c["search_rows"] for c in chunks), lanes=L if p else 0,
                batches=sum(1 for c in chunks if c["searches"]), levels=sum(len(c["levels"]) for c in chunks),
                edges=sum(x["fe"] for c in chunks for x in c["levels"]),
                fv=sum(x["fv"] for c in chunks for x in c["levels"]))


def chunk_trace(res):
    """Per chunk: its level lines (batch 1 of its own call) and its call line (lanes, searches, rows, pruned)."""
    return [([(1, x["level"], x["fv"], x["fe"]) for x in c["levels"]], (L, c["searches"], c["search_rows"], 0))
            for c in res["chunks"]]


# ---- shapes -------------------------------------------------------------------------------------------------------------
def reach_shape():
    """A body of 3000 vertices with 1 .. 4 out-edges (into the body and 100 sinks), 100 tops (out-edges, no in-edges:
    internal rows from n_ab on), 50 isolated vertices, cycles of 1 (a self-loop), 2 and 33 vertices each with a tail of
    five, and a chain of 50 vertices whose head has no in-edges."""
    rng = np.random.default_rng(500)
    body, sinks, tops, iso = 3000, 100, 100, 50
    od = rng.integers(1, 5, body)
    src = [np.repeat(np.arange(body), od)]
    dst = [rng.integers(0, body + sinks, len(src[0]))]
    t0 = body + sinks
    src.append(np.repeat(np.arange(t0, t0 + tops), 2))
    dst.append(rng.integers(0, body, 2 * tops))
    nxt = [t0 + tops + iso]
    mark = dict(body=np.arange(body), sinks=np.arange(body, t0), tops=np.arange(t0, t0 + tops),
                iso=np.arange(t0 + tops, nxt[0]))

    def new(k):
        a = np.arange(nxt[0], nxt[0] + k)
        nxt[0] += k
        return a

    for c in (1, 2, 33):
        cyc, tail = new(c), new(5)
        src += [cyc, np.concatenate([cyc[:1], tail[:-1]])]
        dst += [np.roll(cyc, -1), tail]
        mark[f"cyc_{c}"] = cyc
    ch = new(50)
    src.append(ch[:-1])
    dst.append(ch[1:])
    mark["chain"] = ch
    return Shape(nxt[0], np.concatenate(src), np.concatenate(dst)), mark


def wide_shape():
    """A root with an edge to each of 1500 vertices of layer 0, then 44 more layers of 1500, each vertex with three
    edges into the next layer: a frontier of 4500 out-edges for 44 levels."""
    w, layers = 1500, 45
    ids = 1 + np.arange(layers * w).reshape(layers, w)
    j = np.arange(w)
    src, dst = [np.zeros(w, np.int64)], [ids[0]]
    for i in range(layers - 1):
        for t in (j, (j + 1) % w, (j * 7 + 3) % w):
            src.append(ids[i])
            dst.append(ids[i + 1][t])
    return Shape(1 + layers * w, np.concatenate(src), np.concatenate(dst)), dict(root=0, layer0=ids[0])


_shapes = {}


def rshape(name):
    """-> (Shape, marks): "reach", "wide" or "lay:<name of the layout catalogue>"."""
    if name not in _shapes:
        if name.startswith("lay:"):
            _shapes[name] = (layout_shape(name[4:]), {})
        else:
            _shapes[name] = {"reach": reach_shape, "wide": wide_shape}[name]()
    return _shapes[name]


def rgraph(name):
    sh = rshape(name)[0]
    return graph(sh.n, sh.src, sh.dst)


# ---- the catalogue -----------------------------------------------------------------------------------------------------
@dataclass
class RCase:
    shape: str
    ps: np.ndarray
    pd: np.ndarray
    sv: object = None
    dv: object = None
    prev: str = None            # the case run just before on the same workspace (stale_trap_across_calls)
    want: set = field(default_factory=set)


def _arr(x):
    return np.asarray(x, dtype=np.int64)


def _dsts(g, rng, ps):
    """Random destinations with in-edges, none equal to its source."""
    pd = rng.choice(g.has_in, len(ps))
    clash = pd == ps
    pd[clash] = g.has_in[(np.searchsorted(g.has_in, pd[clash]) + 1) % len(g.has_in)]
    return pd


def _pool(g, mark, seed):
    """Body vertices with in-edges, shuffled."""
    b = mark["body"]
    return np.random.default_rng(seed).permutation(b[g.ind[b] > 0])


def build_case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("lay:"):
        return layout_case(name)
    shp = "wide" if name == "early_wide" else "reach"
    sh, mark = rshape(shp)
    g = rgraph(shp)
    n = sh.n
    if shp == "wide":
        r, l0 = mark["root"], mark["layer0"]
        return RCase("wide", _arr([r, r, r]), _arr([l0[0], l0[7], r]), want={"answered_early_wide"})
    pool = _pool(g, mark, 7)
    tops, ch = mark["tops"], mark["chain"]
    if name.startswith("distinct_"):
        k = int(name[9:])
        ps = pool[:k]
        want = {name} | ({"opener_last_row"} if k % L == 0 else set())
        return RCase("reach", ps, _dsts(g, rng, ps), want=want)
    if name == "opener_then_1":
        ps = np.concatenate([pool[:L], pool[3:4]])
        return RCase("reach", ps, _dsts(g, rng, ps), want={"opener_followed_by_1_repeat", "distinct_512"})
    if name == "opener_then_600":
        ps = np.concatenate([pool[:L], rng.permutation(pool[:L]), rng.choice(pool[:L], 88)])
        return RCase("reach", ps, _dsts(g, rng, ps), want={"opener_followed_by_600_repeats", "distinct_512"})
    if name == "nulls_at_opener":
        # [511 sources, NULL, opener] [NULL, 511 sources, NULL, opener] [NULL, NULL, NULL]
        parts = [pool[:511], [-7], pool[511:512], [n + 3], pool[512:1023], [1 << 40], pool[1023:1024], GARBAGE]
        ps = np.concatenate([_arr(x) for x in parts])
        sv = np.ones(len(ps), np.uint8)
        sv[[511, 513, 1025, 1027, 1028, 1029]] = 0
        pd = _dsts(g, rng, np.where(sv == 1, ps, 0))
        return RCase("reach", ps, pd, sv, want={"null_src_before_opener", "null_src_after_opener",
                                                "trailing_null_chunk", "distinct_1024"})
    if name == "null_dst_openers":
        # NULL destinations (ids that must not be read) on the rows that open lanes 0, 511 and 512; behind them rows
        # of the first chunk's sources and of lane 512's source
        ps = np.concatenate([pool[:L + 1], pool[[0, 0, 1]], pool[[L, L]], pool[L + 1:L + 40]])
        pd = _dsts(g, rng, ps)
        dv = np.ones(len(ps), np.uint8)
        for r, x in zip((0, L - 1, L), GARBAGE):
            dv[r], pd[r] = 0, x
        dv[L + 2] = 0
        return RCase("reach", ps, pd, None, dv, want={f"null_dst_opens_lane_{k}" for k in (0, 511, 512)})
    if name == "trivial":
        p0, p1, p2, p3, p4 = pool[:5]
        rows = [(p0, pool[10]), (p1, p1), (p1, p1), (p2, p2), (p3, pool[11]), (p2, pool[12]), (mark["sinks"][0],) * 2,
                (tops[0],) * 2, (mark["iso"][0],) * 2, (p4, p4), (p1, p1)]
        ps, pd = _arr(rows).T
        return RCase("reach", ps, pd, want={"trivial_only_lane", "trivial_first_row_of_source", "trivial_no_out",
                                            "trivial_no_in", "trivial_isolated"})
    if name == "trivial_chunk":
        ps = pool[:600]
        return RCase("reach", ps, ps.copy(), want={"trivial_only_chunk", "trivial_only_lane"})
    if name == "cycles":
        ps = _arr([mark[f"cyc_{c}"][0] for c in (1, 2, 33)])
        return RCase("reach", ps, tops[:3].copy(), want={f"source_on_cycle_{c}" for c in (1, 2, 33)})
    if name == "source_reaches_source":
        return RCase("reach", _arr([ch[0], ch[10], ch[10]]), _arr([tops[3], tops[4], ch[20]]),
                     want={"source_reaches_source"})
    if name == "early_chain":
        return RCase("reach", _arr([ch[0], ch[0], ch[0]]), _arr([ch[1], ch[0], ch[1]]),
                     want={"answered_early_tail_chain"})
    if name == "layout_rows":
        lay = g.lay
        inv, nab = lay["inv"], lay["n_ab"]
        x1, x2, x3 = (int(inv[i]) for i in (nab - 1, nab, n - 1))
        rows = [(x1, pool[0]), (x2, pool[1]), (x3, x3), (x2, x2), (pool[2], x1), (pool[3], x2)]
        ps, pd = _arr(rows).T
        return RCase("reach", ps, pd, want={"source_at_n_ab_minus_1", "source_at_n_ab", "source_at_n_minus_1"})
    if name == "stale_chunks":
        # chunk 1: tops on lanes 0, 300 and 511; chunk 2: rows (Y, top) on the same lanes
        a = pool[:L].copy()
        a[[0, 300, 511]] = tops[10:13]
        b = pool[600:600 + L].copy()
        ps = np.concatenate([a, b])
        pd = _dsts(g, rng, ps)
        pd[[L, L + 300, L + 511]] = tops[10:13]
        return RCase("reach", ps, pd, want={"stale_trap_across_chunks", "opener_last_row"})
    if name == "stale_call_a":
        ps = np.concatenate([tops[20:24], pool[:16]])
        return RCase("reach", ps, _dsts(g, rng, ps))
    if name == "stale_call_b":
        ps = pool[100:120].copy()
        pd = _dsts(g, rng, ps)
        pd[:4] = tops[20:24]
        return RCase("reach", ps, pd, prev="stale_call_a", want={"stale_trap_across_calls"})
    raise KeyError(name)


def layout_case(name):
    """A shape of the layout catalogue: its focus vertices and the vertices at internal rows 0, n_ab - 1, n_ab and
    n - 1 as sources, each towards the next one and towards itself, plus a NULL-source and a NULL-destination row."""
    sh = rshape(name)[0]
    lay = layout(sh.n, sh.src, sh.dst)
    n, inv, nab = sh.n, lay["inv"], lay["n_ab"]
    picks = [int(x) for x in sh.focus[:8]] + [int(inv[i]) for i in (0, nab - 1, nab, n - 1) if 0 <= i < n]
    ps, pd = [], []
    for i, s in enumerate(picks):
        ps += [s, s]
        pd += [picks[(i + 1) % len(picks)], s]
    ps, pd = _arr(ps + [GARBAGE[0], picks[0]]), _arr(pd + [picks[-1], GARBAGE[1]])
    sv, dv = np.ones(len(ps), np.uint8), np.ones(len(ps), np.uint8)
    sv[-2], dv[-1] = 0, 0
    want = {f"layout_{name[4:]}"} | ({"n_equals_n_ab"} if name == "lay:selfloops" else set())
    return RCase(name, ps, pd, sv, dv, want=want)


CUT = [f"distinct_{k}" for k in (511, 512, 513, 1024, 1025)] + ["opener_then_1", "opener_then_600",
                                                                 "nulls_at_opener", "null_dst_openers"]
CASES = (CUT + ["trivial", "trivial_chunk", "cycles", "source_reaches_source", "early_chain", "early_wide",
                "layout_rows", "stale_chunks", "stale_call_a", "stale_call_b"] + [f"lay:{s}" for s in CATALOGUE])
_cases = {}


def case(name):
    if name not in _cases:
        _cases[name] = build_case(name)
    return _cases[name]


def restated(c, ref=True):
    sh = rshape(c.shape)[0]
    return _oracle("reach_run", lambda: reach_run(sh.n, sh.src, sh.dst, c.ps, c.pd, c.sv, c.dv, ref),
                   sh.n, sh.src, sh.dst, c.ps, c.pd, c.sv, c.dv, ref)


def _on_cycle(g, s):
    """Length of the shortest cycle through s (0 = none)."""
    back = g.ins(s)
    d = g.dist(s)[back] if len(back) else np.zeros(0)
    return int(d[d >= 0].min()) + 1 if np.any(d >= 0) else 0


def _traps(g, prev_chunk, c, chunk):
    """Is a source without in-edges on lane k of prev_chunk the destination of a row on lane k of chunk?"""
    dok = np.ones(len(c.ps), bool) if c.dv is None else c.dv != 0
    rows = chunk["rows"]
    for k, x in enumerate(prev_chunk["lane_src"]):
        if g.ind[x] == 0:
            hit = (chunk["lane"] == k) & dok[rows] & (c.pd[rows] == x) & (c.ps[rows] != x)
            if hit.any():
                return True
    return False


def case_hits(name, c):
    """Every boundary of reachability's reference batches that case c hits, by name."""
    sh = rshape(c.shape)[0]
    g = rgraph(c.shape)
    n, p = sh.n, len(c.ps)
    res = restated(c)
    chunks = res["chunks"]
    sok = np.ones(p, bool) if c.sv is None else c.sv != 0
    dok = np.ones(p, bool) if c.dv is None else c.dv != 0
    out = set()
    k = len(np.unique(c.ps[sok]))
    if k in (511, 512, 513, 1024, 1025):
        out.add(f"distinct_{k}")
    first = set(chunks[0]["lane_src"].tolist()) if chunks else set()
    triv = sok & dok & (c.ps == c.pd)
    for ci, ch in enumerate(chunks):
        rows, lane = ch["rows"], ch["lane"]
        if ch["cut"] == "lane_512_opened":
            op, end = ch["end"] - 1, ch["end"]
            after = np.arange(end, p)

            def repeats(rr):
                return len(rr) > 0 and all(sok[r] and int(c.ps[r]) in first for r in rr)

            if op == p - 1:
                out.add("opener_last_row")
            if len(after) == 1 and repeats(after):
                out.add("opener_followed_by_1_repeat")
            if len(after) >= 600 and repeats(after[:600]):
                out.add("opener_followed_by_600_repeats")
            if op > ch["b0"] and not sok[op - 1]:
                out.add("null_src_before_opener")
            if end < p and not sok[end]:
                out.add("null_src_after_opener")
        if ch["searches"] == 0:
            if ci == len(chunks) - 1 and ci > 0:
                out.add("trailing_null_chunk")
            continue
        _, first_at = np.unique(lane, return_index=True)
        leaders = rows[first_at[lane[first_at] >= 0]]
        for r in leaders:
            ordinal = L * ci + lane[r - ch["b0"]]
            if not dok[r] and ordinal in (0, 511, 512):
                out.add(f"null_dst_opens_lane_{ordinal}")
        for l in range(ch["searches"]):
            mine = rows[lane == l]
            if triv[mine].all():
                out.add("trivial_only_lane")
            elif triv[mine[0]]:
                out.add("trivial_first_row_of_source")
        if triv[rows[lane >= 0]].all():
            out.add("trivial_only_chunk")
        at = ch["answered_at"][lane >= 0]
        lv = ch["levels"]
        if at.min() >= 0 and at.max() == 1 and len(lv) - 1 >= 40:
            if all(x["fe"] <= TAIL_EDGES and x["items"] <= TAIL_ITEMS for x in lv):
                out.add("answered_early_tail_chain")
            if sum(x["fe"] > TAIL_EDGES for x in lv[1:]) >= 40:
                out.add("answered_early_wide")
        if ch["searches"] <= 64:
            srcs = ch["lane_src"]
            for s in srcs:
                if np.any((g.dist(int(s))[srcs] > 0)):
                    out.add("source_reaches_source")
            for r in rows[(lane >= 0) & dok[rows] & ~triv[rows]]:
                s, d = int(c.ps[r]), int(c.pd[r])
                cyc = _on_cycle(g, s)
                if cyc in (1, 2, 33) and g.dist(s)[d] < 0:
                    # iterativelength expands a source again when a cycle brings it back; reachability does not
                    il = driver_run(n, sh.src, sh.dst, [s], [d], None, L, NO_PRUNE)
                    rr = reach_run(n, sh.src, sh.dst, [s], [d])
                    if il["edges"] - rr["edges"] == g.od[s] > 0:
                        out.add(f"source_on_cycle_{cyc}")
        if ci + 1 < len(chunks) and _traps(g, ch, c, chunks[ci + 1]):
            out.add("stale_trap_across_chunks")
    for r in np.flatnonzero(triv):
        s = c.ps[r]
        if g.od[s] == 0 and g.ind[s] > 0:
            out.add("trivial_no_out")
        if g.od[s] > 0 and g.ind[s] == 0:
            out.add("trivial_no_in")
        if g.od[s] == 0 and g.ind[s] == 0:
            out.add("trivial_isolated")
    if c.prev:
        pc = case(c.prev)
        assert pc.shape == c.shape
        if chunks and _traps(g, restated(pc)["chunks"][-1], c, chunks[0]):
            out.add("stale_trap_across_calls")
    srcs = np.concatenate([ch["lane_src"] for ch in chunks]) if chunks else np.zeros(0, np.int64)
    internal = g.perm[srcs]
    nab = g.lay["n_ab"]
    for nm, row in (("source_at_n_ab_minus_1", nab - 1), ("source_at_n_ab", nab), ("source_at_n_minus_1", n - 1)):
        if np.any(internal == row):
            out.add(nm)
    if nab == n and len(srcs):
        out.add("n_equals_n_ab")
    if c.shape.startswith("lay:") and len(srcs):
        out.add(f"layout_{c.shape[4:]}")
    return out


REQUIRED = (
    {f"distinct_{k}" for k in (511, 512, 513, 1024, 1025)}
    | {"opener_last_row", "opener_followed_by_1_repeat", "opener_followed_by_600_repeats", "null_src_before_opener",
       "null_src_after_opener", "trailing_null_chunk", "null_src_valid_dst_out_of_range"}
    | {f"null_dst_opens_lane_{k}" for k in (0, 511, 512)}
    | {"trivial_only_lane", "trivial_first_row_of_source", "trivial_no_out", "trivial_no_in", "trivial_isolated",
       "trivial_only_chunk"}
    | {f"source_on_cycle_{c}" for c in (1, 2, 33)} | {"source_reaches_source"}
    | {"answered_early_tail_chain", "answered_early_wide"}
    | {"source_at_n_ab_minus_1", "source_at_n_ab", "source_at_n_minus_1", "n_equals_n_ab"}
    | {f"layout_{s}" for s in CATALOGUE}
    | {"stale_trap_across_chunks", "stale_trap_across_calls"}
)


# ---- CPU: the restatement equals the oracle; the catalogue hits what it names ---------------------------------------------
def _scipy_reach(g, ps, pd):
    """src == dst or a path from src to dst, by scipy."""
    out = np.zeros(len(ps), bool)
    if len(ps):
        srcs = np.unique(ps)
        d = sp_shortest_path(g.mat, method="D", unweighted=True, indices=srcs)
        out = np.isfinite(d[np.searchsorted(srcs, ps), pd])
    return out


@pytest.mark.parametrize("name", CASES)
def test_restatement_equals_the_oracle(name):
    """Answers, written rows, batches, levels and edges of oracle/pgq_oracle_reach.c with the defined batch start;
    answers of scipy; every chunk stops on an empty level; and the default mode answers the same."""
    c = case(name)
    sh = rshape(c.shape)[0]
    g = rgraph(c.shape)
    res = restated(c)
    eo, ew, ost = orr.reachability(sh.n, g.v, g.e, c.ps, c.pd, c.sv, c.dv, restart=False)
    assert np.array_equal(res["valid"], ew) and np.array_equal(res["out"], eo)
    assert (res["batches"], res["levels"], res["edges"]) == (ost.batches, ost.levels, ost.edges_traversed)
    ok = res["valid"] != 0
    assert np.array_equal(res["out"][ok] != 0, _scipy_reach(g, c.ps[ok], c.pd[ok]))
    assert all(ch["stop"] == "frontier_empty" for ch in res["chunks"] if ch["searches"])
    assert res["searches"] == sum(len(set(c.ps[ch["rows"][ch["lane"] >= 0]].tolist())) for ch in res["chunks"])
    d = restated(c, False)
    assert np.array_equal(d["out"], res["out"]) and np.array_equal(d["valid"], res["valid"])


@pytest.mark.parametrize("name", CASES)
def test_reach_catalogue_hits_its_boundaries(name):
    c = case(name)
    got = case_hits(name, c)
    print(f"{name}: p={len(c.ps)} chunks={len(restated(c)['chunks'])} hits {sorted(got)}")
    assert c.want <= got, sorted(c.want - got)


def null_source_range_call():
    """A NULL source next to a valid destination outside [0, n): the device refuses it (every valid id is checked),
    while the oracle, like the reference, never reads a destination behind a NULL source."""
    c = case("trivial")
    n = rshape(c.shape)[0].n
    ps, pd = c.ps.copy(), c.pd.copy()
    sv = np.ones(len(ps), np.uint8)
    sv[4], ps[4], pd[4] = 0, GARBAGE[1], n
    return c, ps, pd, sv


def test_null_source_with_a_destination_out_of_range():
    c, ps, pd, sv = null_source_range_call()
    sh = rshape(c.shape)[0]
    g = rgraph(c.shape)
    for ref in (True, False):
        with pytest.raises(RangeError):
            reach_run(sh.n, sh.src, sh.dst, ps, pd, sv, None, ref)
    eo, ew, _ = orr.reachability(sh.n, g.v, g.e, ps, pd, sv, None, restart=False)
    assert ew[4] == 0 and ew.sum() == len(ps) - 1


def test_reach_catalogue_covers_every_boundary():
    named = set().union(*(case(n).want for n in CASES)) | {"null_src_valid_dst_out_of_range"}
    assert REQUIRED <= named, sorted(REQUIRED - named)


def test_seen_sources_change_the_work_not_the_answer():
    """On the cycles the iterativelength driver (sources not seen) expands every source once more than reach mode:
    edges differ by the sources' out-degrees, answers do not."""
    c = case("cycles")
    sh = rshape(c.shape)[0]
    g = rgraph(c.shape)
    rr = restated(c)
    il = driver_run(sh.n, sh.src, sh.dst, c.ps, c.pd, None, L, NO_PRUNE)
    assert il["edges"] - rr["edges"] == int(g.od[c.ps].sum()) > 0
    assert not rr["out"].any() and not il["valid"].any()


# ---- GPU -----------------------------------------------------------------------------------------------------------------
TAIL_LINE = re.compile(r"\[pgq\] batch \d+ level (\d+) (push|pull|tail) frontier_v=\d+ frontier_e=\d+ items=(-?\d+) ")


def build_csr(ctx, shape_name):
    sh = rshape(shape_name)[0]
    return pgq.DeviceCSR.build(ctx, sh.n, sh.src, sh.dst)


def trace_segments(err):
    """The stderr of one call split at its call lines: [(level lines (batch, level, fv, fe), call line)]."""
    segs, cur = [], []
    for line in err.splitlines():
        m = LEVEL.search(line)
        if m:
            cur.append(tuple(int(x) for x in m.groups()))
            continue
        m = CALL.search(line)
        if m:
            segs.append((cur, tuple(int(x) for x in m.groups())))
            cur = []
    return segs


def check_reference(csr, c, capfd=None):
    res = restated(c)
    if capfd:
        capfd.readouterr()
    out, valid, st = csr.reachability(c.ps, c.pd, c.sv, c.dv, options(0, REF))
    assert np.array_equal(valid, res["valid"]), np.flatnonzero(valid != res["valid"])[:10]
    assert np.array_equal(out, res["out"]), np.flatnonzero(out != res["out"])[:10]
    assert tuple(st[k] for k in COUNTERS) == counters(res)
    if capfd:
        got, want = trace_segments(capfd.readouterr().err), chunk_trace(res)
        assert got == want, next((i, a, b) for i, (a, b) in enumerate(zip(got + [None], want + [None])) if a != b)
    return out


def check_default(csr, c, capfd=None):
    res = restated(c, False)
    if capfd:
        capfd.readouterr()
    out, valid, st = csr.reachability(c.ps, c.pd, c.sv, c.dv)
    assert np.array_equal(valid, res["valid"]) and np.array_equal(out, res["out"])
    assert tuple(st[k] for k in COUNTERS) == counters(res)
    if capfd:
        check_trace(capfd.readouterr().err, res)
    ok = res["valid"]
    lo, lv, lst = csr.iterativelength(c.ps, c.pd, None if c.sv is None and c.dv is None else ok)
    assert np.array_equal(out, lv & ok) and tuple(lst[k] for k in COUNTERS) == tuple(st[k] for k in COUNTERS)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_case_on_the_device(gpu_ctx, monkeypatch, capfd, name):
    """Every case with the reference's batches (answers, valid, the eight counters, each chunk's level lines and call
    line) and in the default mode (driver_run's counters and trace, csr.iterativelength's answers)."""
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", "1")
    c = case(name)
    csr = build_csr(gpu_ctx, c.shape)
    try:
        check_reference(csr, c, capfd)
        check_default(csr, c, capfd)
    finally:
        csr.free()


@pytest.mark.gpu
def test_tail_runs_on_after_every_row_is_answered(gpu_ctx, monkeypatch, capfd):
    """early_chain: every row is answered at level 1, and the chain goes on for 49 levels.  k_tail must not stop at
    the answered level: one launch runs levels 1 .. 32 and the next one the rest, so only levels 1 and 33 open a
    launch (the trace shows the work items on those lines, -1 on the levels a launch ran after its first)."""
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    c = case("early_chain")
    csr = build_csr(gpu_ctx, c.shape)
    try:
        capfd.readouterr()
        check_reference(csr, c)
        lines = [(int(a), k, int(i)) for a, k, i in TAIL_LINE.findall(capfd.readouterr().err)]
        assert len(lines) == restated(c)["levels"] >= TAIL_MAX + 2
        assert all(k == "tail" for _, k, _ in lines)
        assert [lv for lv, _, i in lines if i >= 0] == list(range(1, len(lines) + 1, TAIL_MAX))
    finally:
        csr.free()


@pytest.mark.gpu
def test_null_source_with_a_destination_out_of_range_is_refused(gpu_ctx):
    c, ps, pd, sv = null_source_range_call()
    csr = build_csr(gpu_ctx, c.shape)
    try:
        for opts in (options(0, REF), None):
            with pytest.raises(pgq.InvalidInputException) as ei:
                csr.reachability(ps, pd, sv, None, opts)
            assert ei.value.status == pgq.PGQ_ERR_RANGE
            check_reference(csr, c)
    finally:
        csr.free()


SETTINGS = [f"schedule_{s}" for s in SCHEDULES] + ["no_tail", "pull_skip_0"]
SETTING_CASES = ["nulls_at_opener", "null_dst_openers", "trivial", "cycles", "source_reaches_source", "early_chain",
                 "early_wide", "layout_rows", "stale_chunks", "lay:outdeg_tail", "lay:split_m0"]


@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS)
def test_settings(gpu_ctx, monkeypatch, capfd, setting):
    """Forced direction schedules, no k_tail, and bottom-up levels that do not skip finished rows: the same answers,
    counters and frontiers level by level."""
    if setting.startswith("schedule_"):
        monkeypatch.setenv("PGQ_B200_SCHEDULE", setting[9:])
    elif setting == "no_tail":
        monkeypatch.setenv("PGQ_B200_NO_TAIL", "1")
    else:
        monkeypatch.setenv("PGQ_B200_PULL_SKIP", "0")
    monkeypatch.setenv("PGQ_B200_TRACE", "1")
    monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", "1")
    csrs = {}
    try:
        for name in SETTING_CASES:
            c = case(name)
            if c.shape not in csrs:
                csrs[c.shape] = build_csr(gpu_ctx, c.shape)
            check_reference(csrs[c.shape], c, capfd)
            check_default(csrs[c.shape], c, capfd)
    finally:
        for x in csrs.values():
            x.free()


ROUTE_CASES = ["nulls_at_opener", "null_dst_openers", "trivial", "cycles", "early_chain", "layout_rows",
               "stale_chunks"]


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(ROUTES))
def test_routes(gpu_ctx, route):
    """The reach shape built through every construction route: the same answers and counters in both modes."""
    csr, _, _ = make(gpu_ctx, rshape("reach")[0], route)
    try:
        for name in ROUTE_CASES:
            check_reference(csr, case(name))
            check_default(csr, case(name))
    finally:
        csr.free()


@pytest.mark.gpu
def test_one_workspace_in_turn(monkeypatch):
    """One context with one workspace.  Each BFS consumer runs with tops (sources without in-edges, internal rows from
    n_ab on) on lanes 0 .. 3, then a reachability call with the reference's batches asks, on lanes 0 .. 3, for those
    tops from vertices that cannot reach them: a seen bit any consumer left beyond n_ab answers true."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    sh, mark = rshape("reach")
    g = rgraph("reach")
    pool = _pool(g, mark, 11)
    try:
        csr = build_csr(ctx, "reach")
        v, e, _ = csr.download()
        for t, kind in enumerate(["reach_ref", "reach_default", "iterativelength", "shortestpath", "bidirectional",
                                  "reach_ref"]):
            xs = mark["tops"][40 + 4 * t:44 + 4 * t]
            ps = np.concatenate([xs, pool[:30]])
            a = RCase("reach", ps, _dsts(g, np.random.default_rng(t), ps))
            if kind == "reach_ref":
                check_reference(csr, a)
            elif kind == "reach_default":
                check_default(csr, a)
            elif kind == "iterativelength":
                res = driver_run(sh.n, sh.src, sh.dst, a.ps, a.pd)
                out, valid, st = csr.iterativelength(a.ps, a.pd)
                assert np.array_equal(out, res["out"]) and np.array_equal(valid, res["valid"])
                assert tuple(st[k] for k in COUNTERS) == counters(res)
            elif kind == "shortestpath":
                res = driver_run(sh.n, sh.src, sh.dst, a.ps, a.pd, path=True, edge_id=np.arange(len(sh.src)))
                paths, st = csr.shortestpath(a.ps, a.pd)
                assert paths == res["paths"]
            else:
                bo, bv, _ = csr.iterativelengthbidirectional(a.ps, a.pd)
                eo, ev, _ = orb.iterativelengthbidirectional(sh.n, v, e, a.ps, a.pd, None, None, 512)
                assert np.array_equal(bv, ev) and np.array_equal(bo, eo)
            ps = pool[200 + 8 * t:230 + 8 * t].copy()
            pd = _dsts(g, np.random.default_rng(100 + t), ps)
            pd[:4] = xs
            b = RCase("reach", ps, pd)
            assert not restated(b)["out"][:4].any()
            check_reference(csr, b)
        csr.free()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_eight_threads_one_csr(gpu_ctx):
    """Eight threads with different cases on one CSR, with the reference's batches, twice each."""
    names = ["nulls_at_opener", "null_dst_openers", "trivial", "trivial_chunk", "cycles", "stale_chunks",
             "opener_then_600", "layout_rows"]
    for nm in names:  # (the restatements, computed before the threads start)
        restated(case(nm))
    csr = build_csr(gpu_ctx, "reach")
    try:
        def body(nm):
            for _ in range(2):
                check_reference(csr, case(nm))
            return nm

        with ThreadPoolExecutor(max_workers=8) as pool:
            assert sorted(pool.map(body, names)) == sorted(names)
    finally:
        csr.free()
