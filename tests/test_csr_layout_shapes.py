"""The device CSR at the boundaries of its layout, through every construction route and every consumer.

finalize_from_rows / finish_csr (csrc/pgq_csr.cu) build more than the reference's v / e: a renumbering into four
vertex classes ordered by descending clamped degree, the out-CSR and in-CSC with their head bitmaps and chunk ranks,
and the bottom-up layout (long rows of in-degree >= 32 back to back in 1024-position ranges, short rows of in-degree
1 .. 31 in degree-sorted 32-row slices padded with -1).  Only v / e / edge ids / weights can be downloaded; the rest
shows only in what the consumers answer.  So:

- a catalogue of deterministic shapes, each naming the layout boundaries it hits.  A CPU-only test recomputes the
  device layout in numpy from the edge rows and asserts that every named boundary really is hit;
- every shape built through every route (build, build_device, upload, the chunked create / add_vertex_counts /
  add_edges / finalize from one thread and from eight, weighted BIGINT / DOUBLE) and cloned into a second context;
- the downloaded CSR checked against the CPU restatement of the reference (oracle/pgq_oracle.c), and every consumer
  (iterativelength under forced direction schedules, shortestpath, cheapest_path_length, local_clustering_coefficient,
  pagerank, weakly_connected_component) compared with the restatement run on the downloaded CSR, bit for bit;
- a context with one workspace that builds, checks and frees graphs of equal buffer sizes but different content, so
  every array is recycled dirty; and replicas that outlive their primary."""
import hashlib
import re
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc

SHORT_DEG = 32           # PGQ_SHORT_DEG: in-degree from which a row is stored in the long part
DEG_CLAMP = 0x3FFFFF     # PGQ_DEG_CLAMP: degrees are clamped to this in the vertex sort key
ITEM_EDGES = 256         # PGQ_ITEM_EDGES
TAIL_ITEMS, TAIL_EDGES = 256, 1024  # PGQ_TAIL_ITEMS / PGQ_TAIL_EDGES
LCC_SMEM = 4096          # out-lists up to this length are sorted in shared memory by LCC
SCAN_TILE = 2048         # items per block of the exclusive scan
RS_BITS = 5              # bits per radix-sort pass
STAGE_ROWS = 4096        # rows per staging slot of the chunked build


# ---- the device layout, in numpy --------------------------------------------------------------------------------------
def layout(n, src, dst):
    """What finalize_from_rows / build_pull_graph make of the edge rows (original ids), as far as sizes and
    positions go: classes, the internal order, the long / short split, long-part positions, slices."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    od = np.bincount(src, minlength=n)[:n]
    ind = np.bincount(dst, minlength=n)[:n]
    cls = np.where(od > 0, np.where(ind > 0, 0, 2), np.where(ind > 0, 1, 3))
    deg = np.minimum(np.where(od > 0, od, ind), DEG_CLAMP)
    key = (cls << 22) | (DEG_CLAMP - deg)
    inv = np.argsort(key, kind="stable")          # internal id -> original id
    n_ab = int(np.count_nonzero(cls <= 1))
    row_deg = ind[inv[:n_ab]]                      # in-degree of every in-CSC row with in-edges
    is_long = row_deg >= SHORT_DEG
    long_rows = np.flatnonzero(is_long)
    long_deg = row_deg[long_rows]
    starts = np.concatenate([[0], np.cumsum(long_deg)[:-1]]).astype(np.int64) if len(long_deg) else np.zeros(0, np.int64)
    ends = starts + long_deg
    short_rows = np.flatnonzero(~is_long)
    short_sorted = short_rows[np.argsort(SHORT_DEG - 1 - row_deg[short_rows], kind="stable")]
    sdeg = row_deg[short_sorted]
    n_short = len(short_sorted)
    n_slices = (n_short + 31) // 32
    widths = sdeg[::32] if n_short else np.zeros(0, np.int64)
    padding = int(np.sum(np.repeat(widths, 32)[:n_short] - sdeg)) if n_short else 0
    end_bit = 1
    while end_bit < 31 and (1 << end_bit) < n:
        end_bit += 1
    return dict(n=n, m=len(src), od=od, ind=ind, cls=cls, inv=inv, n_ab=n_ab,
                long_orig=inv[long_rows], long_deg=long_deg, starts=starts, ends=ends, long_total=int(long_deg.sum()),
                short_orig=inv[short_sorted], n_short=n_short, n_slices=n_slices, widths=widths, padding=padding,
                passes=-(-end_bit // RS_BITS), src=src, dst=dst)


def frontier_of(lay, sources):
    """Level-1 frontier of one batch whose lanes start at `sources`: their distinct out-neighbours but the sources
    -> (vertices, work items, out-edges)."""
    s = np.unique(np.asarray(sources, dtype=np.int64))
    nb = np.unique(lay["dst"][np.isin(lay["src"], s)])
    nb = nb[~np.isin(nb, s)]
    d = lay["od"][nb]
    return len(nb), int(np.sum(-(-d // ITEM_EDGES))), int(d.sum())


def hits(lay, batches=()):
    """Every boundary of the layout this graph hits, by name.  batches: the sources of each one-batch call that the
    GPU tests send (their level-1 frontiers are what k_tail is judged on)."""
    out = set()
    n, m, ind, od, cls = lay["n"], lay["m"], lay["ind"], lay["od"], lay["cls"]
    present = set(np.unique(ind).tolist())
    if set(range(1, 41)) <= present:
        out.add("indeg_1_to_40")
    if {31, 32, 33} <= present:
        out.add("split_31_32_33")
    if lay["n_short"]:
        out.add(f"n_short_mod32_{lay['n_short'] % 32}")
        w = lay["widths"]
        if len(w) > 2 and np.count_nonzero(w[1:] != w[:-1]) >= 2:
            out.add("slice_width_changes")
        if lay["padding"]:
            out.add("short_padding")
    for p in (255, 256, 257, 1023, 1024, 1025):
        if p in set(lay["starts"].tolist()):
            out.add(f"long_start_{p}")
        if p in set(lay["ends"].tolist()):
            out.add(f"long_end_{p}")
    if np.any(((lay["ends"] - 1) >> 10) - (lay["starts"] >> 10) >= 2):
        out.add("long_spans_3_ranges")
    if lay["long_total"] and lay["long_total"] % 1024 in (0, 1):
        out.add(f"long_total_mod1024_{lay['long_total'] % 1024}")
    for d in (255, 256, 257, 512, 513):
        if np.any(od == d):
            out.add(f"outdeg_{d}")
    for sources in batches:
        _, items, edges = frontier_of(lay, sources)
        if items in (TAIL_ITEMS, TAIL_ITEMS + 1):
            out.add(f"frontier_items_{items}")
        if edges in (TAIL_EDGES, TAIL_EDGES + 1):
            out.add(f"frontier_edges_{edges}")
    if m and not np.any(cls == 0):
        out.add("class0_empty")
    if n and np.all(cls == 0):
        out.add("only_class0")
    if np.any((cls == 1) & (ind >= 1024)):
        out.add("in_only_hub")
    iso = np.flatnonzero(cls == 3)
    if np.any((iso > 0) & (iso < n - 1)) and len(iso) < n:
        out.add("isolated_interleaved")
    if n and cls[n - 1] == 3:
        out.add("isolated_last")
    out.add(f"n_{n}")
    out.add(f"radix_passes_{lay['passes']}")
    if n + 1 in (SCAN_TILE, SCAN_TILE + 1):
        out.add(f"scan_n_plus_1_{n + 1}")
    if n >= 32:
        _, counts = np.unique(np.stack([cls, np.where(od > 0, od, ind)]), axis=1, return_counts=True)
        if counts.max() * 4 >= n:
            out.add("tied_degrees")
    if m:
        pair = lay["src"] * max(n, 1) + lay["dst"]
        if len(np.unique(pair)) < m:
            out.add("parallel_edges")
    for d in (LCC_SMEM - 1, LCC_SMEM, LCC_SMEM + 1):
        if np.any(od == d):
            out.add(f"lcc_outdeg_{d}")
    if m == 0:
        out.add("m0")
    if n == 1 and m and np.all(lay["src"] == lay["dst"]):
        out.add("n1_self_loop")
    if np.count_nonzero(np.maximum(od, ind) > DEG_CLAMP) >= 2:
        out.add("two_above_deg_clamp")
    return out


# ---- the catalogue -----------------------------------------------------------------------------------------------------
@dataclass
class Shape:
    n: int
    src: np.ndarray
    dst: np.ndarray
    focus: list = field(default_factory=list)  # vertices (original ids) the pairs start and end at
    neg: bool = False                          # weights below zero (no negative cycle: reduced costs)
    nan: bool = False                          # one DOUBLE weight is NaN
    tail: list = field(default_factory=list)   # hubs searched alone: level-1 frontiers at k_tail's limits


def _relabel(rng, n, src, dst, focus):
    p = rng.permutation(n)
    return p[src], p[dst], [int(p[f]) for f in focus]


def _body(rng, nb, mb):
    """A sparse random graph on [0, nb): in-degrees stay far below 32."""
    return rng.integers(0, nb, mb), rng.integers(0, nb, mb)


def split_shape(mod):
    """In-degrees 1 .. 40 (three rows each, half of the heads with an out-edge), topped up with in-only rows of
    in-degree 1 .. 31 until n_short % 32 == mod.  Ids shuffled."""
    rng = np.random.default_rng(10 + mod)
    nb = 600
    s, d = _body(rng, nb, 1500)
    src, dst, nxt = [s], [d], nb
    for i, k in enumerate(list(range(1, 41)) * 3):
        src.append(rng.choice(nb, k))
        dst.append(np.full(k, nxt))
        if i % 2:
            src.append([nxt])
            dst.append([rng.integers(0, nb)])
        nxt += 1
    ind = np.bincount(np.concatenate(dst), minlength=nxt)
    n_short = int(np.count_nonzero((ind > 0) & (ind < SHORT_DEG)))
    for j in range((mod - n_short) % 32):
        k = 1 + (j * 7) % 31
        src.append(rng.choice(nb, k))
        dst.append(np.full(k, nxt))
        nxt += 1
    src, dst = np.concatenate(src), np.concatenate(dst)
    heads = list(range(nb, nxt, 5))
    src, dst, focus = _relabel(rng, nxt, src, dst, heads)
    return Shape(nxt, src, dst, focus, neg=mod == 0)


def long_shape(off, total_mod):
    """Long rows in a chosen order: class-0 rows are ordered by descending out-degree, so head i gets out-degree
    60 - i.  The first row ends at 256 + off, the second at 1024 + off, the third (2100) spans three 1024-position
    ranges; a filler row makes the long total == total_mod (mod 1024).  The body's in-degrees stay short."""
    rng = np.random.default_rng(20 + off)
    nb = 3000
    s, d = _body(rng, nb, 6000)
    src, dst = [s], [d]
    degs = [256 + off, 768, 2100, 32, 33, 40, 63, 64, 65, 100, 255, 300]
    f = (total_mod - sum(degs)) % 1024
    degs.append(f if f >= SHORT_DEG else f + 1024)
    heads = list(range(nb, nb + len(degs)))
    for i, (h, k) in enumerate(zip(heads, degs)):
        src.append(rng.choice(nb, k))
        dst.append(np.full(k, h))
        src.append(np.full(60 - i, h))
        dst.append(rng.choice(nb, 60 - i, replace=False))
    n = nb + len(degs)
    return Shape(n, np.concatenate(src), np.concatenate(dst), heads + [0, 1, nb - 1], neg=off == 0)


def outdeg_tail_shape():
    """Out-degrees 255 / 256 / 257 / 512 / 513 around PGQ_ITEM_EDGES, and hubs whose level-1 frontier has exactly
    256 / 257 work items or 1024 / 1025 out-edges (k_tail's limits) when searched alone (tail_calls)."""
    rng = np.random.default_rng(30)
    nb = 2000
    s, d = _body(rng, nb, 5000)
    src, dst, focus, tail = [s], [d], [], []
    nxt = nb
    for k in (255, 256, 257, 512, 513):
        src.append(np.full(k, nxt))
        dst.append(rng.choice(nb, k, replace=False))
        focus.append(nxt)
        nxt += 1
    for leaves, per in ((256, 1), (257, 1), (128, 8), (128, 8)):
        h = nxt
        lv = np.arange(h + 1, h + 1 + leaves)
        nxt += 1 + leaves
        src.append(np.full(leaves, h))
        dst.append(lv)
        for j, leaf in enumerate(lv):
            k = per + (1 if per == 8 and j == 0 and len(tail) == 3 else 0)
            src.append(np.full(k, leaf))
            dst.append(rng.choice(nb, k, replace=False))
        tail.append(h)
    return Shape(nxt, np.concatenate(src), np.concatenate(dst), focus + tail, tail=tail)


def tail_calls(sh):
    """One call per tail hub whose rows all start at the hub (NULL-free), so that every batch's level-1 frontier is
    exactly the hub's -> [(hub, src, dst)]."""
    out = []
    for h in sh.tail:
        pd = np.concatenate([np.random.default_rng(h).integers(0, sh.n, 6), [h + 1, h + 2, h, 0]])
        out.append((h, np.full(len(pd), h, dtype=np.int64), pd.astype(np.int64)))
    return out


def bipartite_shape():
    """Sources -> sinks only: no vertex has both in- and out-edges (class 0 is empty).  Skewed sink popularity gives
    long and short rows.  Ids shuffled."""
    rng = np.random.default_rng(40)
    ns, nt = 400, 1000
    od = rng.integers(1, 60, ns)
    src = np.repeat(np.arange(ns), od)
    dst = ns + (rng.random(len(src)) ** 3 * nt).astype(np.int64)
    src, dst, focus = _relabel(rng, ns + nt, src, dst, [0, 1, 2, ns, ns + 1, ns + 2, ns + nt - 1])
    return Shape(ns + nt, src, dst, focus)


def selfloop_shape():
    """Self-loops only, up to 40 parallel ones per vertex: every vertex is in class 0, some rows are long."""
    rng = np.random.default_rng(50)
    n = 3000
    k = np.where(rng.random(n) < 0.05, rng.integers(32, 41, n), rng.integers(1, 4, n))
    v = np.repeat(np.arange(n), k)
    return Shape(n, v, v.copy(), [0, 1, int(np.argmax(k)), n - 1])


def inonly_isolated_shape():
    """An in-only hub of in-degree 3000, every fifth vertex isolated (interleaved with the others), and the last
    vertex isolated."""
    rng = np.random.default_rng(60)
    n = 4000
    live = np.array([i for i in range(n - 1) if i % 5])
    src = rng.choice(live, 12000)
    dst = rng.choice(live, 12000)
    hub = int(live[7])
    keep = src != hub
    src, dst = src[keep], dst[keep]
    src = np.concatenate([src, rng.choice(live, 3000)])
    dst = np.concatenate([dst, np.full(3000, hub)])
    keep = src != hub
    return Shape(n, src[keep], dst[keep], [hub, 0, 5, 10, int(live[0]), n - 2, n - 1])


def size_shape(n):
    """n vertices with tied degrees (out-degree 2 for all, 3 for every fourth): the edge sort's number of radix
    passes and their parity, and the scan's tile count, follow n.  The random edges keep the graph shallow."""
    i = np.arange(n)
    extra = np.concatenate([i, i[i % 4 == 0]])
    src = np.concatenate([i, extra])
    dst = np.concatenate([(i * 7 + 3) % n, np.random.default_rng(n).integers(0, n, len(extra))])
    return Shape(n, src, dst, sorted({0, n // 2, n - 1}), neg=32 <= n <= 2048)


def multigraph_shape():
    """Parallel edges (up to four copies), each with its own edge id and weight: BIGINT weights below zero, one
    DOUBLE weight NaN."""
    rng = np.random.default_rng(70)
    n = 300
    s, d = rng.integers(0, n, 900), rng.integers(0, n, 900)
    twin = rng.integers(0, 900, 400)
    src = np.concatenate([s, s[twin], s[twin[:100]], s[twin[:30]]])
    dst = np.concatenate([d, d[twin], d[twin[:100]], d[twin[:30]]])
    return Shape(n, src, dst, [int(s[twin[0]]), int(d[twin[0]]), 0, n - 1], neg=True, nan=True)


def lcc_shape():
    """Out-degrees 4095 / 4096 / 4097 around LCC_SMEM, two rows of each, over a background graph that closes
    triangles among their out-neighbours."""
    rng = np.random.default_rng(80)
    nb = 8000
    s, d = _body(rng, nb, 30000)
    src, dst, focus = [s], [d], []
    for i, k in enumerate((4095, 4096, 4097, 4097, 4096, 4095)):
        h = nb + i
        src.append(np.full(k, h))
        dst.append(rng.choice(nb, k, replace=False))
        focus.append(h)
    return Shape(nb + 6, np.concatenate(src), np.concatenate(dst), focus)


def empty_shape(n):
    return Shape(n, np.zeros(0, np.int64), np.zeros(0, np.int64), list(range(n)))


SIZES = [1, 2, 32, 33, 1024, 1025, 2047, 2048, 32768, 32769]
CATALOGUE = {
    "split_m0": (lambda: split_shape(0), {"indeg_1_to_40", "split_31_32_33", "n_short_mod32_0", "slice_width_changes",
                                          "short_padding"}),
    "split_m1": (lambda: split_shape(1), {"indeg_1_to_40", "n_short_mod32_1", "slice_width_changes"}),
    "split_m31": (lambda: split_shape(31), {"indeg_1_to_40", "n_short_mod32_31", "slice_width_changes"}),
    "long_m1": (lambda: long_shape(-1, 0), {"long_start_255", "long_end_255", "long_start_1023", "long_end_1023",
                                            "long_spans_3_ranges", "long_total_mod1024_0"}),
    "long_0": (lambda: long_shape(0, 1), {"long_start_256", "long_end_256", "long_start_1024", "long_end_1024",
                                          "long_spans_3_ranges", "long_total_mod1024_1"}),
    "long_p1": (lambda: long_shape(1, 0), {"long_start_257", "long_end_257", "long_start_1025", "long_end_1025",
                                           "long_spans_3_ranges", "long_total_mod1024_0"}),
    "outdeg_tail": (outdeg_tail_shape, {"outdeg_255", "outdeg_256", "outdeg_257", "outdeg_512", "outdeg_513",
                                        "frontier_items_256", "frontier_items_257", "frontier_edges_1024",
                                        "frontier_edges_1025"}),
    "bipartite": (bipartite_shape, {"class0_empty", "short_padding"}),
    "selfloops": (selfloop_shape, {"only_class0", "parallel_edges"}),
    "inonly_isolated": (inonly_isolated_shape, {"in_only_hub", "isolated_interleaved", "isolated_last"}),
    **{f"n{n}": (lambda n=n: size_shape(n), {f"n_{n}"} | ({"tied_degrees"} if n >= 32 else set())) for n in SIZES},
    "multigraph": (multigraph_shape, {"parallel_edges"}),
    "lcc": (lcc_shape, {"lcc_outdeg_4095", "lcc_outdeg_4096", "lcc_outdeg_4097"}),
    "empty_n1": (lambda: empty_shape(1), {"m0", "n_1"}),
    "empty_n5": (lambda: empty_shape(5), {"m0", "n_5"}),
}
CATALOGUE["n1"][1].add("n1_self_loop")
for _n, _p in ((32, 1), (33, 2), (1024, 2), (1025, 3), (32768, 3), (32769, 4)):
    CATALOGUE[f"n{_n}"][1].add(f"radix_passes_{_p}")
CATALOGUE["n2047"][1].add("scan_n_plus_1_2048")
CATALOGUE["n2048"][1].add("scan_n_plus_1_2049")

REQUIRED = (
    {"indeg_1_to_40", "split_31_32_33", "slice_width_changes", "long_spans_3_ranges", "long_total_mod1024_0",
     "long_total_mod1024_1", "class0_empty", "only_class0", "in_only_hub", "isolated_interleaved", "isolated_last",
     "parallel_edges", "m0", "n1_self_loop", "tied_degrees", "scan_n_plus_1_2048", "scan_n_plus_1_2049"}
    | {f"n_short_mod32_{r}" for r in (0, 1, 31)}
    | {f"long_{w}_{p}" for w in ("start", "end") for p in (255, 256, 257, 1023, 1024, 1025)}
    | {f"outdeg_{d}" for d in (255, 256, 257, 512, 513)}
    | {"frontier_items_256", "frontier_items_257", "frontier_edges_1024", "frontier_edges_1025"}
    | {f"n_{n}" for n in SIZES + [5]} | {f"radix_passes_{p}" for p in (1, 2, 3, 4)}
    | {f"lcc_outdeg_{d}" for d in (4095, 4096, 4097)}
)

_shapes = {}


def shape(name):
    if name not in _shapes:
        _shapes[name] = CATALOGUE[name][0]()
    return _shapes[name]


def weights(sh, kind, seed=0):
    """BIGINT: c + p[u] - p[v] with c >= 0, so every cycle costs >= 0 while single edges may cost less than zero;
    DOUBLE: the same integers as doubles (exact sums), one NaN when the shape asks for it."""
    rng = np.random.default_rng(1000 + seed)
    c = rng.integers(0, 30, len(sh.src))
    if sh.neg:
        p = rng.integers(0, 20, sh.n)
        w = c + p[sh.src] - p[sh.dst]
    else:
        w = c + 1
    w = w.astype(np.int64)
    if kind == "i64":
        return w
    w = w.astype(np.float64)
    if sh.nan and len(w):
        w[len(w) // 2] = np.nan
    return w


# ---- CPU only: the catalogue hits what it names -------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_catalogue_hits_its_boundaries(name):
    sh = shape(name)
    lay = layout(sh.n, sh.src, sh.dst)
    got = hits(lay, [ps for _, ps, _ in tail_calls(sh)])
    want = CATALOGUE[name][1]
    print(f"{name}: n={sh.n} m={len(sh.src)} long={len(lay['long_deg'])}/{lay['long_total']} "
          f"short={lay['n_short']} slices={lay['n_slices']} passes={lay['passes']} hits {sorted(want)}")
    assert want <= got, sorted(want - got)
    if sh.neg:  # reduced costs: no cycle below zero, but single edges below zero
        w = weights(sh, "i64")
        assert np.any(w < 0)


def test_catalogue_covers_every_boundary():
    named = set().union(*(want for _, want in CATALOGUE.values()))
    assert REQUIRED <= named, sorted(REQUIRED - named)


def clamp_shape():
    """Two hubs whose out-degree is above PGQ_DEG_CLAMP (4 194 303): equal sort keys, so their order is free."""
    n = 5000
    k0, k1 = DEG_CLAMP + 7, DEG_CLAMP + 2000
    t = np.arange(k0 + k1, dtype=np.int64) % (n - 2)
    t = t + (t >= 17) + (t >= 4321 - 1)  # targets skip the two hubs
    src = np.concatenate([np.full(k0, 4321), np.full(k1, 17)])
    extra = np.arange(0, n - 1, 3)
    src = np.concatenate([src, extra])
    dst = np.concatenate([t, (extra * 11 + 1) % n])
    return Shape(n, src, dst, [4321, 17, 0, 1, n - 1])


def test_clamp_shape_hits_the_clamp():
    sh = clamp_shape()
    assert "two_above_deg_clamp" in hits(layout(sh.n, sh.src, sh.dst))


# ---- routes --------------------------------------------------------------------------------------------------------------
def _edge_ids(sh, seed=0):
    return np.random.default_rng(2000 + seed).permutation(len(sh.src)).astype(np.int64) * 3 + 5


EDGE_CHUNKS = [1, 97, 2048, STAGE_ROWS, STAGE_ROWS + 1]


def _chunks(m, sizes):
    out, o, i = [], 0, 0
    while o < m:
        out.append((o, min(m, o + sizes[i % len(sizes)])))
        o = out[-1][1]
        i += 1
    return out


def build_chunked(ctx, sh, eid, w, threads):
    """create_csr_vertex counts in shuffled order and uneven chunks, then create_csr_edge chunks of 1 / 97 / 2048 /
    4096 / 4097 rows (one thread, in row order) or dealt to eight threads."""
    n, m = sh.n, len(sh.src)
    csr = pgq.DeviceCSR.create(ctx, n)
    cnt = np.bincount(sh.src, minlength=n).astype(np.int64)
    order = np.random.default_rng(n + m).permutation(n)
    total = 0
    for lo, hi in _chunks(n, [1, 7, 300, 2048, 5000]):
        total += csr.add_vertex_counts(order[lo:hi], cnt[order[lo:hi]])
    assert total == m
    chunks = _chunks(m, EDGE_CHUNKS)

    def feed(part):
        for lo, hi in part:
            csr.add_edges(m, m, sh.src[lo:hi], sh.dst[lo:hi], eid[lo:hi], None if w is None else w[lo:hi])

    if threads == 1:
        feed(chunks)
    else:
        with ThreadPoolExecutor(max_workers=threads) as pool:
            list(pool.map(feed, [chunks[t::threads] for t in range(threads)]))
    csr.finalize()
    return csr


def build_device(ctx, sh, eid):
    import torch
    d_src = torch.from_numpy(np.ascontiguousarray(sh.src, dtype=np.int32)).cuda()
    d_dst = torch.from_numpy(np.ascontiguousarray(sh.dst, dtype=np.int32)).cuda()
    d_eid = None if eid is None else torch.from_numpy(eid).cuda()
    m = len(sh.src)
    return pgq.DeviceCSR.build_device(ctx, sh.n, m, d_src.data_ptr() if m else 0, d_dst.data_ptr() if m else 0,
                                      0 if d_eid is None or not m else d_eid.data_ptr())


# route -> (weight kind or None, threads feeding it, edge ids given)
ROUTES = {
    "build": (None, 1, True), "build_noids": (None, 1, False),
    "device": (None, 1, True), "device_noids": (None, 1, False),
    "upload": (None, 1, True), "upload_noids": (None, 1, False),
    "chunked1": (None, 1, True), "chunked8": (None, 8, True),
    "i64_1": ("i64", 1, True), "i64_8": ("i64", 8, True),
    "f64_1": ("f64", 1, True), "f64_8": ("f64", 8, True),
}


def make(ctx, sh, route, seed=0):
    """-> (csr, expected (v, e, ids, w or None), exact order expected?)"""
    kind, threads, with_ids = ROUTES[route]
    n, m = sh.n, len(sh.src)
    eid = _edge_ids(sh, seed) if with_ids else None
    w = None if kind is None else weights(sh, kind, seed)
    if w is None:
        v, e, ids = orc.csr_build(n, sh.src, sh.dst, eid)
        ow = None
    else:
        v, e, ids, ow = orc.csr_build_weighted(n, sh.src, sh.dst, w, eid)
    if route.startswith("build"):
        csr = pgq.DeviceCSR.build(ctx, n, sh.src, sh.dst, eid)
    elif route.startswith("device"):
        csr = build_device(ctx, sh, eid)
    elif route.startswith("upload"):
        csr = pgq.DeviceCSR.upload(ctx, n, v, e, ids if with_ids else None)
        if not with_ids:
            ids = np.arange(m, dtype=np.int64)  # the CSR position
    else:
        csr = build_chunked(ctx, sh, eid if eid is not None else np.arange(m, dtype=np.int64), w, threads)
    return csr, (v, e, ids, ow), threads == 1


def applicable(sh, route):
    return not (ROUTES[route][0] and len(sh.src) == 0)  # an edgeless chunked build has no weight type


# ---- checks --------------------------------------------------------------------------------------------------------------
def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.itemsize]) if a.dtype.kind == "f" else a


def triples(n, v, e, ids, w):
    """Every vertex's (edge, id, weight) triples in a canonical order."""
    row = np.repeat(np.arange(n), np.diff(np.asarray(v[:n + 1], dtype=np.int64)))
    cols = [np.zeros(len(e), np.int64) if w is None else bits(w).astype(np.int64), ids, e, row]
    order = np.lexsort(cols)
    return [np.asarray(c)[order] for c in cols]


def check_download(csr, sh, exp, exact):
    v, e, ids, w = exp
    dv, de, dids = csr.download()
    dw = None if w is None else csr.download_weights()
    if w is not None:
        assert csr.weight_type() == (2 if w.dtype == np.float64 else 1) and dw.dtype == w.dtype
    assert np.array_equal(dv, v)
    if exact:
        assert np.array_equal(de, e) and np.array_equal(dids, ids)
        if w is not None:
            assert np.array_equal(bits(dw), bits(w))
    else:  # concurrent feeding: the order inside a vertex is the arrival order
        for a, b in zip(triples(sh.n, v, e, ids, w), triples(sh.n, dv, de, dids, dw)):
            assert np.array_equal(a, b)
    return dv, de, dids, dw


_oracle_cache = {}


def _oracle(tag, fn, *args):
    """The restatement's answer, computed once per CSR content and query (args: every array the answer depends on)."""
    h = hashlib.sha1(tag.encode())
    for a in args:
        if a is not None:
            h.update(np.ascontiguousarray(a).tobytes() if isinstance(a, np.ndarray) else repr(a).encode())
    key = h.hexdigest()
    if key not in _oracle_cache:
        _oracle_cache[key] = fn()
    return _oracle_cache[key]


def make_pairs(sh, v, e, seed, k=300):
    """The focus vertices as sources and as destinations, plus random pairs (most destinations with in-edges),
    repeated sources, src == dst rows and a few NULL sources, shuffled."""
    rng = np.random.default_rng(seed)
    n = sh.n
    focus = np.asarray(sh.focus, dtype=np.int64)
    indeg = np.bincount(e, minlength=n)[:n]
    has_in = np.flatnonzero(indeg > 0)
    if len(has_in) == 0:
        has_in = np.arange(n)
    rs = rng.integers(0, n, k)
    rd = np.where(rng.random(k) < 0.7, rng.choice(has_in, k), rng.integers(0, n, k))
    ps = np.concatenate([focus, rs, rng.integers(0, n, len(focus)), focus[:5]])
    pd = np.concatenate([rng.permutation(focus) if len(focus) else focus, rd, focus, focus[:5]])
    sv = np.ones(len(ps), np.uint8)
    sv[rng.choice(len(ps), 3)] = 0
    order = rng.permutation(len(ps))
    return ps[order], pd[order], sv[order]


def cheapest_rows(ps, pd, sv):
    """The cheapest_path_length rows of a pair list: the first 150, every 37th destination NULL."""
    q = slice(0, 150)
    dv = np.ones(len(pd[q]), np.uint8)
    dv[::37] = 0
    return ps[q], pd[q], sv[q], dv


ALL_CONFIGS = [(sched, lanes, rb) for sched in "bpta" for lanes in (64, 512) for rb in (False, True)]
SOME_CONFIGS = [("b", 64, True), ("p", 512, False), ("t", 64, False), ("a", 512, True)]


def check_consumers(csr, sh, dl, monkeypatch, configs=ALL_CONFIGS, seed=0):
    """Every consumer of the CSR against the restatement run on the downloaded CSR dl = (v, e, ids, w)."""
    n = sh.n
    v, e, ids, w = dl
    big = n > 5000  # the restatement scans every vertex per level and batch: fewer rows on the large shapes
    ps, pd, sv = make_pairs(sh, v, e, seed, k=60 if big else 300)
    row = np.repeat(np.arange(n), np.diff(v[:n + 1]))
    canon = e[np.lexsort((e, row))]  # lengths and counters do not depend on the order inside a row
    for sched, lanes, rb in configs:
        monkeypatch.setenv("PGQ_B200_SCHEDULE", sched)
        out, valid, st = csr.iterativelength(ps, pd, sv, pgq.Options(lanes, reference_batching=rb))
        if rb:
            exp, expv, ost = _oracle("il", lambda: orc.iterativelength(n, v, e, ps, pd, sv, lanes), v, canon, ps, pd, sv,
                                         lanes)
        else:
            exp, expv, ost, _ = _oracle("ilx", lambda: orc.iterativelength_ex(n, v, e, ps, pd, sv, lanes, prune=True, dedup=True),
                                          v, canon, ps, pd, sv, lanes)
        assert np.array_equal(valid, expv) and np.array_equal(out, exp), (sched, lanes, rb)
        assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
            ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices), (sched, lanes, rb)
    monkeypatch.delenv("PGQ_B200_SCHEDULE")
    q = slice(0, 20 if big else 120)
    exp_paths, _ = _oracle("sp", lambda: orc.shortestpath(n, v, e, ids, ps[q], pd[q], sv[q], 512), v, e, ids, ps[q], pd[q],
                          sv[q])
    for lanes in (64, 256):
        got, _ = csr.shortestpath(ps[q], pd[q], sv[q], pgq.Options(lanes))
        assert got == exp_paths, lanes
    if w is not None and n <= 20000:  # (a sweep relaxes every edge of the graph: the restatement takes ~10 s per batch
        cs, cd, csv, cdv = cheapest_rows(ps, pd, sv)  # of the 32 768-vertex shapes)
        cost, cvalid, _ = csr.cheapest_path_length(cs, cd, csv, cdv)
        ocost, ovalid = _oracle("cp", lambda: orc.cheapest_path_length(n, v, e, w, cs, cd, csv, cdv), v, e, w, cs, cd,
                                csv, cdv)
        assert np.array_equal(cvalid, ovalid) and np.array_equal(bits(cost[cvalid == 1]), bits(ocost[ovalid == 1]))
    check_analytics(csr, sh, dl)


def check_analytics(csr, sh, dl):
    n = sh.n
    v, e, _, _ = dl
    ids = np.arange(-1, n + 3, dtype=np.int64)
    pr, prv, it, _ = csr.pagerank(ids)
    opr, oprv, oit = _oracle("pr", lambda: orc.pagerank(n, v, e, ids), v, e, ids)
    assert it == oit and np.array_equal(prv, oprv) and np.array_equal(bits(pr[prv == 1]), bits(opr[oprv == 1]))
    wcc, wv, _ = csr.weakly_connected_component(ids)
    owcc, owv = _oracle("wcc", lambda: orc.weakly_connected_component(n, v, e, ids), v, e, ids)
    assert np.array_equal(wv, owv) and np.array_equal(wcc[wv == 1], owcc[owv == 1])
    if n <= 5000:
        q = np.arange(n, dtype=np.int64)
    else:
        q = np.concatenate([np.asarray(sh.focus, dtype=np.int64), np.random.default_rng(n).integers(0, n, 1500)])
    q = np.concatenate([q, q[: len(q) // 4]])  # duplicates
    qv = np.ones(len(q), np.uint8)
    qv[1::11] = 0  # NULLs
    lcc, lv, _ = csr.local_clustering_coefficient(q, qv)
    olcc, olv = _oracle("lcc", lambda: orc.local_clustering_coefficient(n, v, e, q, qv), v, e, q, qv)
    assert np.array_equal(lv, olv) and np.array_equal(bits(lcc[lv == 1]), bits(olcc[olv == 1]))


# ---- GPU: every shape, every route, every consumer, and a replica of each ----------------------------------------------
@pytest.fixture(scope="module")
def replica_ctx():
    ctx = pgq.Context(0)
    yield ctx
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_shape_route_consumers(gpu_ctx, replica_ctx, monkeypatch, name, route):
    sh = shape(name)
    if not applicable(sh, route):
        pytest.skip("an edgeless chunked build carries no weights")
    csr, exp, exact = make(gpu_ctx, sh, route)
    rep = None
    try:
        dl = check_download(csr, sh, exp, exact)
        check_consumers(csr, sh, dl, monkeypatch)
        rep = csr.clone(replica_ctx)
        assert check_download(rep, sh, dl, True) is not None
        check_consumers(rep, sh, dl, monkeypatch, SOME_CONFIGS)
    finally:
        if rep is not None:
            rep.free()
        csr.free()


# ---- GPU: recycled buffers on one workspace --------------------------------------------------------------------------------
def relabelled(sh, k):
    """The same degree structure under a vertex permutation: every array of the device CSR has the same size, the
    contents differ."""
    if k == 0:
        return sh
    rng = np.random.default_rng(500 + k)
    src, dst, focus = _relabel(rng, sh.n, sh.src, sh.dst, sh.focus)
    return Shape(sh.n, src, dst, focus, sh.neg, sh.nan)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["build", "upload_noids", "i64_1", "f64_8"])
@pytest.mark.parametrize("name", ["split_m1", "long_0", "outdeg_tail"])
def test_dirty_buffers_one_workspace(monkeypatch, name, route):
    """A fresh context with one workspace: every build and every call shares it, and each CSR takes the freed,
    uncleared buffers of the one before, which has the same sizes but other contents.  Searches, cheapest paths and
    analytics alternate."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        size = None
        for k in range(4):
            sh = relabelled(shape(name), k)
            csr, exp, exact = make(ctx, sh, route, seed=k)
            try:
                if size is None:
                    size = csr.info()[2]
                assert csr.info()[2] == size  # equal sizes: every buffer comes back from the cache
                dl = check_download(csr, sh, exp, exact)
                if k % 2:
                    check_analytics(csr, sh, dl)
                check_consumers(csr, sh, dl, monkeypatch, SOME_CONFIGS[k % 2:] + SOME_CONFIGS[:k % 2], seed=k)
            finally:
                csr.free()
    finally:
        ctx.close()


# ---- GPU: replicas ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,route", [("split_m0", "i64_1"), ("multigraph", "i64_8"), ("long_0", "f64_1"),
                                        ("n1025", "device")])
def test_replica_outlives_its_primary(monkeypatch, name, route):
    """A replica answers after its primary is freed and a new CSR of the same sizes took the primary's buffers; a
    clone of the clone answers too.  split_m0's BIGINT weights go below zero, and some of its cheapest rows are
    reached only through vertices the search never reaches (test_negative_weight_rows_need_unreached_relaxation), so
    cheapest_path_length on its replicas relies on the copied neg_weights flag."""
    ctx_a, ctx_b = pgq.Context(0), pgq.Context(0)
    live = []
    try:
        sh = shape(name)
        prim, exp, exact = make(ctx_a, sh, route)
        live.append(prim)
        dl = check_download(prim, sh, exp, exact)
        rep = prim.clone(ctx_b)
        live.append(rep)
        prim.free()
        sh2 = relabelled(sh, 1)
        other, exp2, exact2 = make(ctx_a, sh2, route, seed=1)
        live.append(other)
        dl2 = check_download(other, sh2, exp2, exact2)
        check_consumers(rep, sh, dl, monkeypatch)
        check_consumers(other, sh2, dl2, monkeypatch, SOME_CONFIGS)
        rep2 = rep.clone(ctx_a)
        live.append(rep2)
        rep.free()
        check_download(rep2, sh, dl, True)
        check_consumers(rep2, sh, dl, monkeypatch, SOME_CONFIGS)
    finally:
        for c in live:
            c.free()
        ctx_a.close()
        ctx_b.close()


NO_PATH = np.iinfo(np.int64).max


def test_negative_weight_rows_need_unreached_relaxation():
    """The BIGINT replica case of split_m0 tells a CSR with neg_weights from one without: the reference relaxes from
    every vertex, unreached ones too (they start at max / 2), so a target reached at a cost below zero from a vertex
    the source never reaches gets a valid, huge cost.  A Bellman-Ford that relaxes only from reached vertices (what
    the device does without the flag) gives another answer on some of the rows the replica test sends."""
    sh = shape("split_m0")
    n = sh.n
    w = weights(sh, "i64")
    v, e, _, cw = orc.csr_build_weighted(n, sh.src, sh.dst, w, _edge_ids(sh))
    cs, cd, csv, cdv = cheapest_rows(*make_pairs(sh, v, e, 0))
    cost, valid = orc.cheapest_path_length(n, v, e, cw, cs, cd, csv, cdv)
    row = np.repeat(np.arange(n), np.diff(v[:n + 1]))
    srcs = np.unique(cs)
    d = np.full((n, len(srcs)), NO_PATH, dtype=np.int64)
    d[srcs, np.arange(len(srcs))] = 0
    for _ in range(n + 1):
        du = d[row]
        cand = np.where(du != NO_PATH, np.where(du != NO_PATH, du, 0) + cw[:, None], NO_PATH)
        new = d.copy()
        np.minimum.at(new, e, cand)
        if np.array_equal(new, d):
            break
        d = new
    reached = d[cd, np.searchsorted(srcs, cs)]
    reached_valid = (reached != NO_PATH) & (csv == 1) & (cdv == 1)
    assert np.any(reached_valid != (valid == 1)) or np.any(reached[valid == 1] != cost[valid == 1])


# ---- GPU: k_tail's limits, one batch per hub ----------------------------------------------------------------------------
LEVEL = re.compile(r"\[pgq\] batch (\d+) level (\d+) (push|pull|tail) frontier_v=(\d+) frontier_e=(\d+) items=(-?\d+)")


@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["t", "pt", "a"])
def test_tail_limits_one_batch_per_hub(gpu_ctx, monkeypatch, capfd, schedule):
    """Each call sends rows that all start at one tail hub, so the level-1 frontier of its batch is the hub's:
    exactly 256 / 257 work items or 1024 / 1025 out-edges.  The per-level trace shows that frontier at level 2, and
    under t / pt level 2 runs k_tail exactly when the frontier is within both limits.  Lengths, counters and paths
    equal the restatement's."""
    sh = shape("outdeg_tail")
    lay = layout(sh.n, sh.src, sh.dst)
    csr, exp, exact = make(gpu_ctx, sh, "build")
    try:
        v, e, ids, _ = check_download(csr, sh, exp, exact)
        monkeypatch.setenv("PGQ_B200_TRACE", "1")
        monkeypatch.setenv("PGQ_B200_BATCH_STREAMS", "1")
        monkeypatch.setenv("PGQ_B200_SCHEDULE", schedule)
        seen = set()
        for h, ps, pd in tail_calls(sh):
            fv, items, fe = frontier_of(lay, [h])
            eligible = items <= TAIL_ITEMS and fe <= TAIL_EDGES
            seen.add((items, fe, eligible))
            for lanes, rb in ((64, True), (64, False), (512, True)):
                capfd.readouterr()
                out, valid, st = csr.iterativelength(ps, pd, None, pgq.Options(lanes, reference_batching=rb))
                if rb:
                    o, ov, ost = orc.iterativelength(sh.n, v, e, ps, pd, None, lanes)
                else:
                    o, ov, ost, _ = orc.iterativelength_ex(sh.n, v, e, ps, pd, None, lanes, prune=True, dedup=True)
                assert np.array_equal(out, o) and np.array_equal(valid, ov), (h, lanes, rb)
                assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
                    ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices), (h, lanes, rb)
                level2 = [(kind, int(a), int(b)) for _, lv, kind, a, b, _ in LEVEL.findall(capfd.readouterr().err)
                          if lv == "2"]
                assert level2 and all((a, b) == (fv, fe) for _, a, b in level2), (h, level2, fv, fe)
                if schedule in ("t", "pt"):
                    assert {kind for kind, _, _ in level2} == {"tail" if eligible else "push"}, (h, level2)
            paths, _ = csr.shortestpath(ps, pd, None, pgq.Options(64))
            assert paths == orc.shortestpath(sh.n, v, e, ids, ps, pd, None, 512)[0]
        assert seen == {(256, 256, True), (257, 257, False), (128, 1024, True), (128, 1025, False)}
    finally:
        csr.free()


# ---- GPU: the reference's batch loop around rows that take no lane ------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("searching,tail", [(64, "null+same"), (128, "null"), (63, "null+same"), (64, "")])
def test_reference_batching_counts_the_trailing_batch(gpu_ctx, searching, tail):
    """With the reference's batch composition the batch loop starts one more batch when the last one filled every
    lane and rows that take no lane follow (NULL rows; for lengths also src == dst): that batch finds no lane and
    ends at once.  batches must count it, for iterativelength and shortestpath alike."""
    sh = shape("n1025")
    csr, exp, exact = make(gpu_ctx, sh, "build")
    try:
        v, e, ids, _ = check_download(csr, sh, exp, exact)
        rng = np.random.default_rng(searching)
        ps = rng.permutation(sh.n)[:searching]
        pd = (ps + 1 + rng.integers(0, sh.n - 1, searching)) % sh.n  # never the source
        sv = [1] * searching
        if "null" in tail:
            ps, pd, sv = np.append(ps, 5), np.append(pd, 9), sv + [0]
        if "same" in tail:
            ps, pd, sv = np.append(ps, 7), np.append(pd, 7), sv + [1]
        sv = np.array(sv, dtype=np.uint8)
        opts = pgq.Options(64, reference_batching=True)
        out, valid, st = csr.iterativelength(ps, pd, sv, opts)
        o, ov, ost = orc.iterativelength(sh.n, v, e, ps, pd, sv, 64)
        assert np.array_equal(out, o) and np.array_equal(valid, ov)
        assert (st["batches"], st["levels"], st["edges_traversed"], st["frontier_vertices"]) == (
            ost.batches, ost.levels, ost.edges_traversed, ost.frontier_vertices)
        paths, pst = csr.shortestpath(ps, pd, sv, opts)
        opaths, opst = orc.shortestpath(sh.n, v, e, ids, ps, pd, sv, 64)
        assert paths == opaths and pst["batches"] == opst.batches
        if searching % 64 == 0 and "null" in tail:
            assert ost.batches == searching // 64 + 1 and opst.batches == searching // 64 + 1
    finally:
        csr.free()


# ---- GPU: degrees above the sort key's clamp ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_degrees_above_the_clamp(gpu_ctx, monkeypatch):
    """Two hubs with out-degree above PGQ_DEG_CLAMP (about 8.4 M edges): their sort keys tie, so which comes first
    internally is free, and no answer may depend on it."""
    sh = clamp_shape()
    csr, exp, exact = make(gpu_ctx, sh, "build")
    try:
        dl = check_download(csr, sh, exp, exact)
        check_consumers(csr, sh, dl, monkeypatch, SOME_CONFIGS)
    finally:
        csr.free()
