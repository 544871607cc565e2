"""pagerank, weakly_connected_component and local_clustering_coefficient at the boundaries of their own kernels
(csrc/pgq_analytics.cu), where test_gpu_graph_analytics.py takes whatever degrees, dangling counts and component
structure its generators give and test_csr_layout_shapes.py aims at the CSR layout.

- a catalogue of deterministic shapes, each naming the kernel boundaries it hits: the number of dangling entries
  around the 32-value groups and 128-value blocks of k_pr_dangling_fold, in-degrees around warp_fold's groups with
  contributions of very different size in one in-list, n around the pass counts of the in-list sort, PageRank runs
  of 1, 2 and many iterations; mutual pairs, hook chains, many Boruvka rounds, edge counts around k_wcc_compact's
  warps, trees in both directions; out-list lengths around k_lcc_rows' padded sizes, repeats, self-loops, counts
  above 2^24.  A CPU-only test recomputes from the edge rows what the kernels see (a numpy restatement of the
  Boruvka rounds included) and asserts that every named boundary is hit;
- CPU only: the oracle (oracle/pgq_oracle.c) on these shapes against independent references: scipy's partition, a
  Python Link loop, the PageRank iteration in long double, an exact integer triangle count;
- GPU: every shape through pgq_csr_build and a subset through the other construction routes, every answer compared
  with the oracle on the downloaded CSR as bit patterns; the iteration and round counts in the stats; the row
  patterns of one local_clustering_coefficient call; and the three computations in both orders on dirty scratch."""
import os

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc

LCC_SMEM = 4096      # out-lists up to this length are sorted in shared memory by k_lcc_rows
RS_BITS = 5          # bits per radix-sort pass
H100_SMS = 132       # k_lcc_rows runs at most sm_count * 16 blocks, k_wcc_compact strides by sm_count * 16 * 256
COMPACT_STRIDE = H100_SMS * 16 * 256

DANGLING = [2, 3, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 159, 160, 161, 255, 256, 257, 384, 385]
INDEG = [0, 1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 3000]
SIZES = [1, 2, 31, 32, 33, 1023, 1024, 1025, 32768, 32769]
COMPACT = [1, 31, 32, 33, 255, 256, 257]
LCC_K = [2, 3, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.itemsize]) if a.dtype.kind == "f" else a


def indeg_name(k):
    return f"indeg_{k}_mixed" if k > 1 else f"indeg_{k}"


def bits_for(count):
    b = 1
    while b < 31 and (1 << b) < count:
        b += 1
    return b


# ---- what the kernels see, in numpy ------------------------------------------------------------------------------------
def ref_csr(n, src, dst):
    """The reference's CSR: rows by source id, a row's edges in arrival order -> (v[n + 2], row of every position, e)."""
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    order = np.argsort(src, kind="stable")
    v = np.zeros(n + 2, dtype=np.int64)
    v[1:n + 1] = np.cumsum(np.bincount(src, minlength=n)[:n])
    v[n + 1] = len(src)
    return v, src[order], dst[order]


def boruvka(n, rows, e):
    """k_wcc_min / k_wcc_hook / k_wcc_jump / k_wcc_compact round by round, keys = reference CSR position (unique, so
    every choice is defined by the algorithm) -> dict(rounds, mutual1, chain, counts, merges [(position, a, b)])."""
    a, b, k = rows.copy(), e.copy(), np.arange(len(e), dtype=np.int64)
    comp = np.arange(n, dtype=np.int64)
    none = np.iinfo(np.int64).max
    out = dict(rounds=0, mutual1=0, chain=0, counts=[], merges=[])
    while len(k):
        ca, cb = comp[a], comp[b]
        x = ca != cb
        best = np.full(n, none)
        np.minimum.at(best, ca[x], k[x])
        np.minimum.at(best, cb[x], k[x])
        pos_a, pos_b = np.full(len(e), -1), np.full(len(e), -1)  # ends of the edge at a position
        pos_a[k], pos_b[k] = a, b
        c = np.flatnonzero(best != none)  # (only roots have incident edges: comp[] holds roots)
        ea, eb = pos_a[best[c]], pos_b[best[c]]
        o = np.where(comp[ea] == c, comp[eb], comp[ea])
        mutual = best[o] == best[c]
        hook = np.arange(n, dtype=np.int64)
        hook[c] = np.where(mutual & (c < o), c, o)
        rec = ~mutual | (c < o)
        out["merges"] += list(zip(best[c][rec].tolist(), ea[rec].tolist(), eb[rec].tolist()))
        if out["rounds"] == 0:
            out["mutual1"] = int(np.count_nonzero(mutual)) // 2
        depth = (hook != np.arange(n)).astype(np.int64)  # list ranking by doubling: the length of every hook chain
        while True:
            nxt = hook[hook]
            if np.array_equal(nxt, hook):
                break
            depth, hook = depth + depth[hook], nxt
        out["chain"] = max(out["chain"], int(depth.max()) if n else 0)
        comp = hook[comp]
        keep = comp[a] != comp[b]
        a, b, k = a[keep], b[keep], k[keep]
        out["rounds"] += 1
        out["counts"].append(len(k))
    out["merges"].sort()
    return out


def link_labels(n, edges):
    """The reference's labels: forest of n + 2 entries, entry i its own root for i <= n and entry n + 1 left at 0;
    Link(a, b) for every edge in the given order hangs root(a) under root(b); roots are found with path halving."""
    forest = list(range(n + 1)) + [0]

    def root(x):
        while forest[x] != x:
            forest[x] = forest[forest[x]]
            x = forest[x]
        return x

    for a, b in edges:
        ra, rb = root(a), root(b)
        if ra != rb:
            forest[ra] = rb
    return np.array([root(x) for x in range(n + 2)], dtype=np.int64)


def pagerank_longdouble(n, rows, e):
    """The reference's iteration (vsize = n + 2 entries, damping 0.85, the rank of the entries without out-edges
    spread over all, stop when the largest change is below 1e-6) in long double -> (ranks, iterations, the least
    distance of any iteration's largest change from the threshold)."""
    L = np.longdouble
    vs = n + 2
    od = np.bincount(rows, minlength=vs).astype(np.int64)
    order = np.argsort(e, kind="stable")
    srcs, tg = rows[order], e[order]
    starts = np.flatnonzero(np.concatenate([[True], tg[1:] != tg[:-1]])) if len(tg) else np.zeros(0, np.int64)
    rank = np.full(vs, L(1) / L(vs))
    d, iters, margin = L(0.85), 0, np.inf
    while True:
        contrib = np.where(od > 0, rank / np.maximum(od, 1).astype(L), L(0))
        temp = np.zeros(vs, dtype=L)
        if len(tg):
            temp[tg[starts]] = np.add.reduceat(contrib[srcs], starts)
        new = (L(1) - d) / L(vs) + d * (temp + rank[od == 0].sum() / L(vs))
        delta = float(np.abs(new - rank).max())
        rank, iters, margin = new, iters + 1, min(margin, abs(delta - 1e-6))
        if delta < 1e-6:
            return rank, iters, margin


def lcc_exact(n, v, e, q):
    """(integer count, k) per queried vertex: over the out-neighbours u of s, with multiplicity, the entries of u's
    list that are out-neighbours of s."""
    counts, ks = np.zeros(len(q), dtype=np.int64), np.zeros(len(q), dtype=np.int64)
    memo = {}
    for r, s in enumerate(np.asarray(q).tolist()):
        if s not in memo:
            nb = e[v[s]:v[s + 1]]
            total = 0
            if len(nb) >= 2:
                uniq, mult = np.unique(nb, return_counts=True)
                for u, times in zip(uniq.tolist(), mult.tolist()):
                    total += times * int(np.count_nonzero(np.isin(e[v[u]:v[u + 1]], uniq)))
            memo[s] = (total, len(nb))
        counts[r], ks[r] = memo[s]
    return counts, ks


def lcc_float(counts, ks):
    k = ks.astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = counts.astype(np.float32) / (k * (k - np.float32(1.0)))
    return np.where(ks >= 2, out, np.float32(0.0)).astype(np.float32)


# ---- the catalogue ------------------------------------------------------------------------------------------------------
def _relabel(seed, n, src, dst):
    p = np.random.default_rng(seed).permutation(n)
    return n, p[np.asarray(src, dtype=np.int64)], p[np.asarray(dst, dtype=np.int64)]


def _cat(parts):
    return np.concatenate([np.asarray(p, dtype=np.int64).ravel() for p in parts]) if parts else np.zeros(0, np.int64)


def edgeless(n):
    return n, np.zeros(0, np.int64), np.zeros(0, np.int64)


def dangling_shape(c):
    """Exactly c entries without out-edges, n and n + 1 among them: 40 live vertices on a ring with chords, and c - 2
    sinks fed by one to nine live vertices of different out-degree, so their ranks differ.  Ids shuffled: the sinks
    lie between the live vertices."""
    rng = np.random.default_rng(100 + c)
    live, sinks = 40, c - 2
    src, dst = [np.arange(live)], [(np.arange(live) + 1) % live]
    heavy = rng.integers(0, live, 150)
    src.append(heavy // 4)  # vertices 0 .. 9 get many chords
    dst.append(rng.integers(0, live, 150))
    for s in range(sinks):
        k = 1 + s % 9
        src.append(rng.integers(0, live, k))
        dst.append(np.full(k, live + s))
    return _relabel(c, live + sinks, _cat(src), _cat(dst))


def indeg_shape(small=False):
    """Two targets of every in-degree in INDEG over 2000 filler vertices, half of them without out-edges.  A third of a target's in-edges come from sources of out-degree 1, the
    rest from six sources of out-degree about 10^4 and sixty of out-degree about 30, so one in-list holds
    contributions four orders of magnitude apart.  Ids shuffled.  small: a tenth of it, without in-degree 3000."""
    rng = np.random.default_rng(200)
    fill, heavy, medium, hdeg = (200, 6, 60, 1000) if small else (2000, 6, 60, 10000)
    hv = np.arange(fill, fill + heavy)
    md = np.arange(fill + heavy, fill + heavy + medium)
    src = [np.repeat(hv, hdeg), np.repeat(md, 30), np.repeat(np.arange(fill // 2), 2)]
    dst = [rng.integers(0, fill, heavy * hdeg), rng.integers(0, fill, medium * 30), rng.integers(0, fill, fill)]
    nxt = fill + heavy + medium
    targets = []
    for k in [k for k in INDEG if not (small and k > 100)] * 2:
        targets.append((nxt, k))
        nxt += 1
    for t, k in targets:
        own = -(-k // 3)
        src += [np.arange(nxt, nxt + own), hv[:min(1, k - own)], rng.choice(np.concatenate([hv, md]), max(k - own - 1, 0))]
        dst += [np.full(k, t)]
        nxt += own
    # the targets of in-degree > 0 point back into the filler, so that they are not all dangling
    src.append([t for t, k in targets if k])
    dst.append(rng.integers(0, fill, sum(1 for _, k in targets if k)))
    return _relabel(201, nxt, _cat(src), _cat(dst))


def size_shape(n):
    """n vertices: a permutation cycle, self-loops on every fifth vertex, 3 n random edges whose sources are skewed
    (a few sources have out-degree in the hundreds), and a sixth of all rows twice (parallel edges in one in-list)."""
    rng = np.random.default_rng(300 + n)
    i = np.arange(n)
    src = _cat([i, i[::5], (rng.random(3 * n) ** 3 * n).astype(np.int64)])
    dst = _cat([(i * 7 + 3) % n, i[::5], rng.integers(0, n, 3 * n)])
    twice = rng.integers(0, len(src), len(src) // 6 + 1)
    src, dst = _cat([src, src[twice]]), _cat([dst, dst[twice]])
    p = rng.permutation(len(src))
    return n, src[p], dst[p]


def path_into_sink(n):
    """A directed path into a sink, ids shuffled: the rank of the k-th vertex settles only after k iterations."""
    return _relabel(400 + n, n, np.arange(n - 1), np.arange(1, n))


def two_cycle_with_tail():
    """a <-> b fed by a 25-long tail."""
    t = np.arange(25)
    return _relabel(410, 27, _cat([t, [25, 26]]), _cat([t + 1, [26, 25]]))


def complete_digraph(n):
    i = np.repeat(np.arange(n), n)
    j = np.tile(np.arange(n), n)
    return _relabel(420, n, i[i != j], j[i != j])


def parallel_x3():
    rng = np.random.default_rng(430)
    s, d = rng.integers(0, 500, 1500), rng.integers(0, 500, 1500)
    p = rng.permutation(4500)
    return 500, np.tile(s, 3)[p], np.tile(d, 3)[p]


def matching(pairs, both=True, loops=False):
    """A perfect matching, a -> b and b -> a: the pair's first edge is the least edge of both ends, so every component
    is a mutual pair in round 1 and no edge is left for round 2.  Ids shuffled."""
    a, b = np.arange(pairs) * 2, np.arange(pairs) * 2 + 1
    src, dst = [a], [b]
    if both:
        src.append(b), dst.append(a)
    if loops:
        src.append(a[::3]), dst.append(a[::3])
    return _relabel(500 + pairs, 2 * pairs, _cat(src), _cat(dst))


def selfloops_only():
    v = np.repeat(np.arange(300), 1 + np.arange(300) % 3)
    return 300, v, v.copy()


def path_increasing(n):
    """i + 1 -> i with identity ids, so the positions increase along the path: every vertex's least edge is its own,
    to its predecessor, and round 1 hooks the whole path into one chain of depth n - 2 that pointer jumping has to
    fold.  Vertex 0 ends as the root of everything."""
    return n, np.arange(1, n), np.arange(n - 1)


def path_bit_reversed(log_n):
    """A path over bit-reversed ids: neighbours on the path are far apart in id, the least edges pair the vertices
    up, and a round only about halves the number of components."""
    n = 1 << log_n
    i = np.arange(n)
    rev = np.zeros(n, dtype=np.int64)
    for b in range(log_n):
        rev |= ((i >> b) & 1) << (log_n - 1 - b)
    return n, rev[:-1], rev[1:]


def binary_tree(n):
    c = np.arange(1, n)
    return _relabel(520, n, (c - 1) // 2, c)


def caterpillar():
    spine, legs = 500, 3
    s = np.arange(spine - 1)
    j = np.arange(spine * legs)
    return _relabel(530, spine * (legs + 1), _cat([s, spine + j]), _cat([s + 1, j // legs]))


def components(c, size):
    """c components of `size` vertices each (a random tree plus a few extra edges), a vertex without edges after
    every component, vertex 0 among those without edges when c > 1."""
    rng = np.random.default_rng(540 + c)
    src, dst = [], []
    first = 1 if c > 1 else 0
    for g in range(c):
        base = first + g * (size + 1)
        child = np.arange(1, size)
        parent = (rng.random(size - 1) * child).astype(np.int64)
        flip = rng.random(size - 1) < 0.5
        extra = rng.integers(0, size, (2, size // 2))
        src += [base + np.where(flip, child, parent), base + extra[0]]
        dst += [base + np.where(flip, parent, child), base + extra[1]]
    n = first + c * (size + 1)
    src, dst = _cat(src), _cat(dst)
    p = rng.permutation(len(src))
    return n, src[p], dst[p]


def _base_tree():
    rng = np.random.default_rng(550)
    n = 600
    child = np.arange(1, n)
    parent = (rng.random(n - 1) * child).astype(np.int64)
    flip = rng.random(n - 1) < 0.5
    p = rng.permutation(n)
    return n, p[np.where(flip, child, parent)], p[np.where(flip, parent, child)]


def tree(variant):
    """One random tree of 600 vertices, as it is, with every edge reversed, with its rows in another arrival order
    (other positions inside a row of the CSR), and with the vertex ids reversed: the partition is the same, the label
    of the component is not."""
    n, s, d = _base_tree()
    if variant == "reversed_edges":
        return n, d, s
    if variant == "permuted_rows":
        p = np.random.default_rng(551).permutation(n - 1)
        return n, s[p], d[p]
    if variant == "reversed_ids":
        return n, n - 1 - s, n - 1 - d
    return n, s, d


def compact_shape(c):
    """c + 1 pairs a_i -> b_i (a in [0, c], b behind them) and c edges b_i -> a_(i+1).  Positions follow the source
    id, so the pair edges come first: round 1 merges every pair as a mutual pair, and exactly the c edges between
    the pairs survive its compaction; self-loops and b_i -> a_i copies are dropped between them."""
    k = c + 1
    a, b = np.arange(k), k + np.arange(k)
    return 2 * k, _cat([a, b[:-1], b, b[::2]]), _cat([b, a[1:], a, b[::2]])


def compact_stride_shape():
    """One edge more than k_wcc_compact's grid covers in one stride on an H100 (132 SMs): the last edge is the only
    one of the second pass."""
    rng = np.random.default_rng(560)
    n, m = 100000, COMPACT_STRIDE + 1
    return n, rng.integers(0, n, m), rng.integers(0, n, m)


def lcc_k_shape(ks=LCC_K, nb=3000, hub=5000):
    """Out-lists of every length in LCC_K, three heads each: distinct neighbours; neighbours with repeats and the head
    itself (a self-loop); all but one entry the same neighbour.  The background graph (3000 vertices, a hub of
    out-degree 5000 among them, a quarter without out-edges) closes triangles.  Ids shuffled."""
    rng = np.random.default_rng(600)
    live = np.arange(nb - nb // 4)
    src, dst = [rng.choice(live, 4 * nb), np.full(hub, 7)], [rng.integers(0, nb, 4 * nb), rng.integers(0, nb, hub)]
    nxt = nb
    for k in ks:
        src += [np.full(k, nxt), np.full(k, nxt + 1), np.full(k, nxt + 2)]
        rep = rng.choice(nb, max(k // 2, 1))
        dst += [np.concatenate([[7], rng.choice(np.arange(8, nb), k - 1, replace=False)]),
                np.concatenate([[nxt + 1], rng.choice(rep, k - 1)]),
                np.concatenate([np.full(k - 1, 11 + k), [12]])]
        nxt += 3
    return _relabel(601, nxt, _cat(src), _cat(dst))


def lcc_words_shape(n):
    """n vertices, vertex n - 1 with 4200 out-edges over all of them (the bitmap path with words = n / 32 + 1 and a
    list of heavy multiplicity), the others with short lists."""
    rng = np.random.default_rng(610 + n)
    src = _cat([np.full(4200, n - 1), rng.integers(0, n - 1, 4 * n)])
    dst = _cat([np.concatenate([np.arange(n), rng.integers(0, n, 4200 - n)]), rng.integers(0, n, 4 * n)])
    p = rng.permutation(len(src))
    return n, src[p], dst[p]


def lcc_big_count_shape():
    """Counts above 2^24, where the conversion to float rounds: vertex 0 lists vertex 1 4095 times (sorted in shared
    memory), vertex 2 lists it 5001 times (bitmap path), and vertex 1 has 4101 self-loops: 4095 * 4101 and
    5001 * 4101 are odd and above 2^24."""
    src = _cat([np.full(4095, 0), np.full(4101, 1), np.full(5001, 2), [3, 3]])
    dst = _cat([np.full(4095, 1), np.full(4101, 1), np.full(5001, 1), [0, 2]])
    return 5, src, dst


SHAPES = {
    **{f"dangling{c}": (lambda c=c: dangling_shape(c), {f"dangling_{c}"}) for c in DANGLING},
    "indeg": (indeg_shape, {indeg_name(k) for k in INDEG} | {"lcc_big_rows_ge_6"}),
    **{f"n{n}": (lambda n=n: size_shape(n), {f"n_{n}", f"sort_passes_{-(-bits_for(n) // RS_BITS)}"}
                 | ({"parallel_in_one_in_list", "self_loops"} if n >= 31 else set())) for n in SIZES},
    "indeg_small": (lambda: indeg_shape(small=True), {indeg_name(k) for k in (31, 32, 33)}),
    "lcc_k_small": (lambda: lcc_k_shape((31, 32, 33), 300, 40), {"lcc_k_31", "lcc_k_32", "lcc_k_33", "lcc_self_in_list",
                                                                 "lcc_repeats"}),
    "edgeless0": (lambda: edgeless(0), {"n_0", "m_0", "pr_iters_1"}),
    "edgeless1": (lambda: edgeless(1), {"m_0", "dangling_3", "pr_iters_1"}),
    "edgeless200": (lambda: edgeless(200), {"m_0", "pr_iters_1"}),
    "self_loop1": (lambda: (1, np.zeros(1, np.int64), np.zeros(1, np.int64)), {"n1_single_self_loop", "dangling_2"}),
    "path60": (lambda: path_into_sink(60), {"pr_iters_ge_40", "wcc_merges_n_minus_1"}),
    "two_cycle_tail": (two_cycle_with_tail, {"pr_iters_ge_40", "dangling_2"}),
    "complete33": (lambda: complete_digraph(33), {"complete_digraph_33", "dangling_2"}),
    "parallel_x3": (parallel_x3, {"every_edge_x3"}),
    "matching": (lambda: matching(1000), {"wcc_all_mutual_round1", "wcc_antiparallel_least_of_both", "wcc_rounds_1",
                                          "wcc_count_0_after_round1", "pr_iters_2", "wcc_components_1000"}),
    "matching_oneway_loops": (lambda: matching(40, both=False, loops=True), {"wcc_all_mutual_round1", "self_loops"}),
    "selfloops_only": (selfloops_only, {"wcc_selfloops_only", "wcc_rounds_1", "lcc_all_one_neighbour"}),
    "path_increasing": (lambda: path_increasing(50000), {"wcc_chain_ge_10000", "wcc_rounds_1", "wcc_merges_n_minus_1",
                                                         "v0_is_root"}),
    "path_bitrev": (lambda: path_bit_reversed(16), {"wcc_rounds_ge_8", "wcc_merges_n_minus_1"}),
    "binary_tree": (lambda: binary_tree(4095), {"wcc_merges_n_minus_1", "wcc_rounds_ge_3"}),
    "caterpillar": (caterpillar, {"wcc_merges_n_minus_1", "wcc_rounds_ge_3"}),
    "components1": (lambda: components(1, 700), {"wcc_components_1"}),
    "components2": (lambda: components(2, 700), {"wcc_components_2", "wcc_singletons_between", "v0_isolated"}),
    "components3": (lambda: components(3, 700), {"wcc_components_3", "wcc_singletons_between", "v0_isolated"}),
    "components1000": (lambda: components(1000, 8), {"wcc_components_1000", "wcc_singletons_between"}),
    "tree": (lambda: tree("base"), {"tree_base", "wcc_merges_n_minus_1"}),
    "tree_reversed_edges": (lambda: tree("reversed_edges"), {"tree_reversed_edges", "wcc_label_differs_from_base"}),
    "tree_permuted_rows": (lambda: tree("permuted_rows"), {"tree_permuted_rows"}),
    "tree_reversed_ids": (lambda: tree("reversed_ids"), {"tree_reversed_ids", "wcc_label_differs_from_base"}),
    **{f"compact{c}": (lambda c=c: compact_shape(c), {f"compact_count_{c}", "v0_not_root"}) for c in COMPACT},
    "compact_stride": (compact_stride_shape, {"compact_stride_plus_1"}),
    "lcc_k": (lcc_k_shape, {f"lcc_k_{k}" for k in LCC_K} | {"lcc_self_in_list", "lcc_repeats", "lcc_all_one_neighbour",
                                                            "lcc_neighbour_with_empty_list", "lcc_neighbour_above_4096",
                                                            "lcc_big_rows_ge_1"}),
    **{f"lcc_words{n}": (lambda n=n: lcc_words_shape(n), {f"lcc_bitmap_n_{n}", "lcc_big_row_multiplicity"})
       for n in (31, 32, 33)},
    "lcc_big_count": (lcc_big_count_shape, {"lcc_count_above_2p24_sorted", "lcc_count_above_2p24_bitmap"}),
}

REQUIRED = (
    {f"dangling_{c}" for c in DANGLING} | {"m_0"}
    | {indeg_name(k) for k in INDEG}
    | {f"n_{n}" for n in [0] + SIZES} | {f"sort_passes_{p}" for p in (1, 2, 3, 4)}
    | {"parallel_in_one_in_list", "self_loops", "pr_iters_1", "pr_iters_2", "pr_iters_ge_40", "n1_single_self_loop",
       "complete_digraph_33", "every_edge_x3"}
    | {"wcc_all_mutual_round1", "wcc_antiparallel_least_of_both", "wcc_selfloops_only", "wcc_count_0_after_round1",
       "wcc_rounds_1", "wcc_rounds_ge_3", "wcc_rounds_ge_8", "wcc_chain_ge_10000", "wcc_merges_n_minus_1",
       "wcc_singletons_between", "tree_base", "tree_reversed_edges", "tree_permuted_rows", "tree_reversed_ids",
       "wcc_label_differs_from_base", "compact_stride_plus_1", "v0_isolated", "v0_is_root", "v0_not_root"}
    | {f"wcc_components_{c}" for c in (1, 2, 3, 1000)} | {f"compact_count_{c}" for c in COMPACT}
    | {f"lcc_k_{k}" for k in LCC_K} | {f"lcc_bitmap_n_{n}" for n in (31, 32, 33)}
    | {"lcc_self_in_list", "lcc_repeats", "lcc_all_one_neighbour", "lcc_neighbour_with_empty_list",
       "lcc_neighbour_above_4096", "lcc_big_rows_ge_1", "lcc_big_rows_ge_6", "lcc_big_row_multiplicity",
       "lcc_count_above_2p24_sorted", "lcc_count_above_2p24_bitmap"}
)

# the shapes the reference binary has answered: tests/golden/refn4_<name>.npz (tests/golden/make_golden_next4.py)
GOLDEN_SHAPES = ["dangling128", "dangling129", "indeg_small", "matching", "tree", "tree_reversed_edges", "lcc_k_small"]

_shapes = {}


def shape(name):
    if name not in _shapes:
        n, s, d = SHAPES[name][0]()
        _shapes[name] = (int(n), np.ascontiguousarray(s, dtype=np.int64), np.ascontiguousarray(d, dtype=np.int64))
    return _shapes[name]


def lcc_queries(name):
    """The rows of the shape's local_clustering_coefficient call: every vertex, or on the large shapes the vertices
    of the largest out-degree and a sample."""
    n, s, _ = shape(name)
    if n <= 12000:
        return np.arange(n, dtype=np.int64)
    top = np.argsort(-np.bincount(s, minlength=n), kind="stable")[:32]
    return np.concatenate([top, np.random.default_rng(n).choice(n, 2000, replace=False)]).astype(np.int64)


def hits(name):
    """Every boundary this shape hits, by name, with the numbers behind them."""
    n, src, dst = shape(name)
    m = len(src)
    v, rows, e = ref_csr(n, src, dst)
    out = {f"n_{n}", f"sort_passes_{-(-bits_for(n) // RS_BITS)}"}
    od = np.bincount(src, minlength=n + 2)          # out-degree of every entry of [0, n + 2)
    ind = np.bincount(dst, minlength=n)[:n]
    dangling = int(np.count_nonzero(od == 0))
    out.add(f"dangling_{dangling}")
    if m == 0:
        out.add("m_0")
    # the in-lists by ascending source: the spread of 1 / out-degree inside each
    order = np.argsort(e, kind="stable")
    tg, sod = e[order], od[rows[order]]
    out |= {f"indeg_{k}" for k in (0, 1) if np.any(ind == k)}
    if m:
        starts = np.flatnonzero(np.concatenate([[True], tg[1:] != tg[:-1]]))
        spread = np.maximum.reduceat(sod, starts) / np.minimum.reduceat(sod, starts)
        for k in INDEG:
            if k > 1 and np.any((ind[tg[starts]] == k) & (spread >= 1000)):
                out.add(f"indeg_{k}_mixed")
        pair = rows * n + e
        if len(np.unique(pair)) < m:
            out.add("parallel_in_one_in_list")
        if np.all(np.unique(pair, return_counts=True)[1] % 3 == 0):
            out.add("every_edge_x3")
        if np.any(rows == e):
            out.add("self_loops")
        if n == 1 and m == 1:
            out.add("n1_single_self_loop")
        if m == n * (n - 1) and len(np.unique(pair)) == m and not np.any(rows == e):
            out.add(f"complete_digraph_{n}")
    if n <= 3000:
        _, iters, _ = pagerank_longdouble(n, rows, e)
        out |= {f"pr_iters_{iters}"} | ({"pr_iters_ge_40"} if iters >= 40 else set())
    # weakly_connected_component
    bo = boruvka(n, rows, e)
    labels = link_labels(n, zip(rows.tolist(), e.tolist()))
    n_comp = len(set(labels[:n].tolist()))
    real = rows != e
    deg = np.bincount(rows[real], minlength=n)[:n] + np.bincount(e[real], minlength=n)[:n]
    big_comp = np.bincount(labels[:n], minlength=n + 2)
    if m:
        out.add(f"wcc_rounds_{bo['rounds']}")
        out |= {f"wcc_rounds_ge_{r}" for r in (3, 8) if bo["rounds"] >= r}
        if not np.any(real):
            out.add("wcc_selfloops_only")
        if np.any(real) and 2 * bo["mutual1"] == np.count_nonzero(deg):
            out.add("wcc_all_mutual_round1")
        if bo["counts"][0] == 0 and np.any(real):
            out.add("wcc_count_0_after_round1")
        if bo["chain"] >= 10000:
            out.add("wcc_chain_ge_10000")
        if len(bo["merges"]) == n - 1:
            out.add("wcc_merges_n_minus_1")
        for c in COMPACT:
            if bo["counts"][0] == c:
                out.add(f"compact_count_{c}")
        if m == COMPACT_STRIDE + 1:
            out.add("compact_stride_plus_1")
        first = {}  # the least position at every vertex
        for k in np.flatnonzero(real)[::-1].tolist():
            first[int(rows[k])] = first[int(e[k])] = k
        anti = set(zip(e[real].tolist(), rows[real].tolist()))
        if any(first[int(rows[k])] == k and first[int(e[k])] == k and (int(rows[k]), int(e[k])) in anti
               for k in np.flatnonzero(real).tolist()):
            out.add("wcc_antiparallel_least_of_both")
        sizes = big_comp[big_comp > 1]
        if len(sizes) and np.all(sizes == sizes[0]):
            out.add(f"wcc_components_{len(sizes)}")
            lone = np.flatnonzero(deg == 0)
            if len(sizes) > 1 and np.any((lone > 0) & (lone < n - 1)):
                out.add("wcc_singletons_between")
        if deg[0] == 0:
            out.add("v0_isolated")
        elif labels[0] == 0:
            out.add("v0_is_root")
        else:
            out.add("v0_not_root")
        bn, bs, bd = _base_tree()
        if n == bn and m == bn - 1:
            same_order = np.array_equal(src, bs) and np.array_equal(dst, bd)
            as_set = lambda a, b: sorted(zip(a.tolist(), b.tolist()))
            if same_order:
                out.add("tree_base")
            elif as_set(src, dst) == as_set(bs, bd):
                out.add("tree_permuted_rows")
            if np.array_equal(src, bd) and np.array_equal(dst, bs):
                out.add("tree_reversed_edges")
            if np.array_equal(n - 1 - src, bs) and np.array_equal(n - 1 - dst, bd):
                out.add("tree_reversed_ids")
            base = link_labels(bn, zip(*[a.tolist() for a in ref_csr(bn, bs, bd)[1:]]))
            if labels[0] != base[0]:
                out.add("wcc_label_differs_from_base")
    # local_clustering_coefficient
    q = lcc_queries(name)
    ks = od[q]
    for k in LCC_K:
        if np.any(ks == k):
            out.add(f"lcc_k_{k}")
    n_big = int(np.count_nonzero(ks > LCC_SMEM))
    out |= {f"lcc_big_rows_ge_{c}" for c in (1, 6) if n_big >= c}
    if n_big and n in (31, 32, 33):
        out.add(f"lcc_bitmap_n_{n}")
    for s in q[(ks >= 2)].tolist():
        nb = e[v[s]:v[s + 1]]
        uniq = np.unique(nb)
        small = len(nb) <= LCC_SMEM
        if small and s in nb:
            out.add("lcc_self_in_list")
        if small and len(uniq) < len(nb):
            out.add("lcc_repeats")
        if small and (len(uniq) == 1 or np.max(np.unique(nb, return_counts=True)[1]) == len(nb) - 1):
            out.add("lcc_all_one_neighbour")
        if small and np.any(od[uniq] == 0):
            out.add("lcc_neighbour_with_empty_list")
        if small and np.any(od[uniq] > LCC_SMEM):
            out.add("lcc_neighbour_above_4096")
        if not small and len(uniq) * 4 < len(nb):
            out.add("lcc_big_row_multiplicity")
    if n <= 100:
        counts, kk = lcc_exact(n, v, e, q)
        for c, k in zip(counts.tolist(), kk.tolist()):
            if c > 1 << 24 and int(np.float32(c)) != c:
                out.add("lcc_count_above_2p24_sorted" if k <= LCC_SMEM else "lcc_count_above_2p24_bitmap")
    return out, dict(n=n, m=m, dangling=dangling, rounds=bo["rounds"], mutual1=bo["mutual1"], chain=bo["chain"],
                     counts=bo["counts"][:4], merges=len(bo["merges"]), components=n_comp, big_rows=n_big)


# ---- CPU only: the catalogue hits what it names ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_hits_its_boundaries(name):
    got, numbers = hits(name)
    want = SHAPES[name][1]
    print(f"{name}: {numbers} hits {sorted(want)}")
    assert want <= got, sorted(want - got)


def test_catalogue_covers_every_boundary():
    named = set().union(*(want for _, want in SHAPES.values()))
    assert named == REQUIRED, (sorted(REQUIRED - named), sorted(named - REQUIRED))


# ---- CPU only: the oracle against independent references ------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_wcc_against_scipy_and_link(name):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    n, src, dst = shape(name)
    v, rows, e = ref_csr(n, src, dst)
    ov, oe, _ = orc.csr_build(n, src, dst)
    assert np.array_equal(ov, v) and np.array_equal(oe, e)
    ids = np.arange(-2, n + 4, dtype=np.int64)
    lab, valid = orc.weakly_connected_component(n, v, e, ids)
    assert valid.tolist() == [0, 0] + [1] * (n + 2) + [0, 0]
    lab = lab[2:n + 4]
    # the labels: Link over every edge in CSR order
    assert np.array_equal(lab, link_labels(n, zip(rows.tolist(), e.tolist())))
    # the partition
    if n:
        _, comp = connected_components(coo_matrix((np.ones(len(e)), (rows, e)), shape=(n, n)), connection="weak")
        _, a = np.unique(lab[:n], return_inverse=True)
        first_a, first_b = {}, {}
        assert [first_a.setdefault(x, i) for i, x in enumerate(a.tolist())] == \
               [first_b.setdefault(x, i) for i, x in enumerate(comp.tolist())]
    assert lab[n] == n and lab[n + 1] == lab[0] if n else lab.tolist() == [0, 0]
    # and the device's argument: the Boruvka merge edges alone, replayed in position order, give the same labels
    bo = boruvka(n, rows, e)
    assert np.array_equal(lab, link_labels(n, [(a, b) for _, a, b in bo["merges"]]))


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_pagerank_against_long_double(name):
    n, src, dst = shape(name)
    v, rows, e = ref_csr(n, src, dst)
    ids = np.arange(n + 2, dtype=np.int64)
    pr, valid, iters = orc.pagerank(n, v, e, ids)
    ref, ref_iters, margin = pagerank_longdouble(n, rows, e)
    assert valid.all()
    assert np.all(np.abs(pr.astype(np.longdouble) - ref) <= 1e-12 * ref)
    assert abs(float(pr.astype(np.longdouble).sum()) - 1.0) <= 1e-12
    if margin > 1e-9:  # otherwise the double and the long double iteration may stop one iteration apart
        assert iters == ref_iters
    else:
        assert abs(iters - ref_iters) <= 1


@pytest.mark.parametrize("name", list(SHAPES))
def test_oracle_lcc_against_integer_count(name):
    n, src, dst = shape(name)
    v, _, e = ref_csr(n, src, dst)
    q = lcc_queries(name)
    if len(q) > 3000:
        od = np.diff(v[:n + 1])
        q = np.concatenate([np.argsort(-od, kind="stable")[:40], np.random.default_rng(7).choice(q, 1500)])
    lcc, valid = orc.local_clustering_coefficient(n, v, e, q)
    counts, ks = lcc_exact(n, v, e, q)
    assert valid.all() and np.array_equal(bits(lcc), bits(lcc_float(counts, ks)))


@pytest.mark.parametrize("name", GOLDEN_SHAPES)
def test_reference_golden_is_of_this_shape(name):
    """tests/golden/refn4_<name>.npz holds what the reference binary answered for exactly this shape (test_oracle_golden
    compares the oracle with it bit for bit, test_gpu_graph_analytics the device); its CSR is ref_csr's, its labels
    are the Link loop's and its ranks the long double iteration's."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"refn4_{name}.npz"))
    n, src, dst = shape(name)
    assert int(g["n"]) == n and np.array_equal(g["src"], src) and np.array_equal(g["dst"], dst)
    v, rows, e = ref_csr(n, src, dst)
    assert np.array_equal(g["csr_v"], v) and np.array_equal(g["csr_e"], e)
    assert np.array_equal(g["wcc"], link_labels(n, zip(rows.tolist(), e.tolist()))[:n])
    ref = pagerank_longdouble(n, rows, e)[0][:n]
    assert np.all(np.abs(g["pagerank"].astype(np.longdouble) - ref) <= 1e-12 * ref)
    q = np.arange(n)
    assert np.array_equal(bits(g["lcc"]), bits(lcc_float(*lcc_exact(n, v, e, q))))


# ---- GPU -----------------------------------------------------------------------------------------------------------------
_oracle_cache, _rounds = {}, {}


def boruvka_rounds(name):
    if name not in _rounds:
        n, src, dst = shape(name)
        _rounds[name] = boruvka(n, *ref_csr(n, src, dst)[1:])["rounds"]
    return _rounds[name]


def oracle_answers(name, v, e):
    """The oracle on the downloaded CSR, once per shape (every route downloads the same CSR, which is asserted)."""
    n = shape(name)[0]
    if name not in _oracle_cache:
        ids = np.arange(-2, n + 4, dtype=np.int64)
        q = lcc_queries(name)
        uq, back = np.unique(q, return_inverse=True)
        olcc, olv = orc.local_clustering_coefficient(n, v, e, uq)
        _oracle_cache[name] = (v.copy(), e.copy(), orc.pagerank(n, v, e, ids), orc.weakly_connected_component(n, v, e, ids),
                               (olcc[back], olv[back]))
    got = _oracle_cache[name]
    assert np.array_equal(got[0], v) and np.array_equal(got[1], e)
    return got[2:]


def check(csr, name, first=True, order="pwl"):
    """PageRank and WCC for every id of [-2, n + 4), LCC for the shape's rows, as bit patterns against the oracle on the
    downloaded CSR; on a CSR's first calls also the iteration and round counts in the stats."""
    n, src, dst = shape(name)
    v, e, _ = csr.download()
    rv, rrows, re_ = ref_csr(n, src, dst)
    assert np.array_equal(v, rv) and np.array_equal(e, re_)
    (opr, oprv, oit), (owcc, owv), (olcc, olv) = oracle_answers(name, v, e)
    ids = np.arange(-2, n + 4, dtype=np.int64)
    got = {}
    for what in order:
        if what == "p":
            pr, prv, it, st = csr.pagerank(ids)
            assert it == oit and prv.tolist() == [0, 0] + [1] * (n + 2) + [0, 0]
            assert np.array_equal(prv, oprv) and np.array_equal(bits(pr[prv == 1]), bits(opr[oprv == 1]))
            if first:
                assert st["levels"] == oit and st["kernel_launches"] > 0
                _, _, it2, st2 = csr.pagerank(ids[:5])
                assert it2 == oit and st2["levels"] == 0 and st2["kernel_launches"] == 0
            got["p"] = bits(pr).tobytes()
        elif what == "w":
            wcc, wv, st = csr.weakly_connected_component(ids)
            assert np.array_equal(wv, owv) and np.array_equal(wcc[wv == 1], owcc[owv == 1])
            if first:
                assert st["levels"] == boruvka_rounds(name)
                _, _, st2 = csr.weakly_connected_component(ids[:5])
                assert st2["levels"] == 0 and st2["kernel_launches"] == 0
            got["w"] = wcc.tobytes()
        else:
            q = lcc_queries(name)
            lcc, lv, _ = csr.local_clustering_coefficient(q)
            assert np.array_equal(lv, olv) and np.array_equal(bits(lcc), bits(olcc))
            got["l"] = bits(lcc).tobytes()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_against_oracle(gpu_ctx, name):
    n, src, dst = shape(name)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    try:
        check(csr, name)
    finally:
        csr.free()


ROUTED = ["dangling128", "dangling129", "dangling385", "indeg", "n33", "n1025", "n32769", "self_loop1",
          "matching", "path_bitrev", "tree_reversed_edges", "tree_permuted_rows", "compact33", "compact257", "lcc_k",
          "lcc_words33", "lcc_big_count"]


@pytest.fixture(scope="module")
def replica_ctx():
    ctx = pgq.Context(0)
    yield ctx
    ctx.close()


def build_route(ctx, route, n, src, dst):
    """The same CSR through another construction route: other buffers, other recycled workspaces."""
    m = len(src)
    if route == "eid":  # edge rowids in another order than the rows: they travel along, the positions stay
        return pgq.DeviceCSR.build(ctx, n, src, dst, np.random.default_rng(m).permutation(m) * 3 + 5)
    if route == "upload":
        v, _, e = ref_csr(n, src, dst)
        return pgq.DeviceCSR.upload(ctx, n, v, e)
    if route == "keys":  # vertex row i carries key keys[i]
        keys = np.random.default_rng(n).permutation(n).astype(np.int64) * 1000003 - 10**9
        return pgq.DeviceCSR.build_from_keys(ctx, keys, keys[src], keys[dst])
    csr = pgq.DeviceCSR.create(ctx, n)  # chunked
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    for o in range(0, m, 4097):
        csr.add_edges(m, m, src[o:o + 4097], dst[o:o + 4097], np.arange(o, min(o + 4097, m)))
    csr.finalize()
    return csr


@pytest.mark.gpu
@pytest.mark.parametrize("route", ["eid", "upload", "chunked", "keys", "clone"])
@pytest.mark.parametrize("name", ROUTED)
def test_routes_against_oracle(gpu_ctx, replica_ctx, name, route):
    n, src, dst = shape(name)
    if route == "clone":
        prim = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
        try:
            csr = prim.clone(replica_ctx)
        finally:
            prim.free()
    else:
        csr = build_route(gpu_ctx, route, n, src, dst)
    try:
        check(csr, name, order="lwp" if route in ("upload", "keys") else "pwl")
    finally:
        csr.free()


def lcc_rows_against_oracle(csr, n, q, qv=None):
    """One call with these rows, every row compared with the oracle's answer for its vertex."""
    v, e, _ = csr.download()
    q = np.asarray(q, dtype=np.int64)
    live = np.ones(len(q), bool) if qv is None else np.asarray(qv) == 1
    uq, back = np.unique(q[live], return_inverse=True)
    olcc, _ = orc.local_clustering_coefficient(n, v, e, uq)
    lcc, lv, st = csr.local_clustering_coefficient(q, qv)
    assert np.array_equal(lv, live.astype(np.uint8))
    assert np.array_equal(bits(lcc[live]), bits(olcc[back])) and not np.any(bits(lcc[~live]))
    return st


@pytest.mark.gpu
def test_lcc_many_rows_per_block(gpu_ctx):
    """Far more rows than k_lcc_rows has blocks (sm_count * 16), of every k in LCC_K shuffled with short rows, rows of
    k < 2, NULL rows and the rows of the bitmap path: a block sorts one list after another in the same shared memory,
    and the queue of long rows fills from many blocks."""
    n, src, dst = shape("lcc_k")
    od = np.bincount(src, minlength=n)
    rng = np.random.default_rng(3)
    heads = np.flatnonzero(od >= 31)
    q = np.concatenate([rng.integers(0, n, 20000), np.tile(heads, 60)])
    q = q[rng.permutation(len(q))]
    qv = (rng.random(len(q)) > 0.15).astype(np.uint8)
    assert len(q) > 8 * H100_SMS * 16 and np.count_nonzero(od[q[qv == 1]] > LCC_SMEM) >= 30
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    try:
        lcc_rows_against_oracle(csr, n, q, qv)
        lcc_rows_against_oracle(csr, n, q[::-1].copy())
    finally:
        csr.free()


@pytest.mark.gpu
@pytest.mark.parametrize("name,times", [("lcc_words33", 1), ("lcc_words33", 2), ("lcc_words33", 70000), ("indeg", 70000)])
def test_lcc_big_rows_many_times(gpu_ctx, name, times):
    """The same row of the bitmap path 1, 2 and 70 000 times in one call, with short rows between them: above 65 535
    rows (the grid's y limit) the long rows take two groups, and the second group's bitmaps are the first's with the
    marked words cleared.  On `indeg` the rows go round six sources whose 10^4-long lists differ, so a bitmap of the
    second group that kept a bit of the first counts too much."""
    n, src, dst = shape(name)
    od = np.bincount(src, minlength=n)
    big = np.flatnonzero(od > LCC_SMEM)
    assert len(big) == (1 if name == "lcc_words33" else 6)
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    try:
        q = big[np.arange(times) % len(big)]
        if times > 2:
            q[1::1000] = np.flatnonzero((od >= 2) & (od <= LCC_SMEM))[0]
        st = lcc_rows_against_oracle(csr, n, q)
        groups = -(-int(np.count_nonzero(od[q] > LCC_SMEM)) // 65535)
        assert groups == (2 if times > 2 else 1) and st["kernel_launches"] == 1 + 3 * groups + 1
    finally:
        csr.free()


@pytest.mark.gpu
def test_lcc_big_small_null_interleaved(gpu_ctx):
    """Rows of the bitmap path (six sources of out-degree 10^4), short rows and NULL rows in turn."""
    n, src, dst = shape("indeg")
    od = np.bincount(src, minlength=n)
    big = np.flatnonzero(od > LCC_SMEM)
    small = np.flatnonzero((od >= 2) & (od <= 40))[:200]
    q = np.zeros(3 * 200, dtype=np.int64)
    q[0::3], q[1::3], q[2::3] = np.resize(big, 200), small, -77
    qv = np.ones(len(q), np.uint8)
    qv[2::3] = 0
    csr = pgq.DeviceCSR.build(gpu_ctx, n, src, dst)
    try:
        lcc_rows_against_oracle(csr, n, q, qv)
    finally:
        csr.free()


@pytest.mark.gpu
def test_call_order_on_one_dirty_workspace(monkeypatch):
    """The three computations share the scratch slots of a workspace.  In a context limited to one workspace, one CSR
    answers LCC, WCC, PageRank in that order and a second CSR of the same edges PageRank, WCC, LCC: every array of
    the later computations is what the earlier ones left behind.  The answers are the same bytes."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    try:
        for name in ("indeg", "lcc_k"):
            n, src, dst = shape(name)
            got = []
            for order in ("lwp", "pwl"):
                csr = pgq.DeviceCSR.build(ctx, n, src, dst)
                try:
                    got.append(check(csr, name, order=order))
                finally:
                    csr.free()
            assert got[0] == got[1]
    finally:
        ctx.close()
