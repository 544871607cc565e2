"""The CSR builds from vertex-key and edge-key columns at the boundaries of their sorts, joins and de-duplication.

pgq_csr_build_keys[_device] (directed) and pgq_csr_build_keys_undirected[_device] (csrc/pgq_csr.cu, key_bits to
build_from_key_columns) sort the vertex keys with a 64-bit LSD radix sort, find every edge's ranges of matching
vertex rows with key_range (a binary search, then a gallop and a bisection), and the undirected build packs the
(p, q) rows into 2b+1-bit keys, sorts and de-duplicates them and counts the unmatched and NULL ends with a second
sort.  So:

- a catalogue of deterministic key tables, each naming the boundaries it hits for the directed build ("d:..."), the
  undirected build ("u:...") or both.  A CPU-only numpy restatement of the device's intermediate quantities (sorted
  keys, nv, ms / md, b and the pass counts, t, h, r, tiles and scan levels, gallop runs) asserts that every named
  boundary really is hit, and that every boundary in REQUIRED is named by some entry;
- on the CPU, the oracle (oracle/pgq_oracle_keys[_undirected]) against two independent numpy restatements on every
  small entry: this pins the oracle at exactly the inputs the GPU tests use;
- on the GPU, every entry through host columns and device columns, byte for byte against the oracle (or the same
  ConstraintException), with the consumers of the small ones compared to the oracle's restatements;
- the range edges (exactly 2^31 - 1 directed join rows, exactly 2^31 undirected rows before de-duplication), builds
  on one workspace with dirty buffers, eight threads building at once, and device columns still being written on a
  side stream when the call starts.

Grid-stride boundaries assume an H100 SXM's 132 SMs: the edge kernels' grid is capped at 132 * 16 blocks of 256
threads and k_ukey_check's at 132 * 8."""
import threading
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from types import SimpleNamespace

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys as orck
from oracle import pgq_oracle_keys_undirected as orcu
from test_csr_layout_shapes import check_analytics
from test_oracle_keys_undirected_golden import numpy_restatement as numpy_undirected

I64_MIN, I64_MAX = int(np.iinfo(np.int64).min), int(np.iinfo(np.int64).max)
SCAN_TILE = 2048            # items per block of the exclusive scan
RS_TILE = 2048              # pairs per tile of the radix sort
RS_BITS = 5                 # bits per radix-sort pass
RS_BINS = 32
H100_SMS = 132
EDGE_GRID = H100_SMS * 16 * 256   # threads of k_key_edges / k_ukey_edges / k_ukey_half / k_ukey_expand
CHECK_GRID = H100_SMS * 8 * 256   # threads of k_ukey_check
ROW_LIMIT = 2**31 - 1       # join rows (directed) or rows before de-duplication (undirected) refused from here on
SMALL = 5000                # entries with fewer edge rows are checked against numpy; fewer vertices, consumers too
FRESH = 10**15              # unmatched values used to balance the undirected ends start here

RUNS = [2, 1, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 6]  # first at 0, last ends at nv
N_LIST = [1, 2, 3, 4, 5, 8, 9, 32, 33, 64, 65, 128, 129, 1024, 1025, 2047, 2048, 2049]


# ---- tables -------------------------------------------------------------------------------------------------------------
@dataclass
class Table:
    vkey: np.ndarray
    src: np.ndarray
    dst: np.ndarray
    vvalid: np.ndarray = None
    svalid: np.ndarray = None
    dvalid: np.ndarray = None

    @property
    def n(self):
        return len(self.vkey)

    @property
    def m(self):
        return len(self.src)

    def args(self):
        return self.vkey, self.src, self.dst, self.vvalid, self.svalid, self.dvalid


def table(vkey, src, dst, vvalid=None, svalid=None, dvalid=None):
    i64 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1))
    u8 = lambda a: None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.uint8).reshape(-1))
    return Table(i64(vkey), i64(src), i64(dst), u8(vvalid), u8(svalid), u8(dvalid))


def _valid(a, k):
    return np.ones(k, bool) if a is None else a.astype(bool)


def u64(x):
    return np.asarray(x, dtype=np.int64).view(np.uint64)


def i64(x):
    return np.asarray(x, dtype=np.uint64).view(np.int64)


def key_ends(tb):
    """valid key -> (rows holding it, distinct matched neighbour keys, distinct unmatched or NULL other ends), as the
    undirected CTE counts them: every row of a key has the same neighbours."""
    vv, sv, dv = _valid(tb.vvalid, tb.n), _valid(tb.svalid, tb.m), _valid(tb.dvalid, tb.m)
    cnt = defaultdict(int)
    for x in tb.vkey[vv].tolist():
        cnt[x] += 1
    nbr, ends = defaultdict(set), defaultdict(set)
    for s, d, a, c in zip(tb.src.tolist(), tb.dst.tolist(), sv.tolist(), dv.tolist()):
        so, do = a and s in cnt, c and d in cnt
        for x, xo, y, yo, yv in ((s, so, d, do, c), (d, do, s, so, a)):
            if xo:
                if yo:
                    nbr[x].add(y)
                else:
                    ends[x].add(y if yv else None)
    return cnt, nbr, ends


def balance(tb, null_first=False, extra_end_on=None):
    """Adds ends (x, fresh unmatched value) until every key's R - M (the extra rows its duplicated neighbour keys
    give) equals its number of distinct unmatched or NULL ends, so that the undirected build accepts the table; the
    first end of a key is a NULL one when null_first.  extra_end_on: a key that gets one end too many (refused)."""
    cnt, nbr, ends = key_ends(tb)
    src, dst, sv, dv = [tb.src], [tb.dst], [_valid(tb.svalid, tb.m)], [_valid(tb.dvalid, tb.m)]
    fresh = FRESH + 1000 * (tb.n + tb.m)
    for x in sorted(cnt):
        deficit = sum(cnt[y] - 1 for y in nbr[x]) - len(ends[x])
        assert deficit >= 0, (x, deficit)
        if extra_end_on is not None and x == extra_end_on:
            deficit += 1
        for j in range(deficit):
            null = null_first and j == 0 and None not in ends[x]
            fwd = (fresh + j) % 2 == 0
            src.append([x if fwd else fresh + j])
            dst.append([fresh + j if fwd else x])
            sv.append([True if fwd else not null])
            dv.append([not null if fwd else True])
        fresh += deficit + 1
    return table(tb.vkey, np.concatenate(src), np.concatenate(dst), tb.vvalid, np.concatenate(sv), np.concatenate(dv))


def bits_keys(seed, ones=False):
    """Keys that differ from another key only in bit 63 (key_bits flips it), only in bits 60-63 (the last radix pass
    reads bits 60-63 alone) and only in the two bits on either side of a 5-bit digit boundary.  Every key unique:
    the edges are a permutation of sources onto a permutation of destinations plus random ones."""
    rng = np.random.default_rng(seed)
    out = set()
    for x in u64([0, 5, -1, 123456789, 1 << 40, -(1 << 50) + 7]).tolist():
        out.add(x)
        out.add(x ^ (1 << 63))
        for k in (1, 2, 3, 7, 9, 15):
            out.add(x ^ (k << 60))
        for j in range(1, 13):
            out.add(x ^ (3 << (5 * j - 1)))
    keys = rng.permutation(i64(np.array(sorted(out), dtype=np.uint64)))
    n = len(keys)
    src = np.concatenate([rng.permutation(keys), rng.choice(keys, 2 * n)])
    dst = np.concatenate([rng.permutation(keys), rng.choice(keys, 2 * n)])
    if ones:
        return table(keys, src, dst, np.ones(n), np.ones(len(src)), np.ones(len(src)))
    return table(keys, src, dst)


def i64max_nulls(undirected):
    """A valid INT64_MAX run of three rows with NULL rows behind it in the sorted order (stored values INT64_MAX, 7, a
    live key, and -1): the NULL rows' sort key ~0 equals INT64_MAX's, only stability and nv keep them apart."""
    vkey = [7, I64_MAX, 3, I64_MAX, I64_MAX, 9, I64_MAX, 7, I64_MAX, -1, 11]
    vvalid = [1, 1, 1, 0, 1, 1, 0, 0, 1, 0, 1]
    src = [I64_MAX, I64_MAX, 3, 9, 7, -1, I64_MAX, 11, 5]
    dst = [7, 3, 9, 7, 3, 11, 11, 9, 3]
    tb = table(vkey, src, dst, vvalid)
    if undirected:  # -1 (a NULL row's value) as an unmatched end of 3
        tb = balance(table(vkey, src + [3, -1], dst + [-1, 7], vvalid))
    return tb


def i64max_dst_refused():
    """An edge into the three-row INT64_MAX key from a matched source: md = 3, refused."""
    return table([7, I64_MAX, I64_MAX, 0, I64_MAX], [7, 0], [0, I64_MAX], [1, 1, 1, 0, 1])


def runs_table(undirected, nulls):
    """Vertex keys in runs of RUNS rows (ids shuffled): the first run at sorted position 0, the last ending at nv,
    with NULL rows behind it when `nulls`.  Run i is the source of edges to a one-row key; edges from absent keys
    below the minimum, above the maximum and in the gaps look up nothing."""
    rng = np.random.default_rng(70 + nulls)
    run_keys = -5000 + 1000 * np.arange(len(RUNS))
    targets = run_keys[:-1] + 500
    vkey = np.concatenate([np.repeat(run_keys, RUNS), targets])
    vvalid = np.ones(len(vkey), np.uint8)
    if nulls:
        vkey = np.concatenate([vkey, [run_keys[-1], I64_MAX, run_keys[0], 0]])
        vvalid = np.concatenate([vvalid, [0, 0, 0, 0]])
    p = rng.permutation(len(vkey))
    vkey, vvalid = vkey[p], vvalid[p]
    src = list(run_keys[:-1]) + [run_keys[-1]] + list(run_keys[3:9])
    dst = list(targets) + [targets[0]] + list(targets[3:9])
    absent = [-10**12, run_keys[0] - 1, 10**12, run_keys[-1] + 1, run_keys[4] + 1, targets[6] + 1, I64_MIN, I64_MAX]
    src += absent
    dst += [targets[19]] * len(absent)
    tb = table(vkey, src, dst, vvalid)
    return balance(tb) if undirected else tb


def all_null_vertices():
    """n > 0, every vertex key NULL (nv = 0): nothing matches, not even the NULL rows' stored values."""
    vkey = [1, 2, 3, I64_MAX, 0, -1]
    return table(vkey, [1, 2, 3, I64_MAX, 0, -1, 5, 2], [2, 3, I64_MAX, 0, -1, 1, 5, 2], np.zeros(6),
                 [1, 1, 1, 1, 1, 1, 0, 1], [1, 1, 1, 1, 1, 1, 1, 0])


def packing(n, balanced):
    """n rows: 0 .. n-3 with unique keys (shuffled against the rowids) joined in a ring-like pattern, rows n-2 and
    n-1 sharing one key D with a self-loop and an edge from row n-3's key, which makes the flag bit 1.  Balanced by
    unmatched ends (accepted) or one end too many (refused).  Where the p field has a top bit (rows 2^(b-1) + 3 and
    3), the edges (hi, q), (lo, q), (q, hi) put (hi, q) twice with (lo, q) between them in a sort that drops the top
    bit of p."""
    rng = np.random.default_rng(100 + n)
    b = b_bits(n)
    if n == 1:
        tb = table([42], [42], [42])
        return balance(tb, extra_end_on=None if balanced else 42)
    u = n - 2
    keys = np.concatenate([rng.permutation(u) * 5 - 2 * n, [5 * n + 2, 5 * n + 2]])
    src, dst = [], []
    for i in range(u):
        src.append(keys[i])
        dst.append(keys[(7 * i + 3) % u])
    hi, lo, q = (1 << (b - 1)) + 3, 3, 5
    if hi < u:
        src += [keys[hi], keys[lo], keys[q]]
        dst += [keys[q], keys[q], keys[hi]]
    dk = keys[-1]
    src.append(dk)
    dst.append(dk)
    if u:
        src.append(keys[u - 1])
        dst.append(dk)
    return balance(table(keys, src, dst), extra_end_on=None if balanced else dk)


def half_mix(n, balanced=True):
    """Half edges and NULL ends: one unmatched value reached from both directions of one key and from several keys
    (keys at sorted positions p and p + 2^(b-1), each pair twice); unmatched INT64_MIN and INT64_MAX; an unmatched
    value equal to a NULL row's stored value; a NULL end and half edges on one key; duplicated keys T (4 rows) and
    D (2 rows) balanced by those ends."""
    b = b_bits(n)
    vkey = 10 * np.arange(n, dtype=np.int64)
    vvalid = np.ones(n, np.uint8)
    vkey[5], vvalid[5] = 7777, 0
    vkey[n - 4:] = vkey[n - 4]          # T: rows n-4 .. n-1
    vkey[n - 7:n - 5] = vkey[n - 7]     # D: rows n-7, n-6
    T, D = int(vkey[n - 4]), int(vkey[n - 7])
    A, B = 20, 10 * (3 + (1 << (b - 1)))   # sorted positions 2 and 2 + 2^(b-1) (row 5 is NULL)
    C, E, F = 30, 40, 60
    X = 123457
    src = [A, B, X, X, A, B, X, B, C, I64_MAX, E, F, F, A, B, C, F, E, D]
    dst = [X, X, A, B, X, X, B, X, I64_MIN, C, 7777, 0, 99991, T, T, T, T, D, 80]
    sv = np.ones(len(src), np.uint8)
    dv = np.ones(len(src), np.uint8)
    dv[11] = 0  # F -> NULL
    ring = [10 * i for i in range(n - 7) if i != 5]
    src += ring
    dst += ring[1:] + ring[:1]
    sv = np.concatenate([sv, np.ones(len(ring), np.uint8)])
    dv = np.concatenate([dv, np.ones(len(ring), np.uint8)])
    return balance(table(vkey, src, dst, vvalid, sv, dv), extra_end_on=None if balanced else D)


def sized_directed(n, m, seed):
    """n unique keys (shuffled, signed), m edges between random ones: every join has md = 1."""
    rng = np.random.default_rng(seed)
    keys = rng.permutation(n).astype(np.int64) * 7 - 3 * n
    return table(keys, rng.choice(keys, m), rng.choice(keys, m))


def sized_undirected(n, m, seed):
    """n unique keys, m edges between random ones: t = 2m, no half edges."""
    return sized_directed(n, m, seed)


def half_count(h, seed):
    """Exactly h half edges over about h / 4 keys y (each with up to four copies of one unmatched value, in both
    directions) and a two-row key that balances every y."""
    rng = np.random.default_rng(seed)
    ny = (h + 3) // 4
    ys = rng.permutation(ny).astype(np.int64) * 3 + 1
    dk = -7
    vkey = rng.permutation(np.concatenate([ys, [dk, dk]]))
    copies = np.full(ny, 4)
    copies[: 4 * ny - h] -= 1
    owner = np.repeat(ys, copies)
    val = FRESH + np.repeat(np.arange(ny), copies)
    fwd = np.arange(len(owner)) % 2 == 0
    src = np.concatenate([ys, np.where(fwd, owner, val)])
    dst = np.concatenate([np.full(ny, dk), np.where(fwd, val, owner)])
    order = rng.permutation(len(src))
    return table(vkey, src[order], dst[order])


def big_directed():
    """About 4.2 M edges: the scan of m + 1 elements takes a third level, the edge kernels loop past their grid."""
    return sized_directed(300_000, 2048 * 2048, 4)


def big_undirected():
    """t = 2048^2 rows before de-duplication (t + 1 needs a third scan level), 300 000 vertex rows (k_ukey_check loops
    past its grid)."""
    return sized_undirected(300_000, 2048 * 2048 // 2, 5)


# name -> (maker, {build: boundaries it is meant to hit})
CATALOGUE = {
    "bits": (lambda: bits_keys(1), {"d": {"bit63", "bits60_63", "digit_boundary", "accepted", "valid_none"},
                                    "u": {"bit63", "bits60_63", "digit_boundary", "accepted", "valid_none"}}),
    "bits_ones": (lambda: bits_keys(1, ones=True), {"d": {"valid_ones", "accepted"}, "u": {"valid_ones"}}),
    "i64max_nulls_d": (lambda: i64max_nulls(False), {"d": {"i64max_null_rows", "null_row_holds_live_key",
                                                           "run_3", "accepted", "run_ends_at_nv_before_nulls"}}),
    "i64max_nulls_u": (lambda: i64max_nulls(True), {"u": {"i64max_null_rows", "null_row_holds_live_key", "run_3",
                                                          "flag_accepted", "half_value_is_null_row_value",
                                                          "run_ends_at_nv_before_nulls"}}),
    "i64max_dst_refused": (i64max_dst_refused, {"d": {"i64max_null_rows", "refused"}}),
    "runs_d": (lambda: runs_table(False, False), {"d": {*(f"run_{k}" for k in RUNS), "run_at_0", "run_ends_at_nv",
                                                        "absent_below", "absent_above", "absent_gap"}}),
    "runs_nulls_d": (lambda: runs_table(False, True), {"d": {"run_at_0", "run_ends_at_nv_before_nulls", "run_129"}}),
    "runs_u": (lambda: runs_table(True, False), {"u": {*(f"run_{k}" for k in RUNS), "run_at_0", "run_ends_at_nv",
                                                       "absent_below", "absent_above", "absent_gap", "accepted"}}),
    "runs_nulls_u": (lambda: runs_table(True, True), {"u": {"run_at_0", "run_ends_at_nv_before_nulls", "accepted"}}),
    "all_null": (all_null_vertices, {"d": {"all_null_vertices"}, "u": {"all_null_vertices"}}),
    "n0": (lambda: table([], [1, 2], [2, 1]), {"d": {"n0"}, "u": {"n0"}}),
    "m0": (lambda: table([3, 1, 2], [], []), {"d": {"m0"}, "u": {"m0"}}),
    **{f"pack{n}": (lambda n=n: packing(n, True), {"u": {f"n_{n}", "accepted"}}) for n in N_LIST},
    **{f"pack{n}_refused": (lambda n=n: packing(n, False),
                            {"u": {f"n_{n}", "dup_unbalanced_refused" if n > 1 else "refused"}}) for n in N_LIST},
    "half_mix64": (lambda: half_mix(64), {"u": {"half_both_directions", "half_several_keys", "half_i64min",
                                                "half_i64max", "half_value_is_null_row_value",
                                                "null_end_and_half_same_key", "half_dups_alias", "flag_accepted",
                                                "half_passes_b6"}}),
    "half_mix64_refused": (lambda: half_mix(64, False), {"u": {"dup_unbalanced_refused", "half_dups_alias"}}),
    "half_mix2048": (lambda: half_mix(2048), {"u": {"half_dups_alias", "half_passes_b11", "flag_accepted",
                                                    "scan_n1_2049", "rs_n_2048"}}),
    "d_n2047": (lambda: sized_directed(2047, 2047, 11), {"d": {"scan_n1_2048", "scan_m1_2048"}}),
    "d_n2048": (lambda: sized_directed(2048, 2048, 12), {"d": {"scan_n1_2049", "scan_m1_2049", "rs_n_2048"}}),
    "d_n2049": (lambda: sized_directed(2049, 3000, 13), {"d": {"rs_n_2049"}}),
    "d_n131072": (lambda: sized_directed(131072, 131072, 14), {"d": {"rs_n_131072"}}),
    "d_n131073": (lambda: sized_directed(131073, 131073, 15), {"d": {"rs_n_131073"}}),
    "u_t2046": (lambda: sized_undirected(700, 1023, 21), {"u": {"scan_t1_2047"}}),
    "u_t2048": (lambda: sized_undirected(2047, 1024, 22), {"u": {"rs_t_2048", "scan_t1_2049", "scan_n1_2048", "h_0"}}),
    "u_t2050": (lambda: sized_undirected(2048, 1025, 23), {"u": {"rs_t_2050", "scan_n1_2049", "rs_n_2048"}}),
    "u_m2047": (lambda: sized_undirected(2049, 2047, 24), {"u": {"scan_m1_2048", "rs_n_2049"}}),
    "u_m2048": (lambda: sized_undirected(1500, 2048, 25), {"u": {"scan_m1_2049"}}),
    "u_t131072": (lambda: sized_undirected(131072, 65536, 26), {"u": {"rs_t_131072", "rs_n_131072"}}),
    "u_t131074": (lambda: sized_undirected(131073, 65537, 27), {"u": {"rs_t_131074", "rs_n_131073"}}),
    "u_h2047": (lambda: half_count(2047, 31), {"u": {"h_2047", "accepted"}}),
    "u_h2048": (lambda: half_count(2048, 32), {"u": {"h_2048", "accepted"}}),
    "u_h2049": (lambda: half_count(2049, 33), {"u": {"h_2049", "accepted"}}),
    "u_h131073": (lambda: half_count(131073, 34), {"u": {"h_131073", "accepted"}}),
    "d_big": (big_directed, {"d": {"scan_m1_level3", "grid_edges_strided"}}),
    "u_big": (big_undirected, {"u": {"scan_t1_level3", "grid_edges_strided", "grid_check_strided"}}),
}
CATALOGUE["pack2"][1]["u"].add("h_1")
for _n, _b, _p in ((1, 1, 1), (3, 2, 1), (5, 3, 2), (9, 4, 2), (32, 5, 3), (33, 6, 3), (65, 7, 3), (129, 8, 4),
                   (1024, 10, 5), (1025, 11, 5), (2049, 12, 5)):
    CATALOGUE[f"pack{_n}"][1]["u"] |= {f"b_{_b}", f"row_passes_{_p}"}
for _n in (2, 4, 8, 32, 64, 128, 1024, 2048):
    CATALOGUE[f"pack{_n}"][1]["u"].add("row_last_fills_field")
for _n, _b in ((32, 5), (33, 6), (1024, 10), (1025, 11)):
    CATALOGUE[f"pack{_n}"][1]["u"] |= {f"half_passes_b{_b}", "flag_accepted"}
CATALOGUE["pack32"][1]["u"].add("p_high_b5")
CATALOGUE["pack1024"][1]["u"].add("p_high_b10")
CATALOGUE["pack2047"][1]["u"] |= {"scan_n1_2048", "rs_n_2047"}

_BOTH = ({"bit63", "bits60_63", "digit_boundary", "i64max_null_rows", "null_row_holds_live_key", "run_at_0",
          "run_ends_at_nv", "run_ends_at_nv_before_nulls", "absent_below", "absent_above", "absent_gap",
          "all_null_vertices", "scan_n1_2048", "scan_n1_2049", "scan_m1_2048", "scan_m1_2049", "rs_n_2048", "rs_n_2049",
          "rs_n_131072", "rs_n_131073", "grid_edges_strided", "m0", "n0", "valid_ones", "valid_none", "accepted"}
         | {f"run_{k}" for k in RUNS})
REQUIRED = ({f"d:{x}" for x in _BOTH | {"refused", "scan_m1_level3"}}
            | {f"u:{x}" for x in _BOTH | {f"n_{n}" for n in N_LIST}
               | {f"b_{b}" for b in (1, 2, 3, 4, 5, 6, 7, 8, 10, 11, 12)} | {f"row_passes_{p}" for p in range(1, 6)}
               | {f"half_passes_b{b}" for b in (5, 6, 10, 11)}
               | {"row_last_fills_field", "flag_accepted", "dup_unbalanced_refused", "p_high_b5", "p_high_b10",
                  "h_0", "h_1", "h_2047", "h_2048", "h_2049", "h_131073", "half_both_directions",
                  "half_several_keys", "half_i64min", "half_i64max", "half_value_is_null_row_value",
                  "null_end_and_half_same_key", "half_dups_alias", "scan_t1_2047", "scan_t1_2049", "scan_t1_level3",
                  "rs_t_2048", "rs_t_2050", "rs_t_131072", "rs_t_131074", "grid_check_strided"}})

_tables = {}


def entry(name):
    if name not in _tables:
        _tables[name] = CATALOGUE[name][0]()
    return _tables[name]


def kinds(name):
    return sorted(CATALOGUE[name][1])


# ---- the device's intermediate quantities, in numpy ---------------------------------------------------------------------
def b_bits(n):
    b = 1
    while b < 31 and (1 << b) < n:
        b += 1
    return b


def scan_levels(count):
    """levels of pgq_scan_exclusive_i32 over count elements (one block per level up to SCAN_TILE)"""
    if count <= 0:
        return 0
    lv = 1
    while count > SCAN_TILE:
        count = -(-count // SCAN_TILE)
        lv += 1
    return lv


def radix(count, end_bit):
    """(tiles, passes, scan levels of the digit histogram) of radix_sort_pairs"""
    tiles = -(-count // RS_TILE)
    return tiles, -(-end_bit // RS_BITS), scan_levels(RS_BINS * tiles)


def quantities(tb, kind):
    """What build_from_keys / build_from_keys_undirected compute on the way, from the columns alone."""
    n, m = tb.n, tb.m
    vv, sv, dv = _valid(tb.vvalid, n), _valid(tb.svalid, m), _valid(tb.dvalid, m)
    kb = u64(tb.vkey) ^ np.uint64(1 << 63)
    vrows = np.flatnonzero(vv)
    order = vrows[np.argsort(kb[vrows], kind="stable")]
    nv = len(order)
    sorted_key = kb[order]
    sorted_row = np.concatenate([order, np.flatnonzero(~vv)]).astype(np.int64)
    sk, dk = u64(tb.src) ^ np.uint64(1 << 63), u64(tb.dst) ^ np.uint64(1 << 63)
    slo, shi = np.searchsorted(sorted_key, sk, "left"), np.searchsorted(sorted_key, sk, "right")
    dlo, dhi = np.searchsorted(sorted_key, dk, "left"), np.searchsorted(sorted_key, dk, "right")
    ms = np.where(sv, shi - slo, 0).astype(np.int64)
    md = np.where(dv, dhi - dlo, 0).astype(np.int64)
    q = dict(n=n, m=m, nv=nv, sorted_key=sorted_key, sorted_row=sorted_row, ms=ms, md=md, stored_null=tb.vkey[~vv])
    # every key_range call: the source of every valid key, the destination where the build looks it up
    dlook = dv & (ms > 0) if kind == "d" else dv
    q["lookups"] = (np.concatenate([slo[sv], dlo[dlook]]), np.concatenate([shi[sv], dhi[dlook]]),
                    np.concatenate([sk[sv], dk[dlook]]))
    if kind == "d":
        q["refused"] = bool(np.any((ms > 0) & (md != 1)))
        q["rows"] = int(np.sum(ms * md))
        return q
    b = b_bits(n)
    t = 2 * int(np.sum(ms * md))
    half = (ms > 0) != (md > 0)
    other_valid = np.where(ms > 0, dv, sv)
    h_sel = half & other_valid
    h_lo = np.where(ms > 0, slo, dlo)[h_sel]
    h_val = np.where(ms > 0, dk, sk)[h_sel]
    q.update(b=b, t=t, h=int(h_sel.sum()), h_lo=h_lo, h_val=h_val, h_from_src=(ms == 0)[h_sel],
             null_lo=np.where(ms > 0, slo, dlo)[half & ~other_valid],
             row_radix=radix(t, 2 * b + 1), half_radix=radix(int(h_sel.sum()), b))
    # the expanded rows: edge k -> (a_i, c_j) with flag j != 0 and (c_j, a_i) with flag i != 0
    c = ms * md
    k = np.repeat(np.arange(m), c)
    w = np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)
    i, j = w // np.maximum(md[k], 1), w % np.maximum(md[k], 1)
    a, cc = sorted_row[slo[k] + i], sorted_row[dlo[k] + j]
    p = np.concatenate([a, cc])
    qq = np.concatenate([cc, a])
    flag = np.concatenate([j != 0, i != 0])
    pairs = np.unique(p * (1 << 32) + qq)
    up, uq = pairs >> 32, pairs & 0xFFFFFFFF
    q.update(p=p, flag=flag, r=len(pairs))
    # the check: per key, R - M (distinct rows minus distinct neighbour keys) against the distinct ends
    rank = np.full(n, -1, np.int64)
    if nv:
        first = np.concatenate([[True], sorted_key[1:] != sorted_key[:-1]])
        rank[order] = np.cumsum(first) - 1
        nkeys = int(first.sum())
        R = np.bincount(up, minlength=n)
        M = np.bincount(np.unique(up * (1 << 32) + rank[uq]) >> 32, minlength=n)
        krank = np.cumsum(first) - 1
        hk = krank[h_lo] if len(h_lo) else np.zeros(0, np.int64)
        hv = np.unique(np.stack([hk, h_val.astype(np.int64) if len(h_val) else hk]), axis=1)[0] \
            if len(hk) else np.zeros(0, np.int64)
        D = np.bincount(hv, minlength=nkeys)
        nk = np.unique(krank[q["null_lo"]]) if len(q["null_lo"]) else np.zeros(0, np.int64)
        D[nk] += 1
        q["refused"] = bool(np.any((R - M)[vv] != D[rank[vv]]))
    else:
        q["refused"] = False
    return q


def hits(tb, kind, q):
    """Every boundary the table hits in the given build, by name (without the "d:" / "u:" prefix)."""
    out = set()
    n, m, nv = q["n"], q["m"], q["nv"]
    keys = np.unique(q["sorted_key"][:nv] ^ np.uint64(1 << 63))
    if len(keys):
        def pair(mask):
            return bool(np.any(np.isin(keys ^ np.uint64(mask), keys)))
        if pair(1 << 63):
            out.add("bit63")
        if any(pair(k << 60) for k in range(1, 16) if k != 8):
            out.add("bits60_63")
        if any(pair(3 << (5 * j - 1)) for j in range(1, 13)):
            out.add("digit_boundary")
    live = set(i64(keys).tolist())
    if I64_MAX in live and nv < n:
        out.add("i64max_null_rows")
    if any(x in live for x in q["stored_null"].tolist()):
        out.add("null_row_holds_live_key")
    lo, hi, x = q["lookups"]
    found = hi > lo
    for ln in np.unique(hi[found] - lo[found]).tolist():
        out.add(f"run_{ln}")
    if np.any(found & (lo == 0)):
        out.add("run_at_0")
    if nv and np.any(found & (hi == nv)):
        out.add("run_ends_at_nv" if nv == n else "run_ends_at_nv_before_nulls")
    if nv:
        miss = x[~found]
        kmin, kmax = q["sorted_key"][0], q["sorted_key"][nv - 1]
        out |= {name for name, hit in (("absent_below", np.any(miss < kmin)), ("absent_above", np.any(miss > kmax)),
                                       ("absent_gap", np.any((miss > kmin) & (miss < kmax)))) if hit}
    elif n and m:
        out.add("all_null_vertices")
    for what, count in (("n1", n + 1), ("m1", m + 1)):
        if count in (SCAN_TILE, SCAN_TILE + 1):
            out.add(f"scan_{what}_{count}")
    if scan_levels(m + 1) == 3:
        out.add("scan_m1_level3")
    if n in (2047, 2048, 2049, 131072, 131073):
        out.add(f"rs_n_{n}")
    if m > EDGE_GRID:
        out.add("grid_edges_strided")
    if m == 0:
        out.add("m0")
    if n == 0:
        out.add("n0")
    given = [a for a in (tb.vvalid, tb.svalid, tb.dvalid) if a is not None]
    if not given:
        out.add("valid_none")
    elif len(given) == 3 and all(np.all(a == 1) for a in given):
        out.add("valid_ones")
    out.add("refused" if q["refused"] else "accepted")
    if kind == "d":
        return out
    b, t, h = q["b"], q["t"], q["h"]
    out |= {f"n_{n}", f"b_{b}", f"h_{h}"}
    if t + 1 in (2047, 2049):
        out.add(f"scan_t1_{t + 1}")
    if scan_levels(t + 1) == 3:
        out.add("scan_t1_level3")
    if t in (2048, 2050, 131072, 131074):
        out.add(f"rs_t_{t}")
    if nv > CHECK_GRID:
        out.add("grid_check_strided")
    if h:
        out.add(f"half_passes_b{b}")
        hl, hv = q["h_lo"].astype(np.int64), q["h_val"].view(np.int64)
        (pl, pv), pc = np.unique(np.stack([hl, hv]), axis=1, return_counts=True)  # distinct (key, value) pairs
        if np.any(np.unique(pv, return_counts=True)[1] > 1):
            out.add("half_several_keys")
        dirs = np.unique(np.stack([hl, hv, q["h_from_src"].astype(np.int64)]), axis=1)
        if np.any(np.unique(dirs[:2], axis=1, return_counts=True)[1] > 1):
            out.add("half_both_directions")
        # a duplicated (key, value) pair whose value another key reaches at a position equal below bit b-1
        low = np.unique(np.stack([pv, pl & ((1 << (b - 1)) - 1)]), axis=1, return_counts=True)
        aliased = low[0][0][low[1] > 1]
        if np.any(np.isin(pv[pc > 1], aliased)):
            out.add("half_dups_alias")
        vals = set(i64(q["h_val"] ^ np.uint64(1 << 63)).tolist())
        if I64_MIN in vals:
            out.add("half_i64min")
        if I64_MAX in vals:
            out.add("half_i64max")
        if vals & set(q["stored_null"].tolist()):
            out.add("half_value_is_null_row_value")
        if len(np.intersect1d(q["null_lo"], hl)):
            out.add("null_end_and_half_same_key")
    if not q["refused"] and t:
        out.add(f"row_passes_{q['row_radix'][1]}")
        if np.any(q["flag"]):
            out.add("flag_accepted")
        if n == 1 << b and np.any(q["p"] == n - 1):
            out.add("row_last_fills_field")
        if np.any(q["p"] >= 1 << (b - 1)):
            out.add(f"p_high_b{b}")
    if q["refused"] and nv and np.any(np.unique(q["sorted_key"][:nv], return_counts=True)[1] > 1):
        out.add("dup_unbalanced_refused")
    return out


# ---- CPU only: the catalogue hits what it names ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CATALOGUE))
def test_catalogue_hits_its_boundaries(name):
    tb = entry(name)
    for kind, want in CATALOGUE[name][1].items():
        q = quantities(tb, kind)
        got = hits(tb, kind, q)
        extra = "" if kind == "d" else (f" b={q['b']} t={q['t']} h={q['h']} r={q['r']} row_radix={q['row_radix']}"
                                        f" half_radix={q['half_radix']}")
        print(f"{name} [{kind}]: n={tb.n} m={tb.m} nv={q['nv']} refused={q['refused']} "
              f"scan(n+1, m+1)={scan_levels(tb.n + 1)},{scan_levels(tb.m + 1)}{extra}")
        assert want <= got, (kind, sorted(want - got))


def test_catalogue_covers_every_boundary():
    named = {f"{k}:{x}" for _, want in CATALOGUE.values() for k, xs in want.items() for x in xs}
    assert REQUIRED <= named, sorted(REQUIRED - named)


# ---- CPU only: the oracle against numpy on the small entries ------------------------------------------------------------
def numpy_directed(vkey, src, dst, vv=None, sv=None, dv=None):
    """(v, e, ids) or None for the ConstraintException: edge k joins every vertex row holding its source key to the
    one row holding its destination key (refused when an edge with a source has no or several), rows grouped by
    source row in edge rowid order, in the reference layout v[n + 2]."""
    vkey, src, dst = (np.asarray(a, dtype=np.int64) for a in (vkey, src, dst))
    n, m = len(vkey), len(src)
    vv, sv, dv = _valid(vv, n), _valid(sv, m), _valid(dv, m)
    rows = defaultdict(list)
    for i in np.flatnonzero(vv).tolist():
        rows[int(vkey[i])].append(i)
    a_all, c_all, k_all = [], [], []
    for k in range(m):
        a = rows.get(int(src[k]), []) if sv[k] else []
        if not a:
            continue
        c = rows.get(int(dst[k]), []) if dv[k] else []
        if len(c) != 1:
            return None
        a_all += a
        c_all += c * len(a)
        k_all += [k] * len(a)
    a_all, c_all, k_all = (np.asarray(x, dtype=np.int64) for x in (a_all, c_all, k_all))
    o = np.lexsort((k_all, a_all))
    v = np.zeros(n + 2, dtype=np.int64)
    v[1:n + 1] = np.cumsum(np.bincount(a_all, minlength=n)[:n])
    v[n + 1] = v[n]
    return v, c_all[o], k_all[o]


def oracle(tb, kind):
    """The oracle's (v, e, ids), or None for its ConstraintError."""
    try:
        return (orck.csr_build_keys if kind == "d" else orcu.csr_build_keys_undirected)(*_oracle_args(tb))
    except orc.ConstraintError:
        return None


def _oracle_args(tb):
    return tb.vkey, tb.src, tb.dst, tb.vvalid, tb.svalid, tb.dvalid


LARGE = {"d_n131072", "d_n131073", "u_t131072", "u_t131074", "u_h131073", "d_big", "u_big"}  # SMALL edge rows or more


@pytest.mark.parametrize("name,kind", [(nm, k) for nm in CATALOGUE if nm not in LARGE for k in kinds(nm)])
def test_oracle_equals_numpy(name, kind):
    tb = entry(name)
    assert tb.m < SMALL
    want = (numpy_directed if kind == "d" else numpy_undirected)(*_oracle_args(tb))
    got = oracle(tb, kind)
    assert (got is None) == (want is None)
    assert (got is None) == quantities(tb, kind)["refused"]
    if want is not None:
        for a, b in zip(got, want):
            assert np.array_equal(a, b)


def test_numpy_directed_on_random_tables():
    """The directed restatement against the oracle on small random tables with duplicated keys and NULLs."""
    rng = np.random.default_rng(45)
    accepted = refused = 0
    for _ in range(300):
        n, m = int(rng.integers(0, 14)), int(rng.integers(0, 30))
        pool = np.arange(-4, 12)
        vkey = rng.choice(pool, n) if rng.random() < 0.5 else rng.permutation(pool)[:n]
        src, dst = rng.choice(pool, m), rng.choice(pool, m)
        vv, sv, dv = ((rng.random(k) > 0.1).astype(np.uint8) for k in (n, m, m))
        want = numpy_directed(vkey, src, dst, vv, sv, dv)
        got = oracle(table(vkey, src, dst, vv, sv, dv), "d")
        assert (got is None) == (want is None)
        if want is None:
            refused += 1
            continue
        accepted += 1
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
    assert accepted > 20 and refused > 20


# ---- GPU: every entry, both routes, against the oracle -----------------------------------------------------------------
_oracle_cache = {}


def expected(name, kind):
    if (name, kind) not in _oracle_cache:
        _oracle_cache[(name, kind)] = oracle(entry(name), kind)
    return _oracle_cache[(name, kind)]


def device_columns(tb):
    """The columns as CUDA tensors (None for an absent validity column or an empty column)."""
    import torch
    return [None if a is None or len(a) == 0 else torch.from_numpy(np.ascontiguousarray(a)).cuda()
            for a in (tb.vkey, tb.src, tb.dst, tb.vvalid, tb.svalid, tb.dvalid)]


def build(ctx, tb, kind, route, cols=None):
    if route == "host":
        return pgq.DeviceCSR.build_from_keys(ctx, *tb.args(), undirected=kind == "u")
    cols = device_columns(tb) if cols is None else cols
    ptr = [0 if c is None else c.data_ptr() for c in cols]
    return pgq.DeviceCSR.build_from_keys_device(ctx, tb.n, tb.m, ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], ptr[5],
                                                undirected=kind == "u")


def same_bytes(got, ref):
    for a, b in zip(got, ref):
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.tobytes() == b.tobytes()


def check_build(ctx, tb, kind, route, ref, cols=None, keep=False):
    """The device build equals the oracle's arrays byte for byte, or raises its ConstraintException."""
    if ref is None:
        with pytest.raises(pgq.ConstraintException) as ex:
            build(ctx, tb, kind, route, cols)
        assert str(ex.value) == orc.CONSTRAINT_TEXT
        return None
    csr = build(ctx, tb, kind, route, cols)
    try:
        same_bytes(csr.download(), ref)
    except BaseException:
        csr.free()
        raise
    if keep:
        return csr
    csr.free()
    return None


def check_paths(csr, n, ref, seed):
    v, e, ids = ref
    rng = np.random.default_rng(seed)
    ps, pd = rng.integers(0, n, 300), rng.integers(0, n, 300)
    sv = np.ones(300, np.uint8)
    sv[::29] = 0
    out, valid, _ = csr.iterativelength(ps, pd, sv)
    exp, expv, _ = orc.iterativelength(n, v, e, ps, pd, sv)
    assert np.array_equal(valid, expv) and np.array_equal(out, exp)
    paths, _ = csr.shortestpath(ps[:100], pd[:100], sv[:100])
    assert paths == orc.shortestpath(n, v, e, ids, ps[:100], pd[:100], sv[:100])[0]


GPU_CASES = [(nm, k, r) for nm in CATALOGUE for k in kinds(nm) for r in ("host", "device")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,route", GPU_CASES)
def test_build_equals_oracle(gpu_ctx, name, kind, route):
    tb = entry(name)
    ref = expected(name, kind)
    csr = check_build(gpu_ctx, tb, kind, route, ref, keep=True)
    if csr is None:
        return
    try:
        if 0 < tb.n < SMALL:
            if kind == "d":
                check_paths(csr, tb.n, ref, tb.n + tb.m)
            else:
                check_analytics(csr, SimpleNamespace(n=tb.n, focus=[]), (ref[0], ref[1], ref[2], None))
    finally:
        csr.free()


# ---- GPU: the range edges -------------------------------------------------------------------------------------------------
# The accepted side of each edge, 2^31 - 2 rows, is not built here: the rows, their sort buffers and the CSR take more
# than the 80 GB of an H100.  Neither edge calls the oracle, which would materialise the rows.
@pytest.mark.gpu
def test_directed_refuses_exactly_2_31_minus_1_join_rows(gpu_ctx):
    """Key 0 held by 65 536 rows is the source of 32 767 edges, 65 535 one-row keys of one edge each, all into the
    one-row key 1: 65 536 * 32 767 + 65 535 = 2^31 - 1 rows."""
    singles = np.arange(2, 2 + 65535, dtype=np.int64)
    vkey = np.concatenate([np.zeros(65536, np.int64), [1], singles])
    src = np.concatenate([np.zeros(32767, np.int64), singles])
    assert 65536 * 32767 + len(singles) == ROW_LIMIT
    with pytest.raises(pgq.InvalidInputException) as ex:
        pgq.DeviceCSR.build_from_keys(gpu_ctx, vkey, src, np.ones(len(src), np.int64))
    assert str(ROW_LIMIT) in str(ex.value)


@pytest.mark.gpu
def test_undirected_refuses_exactly_2_31_rows_before_deduplication(gpu_ctx):
    """One edge between two keys of 32 768 rows each: 2 * 32 768^2 = 2^31 rows (each per-edge term is capped at 2^31,
    so the cap itself is reached); t is even, so 2^31 is the first refused value."""
    vkey = np.concatenate([np.zeros(32768, np.int64), np.ones(32768, np.int64)])
    with pytest.raises(pgq.InvalidInputException) as ex:
        pgq.DeviceCSR.build_from_keys(gpu_ctx, vkey, [0], [1], undirected=True)
    assert str(2**31) in str(ex.value)


# ---- GPU: one workspace, dirty buffers ------------------------------------------------------------------------------------
WS_N, WS_M = 512, 1400


def ws_table(seed, dup_rows, n_y, null_ends, balanced=True, directed=False):
    """WS_N vertex rows, WS_M edges (padded with edges whose both ends are NULL, which neither build sees): a key of
    dup_rows rows joined to n_y one-row keys (each balanced by unmatched ends, NULL ones first when null_ends), over
    a random graph of unique keys."""
    rng = np.random.default_rng(seed)
    uniq = rng.permutation(WS_N - dup_rows).astype(np.int64) * 3 - 500
    dk = 10**6 + seed
    vkey = rng.permutation(np.concatenate([uniq, np.full(dup_rows, dk)]))
    ys = uniq[:n_y]
    if directed:
        src = np.concatenate([np.full(n_y, dk), rng.choice(uniq, 300)])
        dst = np.concatenate([ys, rng.choice(uniq, 300)])
        if not balanced:
            dst[-1] = dk
        tb = table(vkey, src, dst)
    else:
        src = np.concatenate([ys, rng.choice(uniq, 300)])
        dst = np.concatenate([np.full(n_y, dk), rng.choice(uniq, 300)])
        tb = balance(table(vkey, src, dst), null_first=null_ends, extra_end_on=None if balanced else int(ys[0]))
    pad = WS_M - tb.m
    assert pad >= 0
    sv = np.concatenate([_valid(tb.svalid, tb.m), np.zeros(pad, bool)])
    dv = np.concatenate([_valid(tb.dvalid, tb.m), np.zeros(pad, bool)])
    return table(vkey, np.concatenate([tb.src, np.full(pad, dk)]), np.concatenate([tb.dst, np.full(pad, dk)]), None,
                 sv, dv)


WS_SEQUENCE = [  # (kind, table): the largest t and h first, then h = 0, NULL ends then none, refusals in between
    ("u", lambda: ws_table(1, 20, 50, True)),
    ("u", lambda: ws_table(2, 1, 0, False)),
    ("d", lambda: ws_table(3, 6, 80, False, directed=True)),
    ("u", lambda: ws_table(4, 8, 30, True, balanced=False)),
    ("d", lambda: ws_table(5, 1, 0, False, directed=True)),
    ("u", lambda: ws_table(6, 3, 40, False)),
    ("d", lambda: ws_table(7, 4, 10, False, balanced=False, directed=True)),
    ("u", lambda: ws_table(8, 1, 0, False)),
]


def test_workspace_sequence_is_what_it_says():
    qs = [quantities(make(), kind) for kind, make in WS_SEQUENCE]
    assert [q["refused"] for q in qs] == [False, False, False, True, False, False, True, False]
    u = [q for (kind, _), q in zip(WS_SEQUENCE, qs) if kind == "u"]
    assert u[0]["t"] == max(q["t"] for q in u) and u[0]["h"] == max(q["h"] for q in u)
    assert u[0]["h"] > 0 and u[1]["h"] == 0 and len(u[0]["null_lo"]) and not len(u[1]["null_lo"])


@pytest.mark.gpu
def test_dirty_buffers_one_workspace(monkeypatch):
    """A fresh context with one workspace: every build takes the key slots the one before left, with the same n and
    m but other contents.  After the sequence a search on a CSR built in the middle of it still equals the oracle."""
    monkeypatch.setenv("PGQ_B200_MAX_WORKSPACES", "1")
    ctx = pgq.Context(0)
    kept = None
    try:
        for i, (kind, make) in enumerate(WS_SEQUENCE):
            tb = make()
            ref = oracle(tb, kind)
            for route in ("host", "device"):
                csr = check_build(ctx, tb, kind, route, ref, keep=True)
                if csr is not None and i == 4 and route == "host":
                    kept, kept_ref = csr, ref
                elif csr is not None:
                    csr.free()
        check_paths(kept, WS_N, kept_ref, 9)
    finally:
        if kept is not None:
            kept.free()
        ctx.close()


# ---- GPU: eight threads on one context ----------------------------------------------------------------------------------
CONCURRENT = [("bits", "d", "host"), ("i64max_nulls_u", "u", "device"), ("runs_d", "d", "device"),
              ("half_mix64", "u", "host"), ("pack1025", "u", "device"), ("pack33_refused", "u", "host"),
              ("i64max_dst_refused", "d", "device"), ("runs_nulls_u", "u", "host")]


@pytest.mark.gpu
def test_eight_threads_one_context(gpu_ctx):
    jobs = [(entry(nm), k, r, expected(nm, k)) for nm, k, r in CONCURRENT]
    barrier = threading.Barrier(len(jobs))

    def run(job):
        tb, kind, route, ref = job
        cols = device_columns(tb) if route == "device" else None
        barrier.wait()
        for _ in range(3):
            check_build(gpu_ctx, tb, kind, route, ref, cols)
        return True

    with ThreadPoolExecutor(max_workers=len(jobs)) as pool:
        assert all(pool.map(run, jobs))


# ---- GPU: device columns still being written on a side stream -----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,kind", [("half_mix2048", "u"), ("d_n2049", "d")])
def test_device_columns_from_an_unsynchronised_stream(gpu_ctx, name, kind):
    """The columns are written by torch on a side stream behind a long-running kernel, and the call starts without
    synchronising it: the build must see the final columns and leave them as they were."""
    import torch
    tb = entry(name)
    ref = expected(name, kind)
    arrays = [a for a in (tb.vkey, tb.src, tb.dst, tb.vvalid, tb.svalid, tb.dvalid)]
    cols = [None if a is None else torch.full((len(a),), -1 if a.dtype == np.int64 else 0,
                                              dtype=torch.int64 if a.dtype == np.int64 else torch.uint8,
                                              device="cuda") for a in arrays]
    pinned = [None if a is None else torch.from_numpy(a).pin_memory() for a in arrays]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        for c, p in zip(cols, pinned):
            if c is not None:
                c.copy_(p, non_blocking=True)
    check_build(gpu_ctx, tb, kind, "device", ref, cols)
    side.synchronize()
    for c, a in zip(cols, arrays):
        if c is not None:
            assert np.array_equal(c.cpu().numpy(), a)
