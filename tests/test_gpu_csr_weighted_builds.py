"""The weighted device CSR through every construction route: the chunked create_csr_edge protocol, the one-shot builds
from host rows, device rows and a finished host CSR, the key builds from host and device columns, and a clone of each.

Every route of one graph gets the same edge rows in the same order within each source row (for the key routes, the
order they define: ascending edge rowid), so their CSRs, edge ids, weight columns and weight types must be equal bit
for bit, and so must what cheapest_path_length, cheapest_path, cheapest_path_count, all_cheapest_paths and
cheapest_k_paths answer on them -- a refusal included.  The key fixtures (tests/golden/refkw_*.npz) also pin the key
routes against the reference binary: its get_csr_w within each source row, and its cheapest_path_length."""
import ctypes as C
import os

import numpy as np
import pytest

from duckpgq_extension_b200 import pgq
from oracle import pgq_oracle as orc
from oracle import pgq_oracle_keys as ork

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEY_FIXTURES = sorted(f[6:-4] for f in os.listdir(GOLDEN) if f.startswith("refkw_") and f.endswith(".npz"))
CHUNKS = [2048, 1, 97, 4097]  # create_csr_edge chunks; 4096 rows fill one staging slot
ROUTES = ["chunked", "build", "build_device", "upload", "build_keys", "build_keys_device"]


@pytest.fixture(scope="module")
def other_ctx():
    ctx = pgq.Context(0)
    yield ctx
    ctx.close()


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype.kind == "f" else a.astype(np.int64)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def addr(t):
    return t.data_ptr() if t.numel() else 0


def weight_addr(w):
    """A device weight column's address; a one-element buffer stands in for an empty one (the pointer names the type)."""
    t = cuda(w if len(w) else np.zeros(1, dtype=w.dtype))
    return t, t.data_ptr()


# ---- one graph, every route ------------------------------------------------------------------------------------------
class Graph:
    """Edge rows in position order (source row, then the key routes' ascending edge rowid) and, for the key routes,
    the key columns they come from."""

    def __init__(self, n, src, dst, eid, w, vkey, ksrc, kdst, sv=None, dv=None, wv=None):
        self.n, self.src, self.dst, self.eid, self.w = n, src, dst, eid, w
        self.vkey, self.ksrc, self.kdst, self.sv, self.dv, self.wv = vkey, ksrc, kdst, sv, dv, wv
        self.wt = 2 if w.dtype.kind == "f" else 1


def graph_from_rows(n, src, dst, w, seed=0):
    """Key columns for rows already in source order: vertex row i holds key 7 * perm[i] - 3; edge row k is the k-th
    row, so the key routes' order (ascending edge rowid within a source row) is the rows' order."""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    order = np.argsort(src, kind="stable")
    src, dst, w = src[order], dst[order], np.asarray(w)[order]
    vkey = np.random.default_rng(seed).permutation(n).astype(np.int64) * 7 - 3
    m = len(src)
    return Graph(n, src, dst, np.arange(m, dtype=np.int64), w, vkey, vkey[src], vkey[dst])


def graph_from_fixture(g):
    """The key fixture's columns; the rows routes get the rows the key join yields, in its position order."""
    v, e, ids = ork.csr_build_keys(g["vkey"], g["src"], g["dst"], None, g["src_valid"], g["dst_valid"])
    n = g["vkey"].shape[0]
    row = np.repeat(np.arange(n), np.diff(v[:n + 1]))
    return Graph(n, row, e, ids, g["w"][ids], g["vkey"], g["src"], g["dst"], g["src_valid"], g["dst_valid"],
                 g["w_valid"]), g["w"]


def make(ctx, gr, route, key_w=None):
    n, m = gr.n, len(gr.src)
    kw = gr.w if key_w is None else key_w
    if route == "chunked":
        csr = pgq.DeviceCSR.create(ctx, n)
        csr.add_vertex_counts(np.arange(n), np.bincount(gr.src, minlength=n)[:n])
        o, i = 0, 0
        while o < m:
            hi = min(m, o + CHUNKS[i % len(CHUNKS)])
            csr.add_edges(m, m, gr.src[o:hi], gr.dst[o:hi], gr.eid[o:hi], gr.w[o:hi])
            o, i = hi, i + 1
        csr.finalize()
        return csr
    if route == "build":
        return pgq.DeviceCSR.build(ctx, n, gr.src, gr.dst, gr.eid, weight=gr.w)
    if route == "build_device":
        s, d, e = cuda(gr.src.astype(np.int32)), cuda(gr.dst.astype(np.int32)), cuda(gr.eid)
        wt, wa = weight_addr(gr.w)
        return pgq.DeviceCSR.build_device(ctx, n, m, addr(s), addr(d), addr(e), d_weight=wa, weight_type=gr.wt)
    if route == "upload":
        v = np.concatenate([[0], np.cumsum(np.bincount(gr.src, minlength=n)[:n])]).astype(np.int64)
        v = np.append(v, v[-1])
        return pgq.DeviceCSR.upload(ctx, n, v, gr.dst, gr.eid, weight=gr.w)
    if route == "build_keys":
        return pgq.DeviceCSR.build_from_keys(ctx, gr.vkey, gr.ksrc, gr.kdst, None, gr.sv, gr.dv, weight=kw,
                                             weight_valid=gr.wv)
    assert route == "build_keys_device"
    cols = [cuda(gr.vkey), cuda(gr.ksrc), cuda(gr.kdst)]
    valid = [None if a is None else cuda(a.astype(np.uint8)) for a in (gr.sv, gr.dv, gr.wv)]
    wt, wa = weight_addr(kw)
    return pgq.DeviceCSR.build_from_keys_device(ctx, n, len(gr.ksrc), addr(cols[0]), addr(cols[1]), addr(cols[2]),
                                                0, *(0 if t is None else addr(t) for t in valid[:2]),
                                                d_weight=wa, d_weight_valid=0 if valid[2] is None else addr(valid[2]),
                                                weight_type=gr.wt)


def outcome(fn):
    """A consumer's answer in a form that compares bit for bit (NaN equal to itself, -0.0 apart from 0.0), or the
    status it was refused with."""
    try:
        out = fn()
    except pgq.PgqError as ex:
        return ("refused", ex.status)
    return ("ok", tuple(bits(x).tolist() if isinstance(x, np.ndarray) else repr(x) for x in out[:-1]))


def answers(csr, ps, pd):
    k = 3
    return {
        "cheapest_path_length": outcome(lambda: csr.cheapest_path_length(ps, pd)),
        "cheapest_path": outcome(lambda: csr.cheapest_path(ps[:64], pd[:64])),
        "cheapest_path_count": outcome(lambda: csr.cheapest_path_count(ps[:64], pd[:64])),
        "all_cheapest_paths": outcome(lambda: csr.all_cheapest_paths(ps[:64], pd[:64], max_paths=4)),
        "cheapest_k_paths": outcome(lambda: csr.cheapest_k_paths(ps[:32], pd[:32], k)),
    }


def state(csr):
    v, e, ids = csr.download()
    return v, e, ids, csr.weight_type(), bits(csr.download_weights()) if csr.weight_type() else None


def check_routes(gr, ctx, other_ctx, ps, pd, routes=ROUTES, key_w=None):
    """Builds gr through every route and a clone of each; everything must equal the first route's.  -> that state and
    its answers."""
    first = None
    for route in routes:
        csr = make(ctx, gr, route, key_w)
        try:
            rep = csr.clone(other_ctx)
            try:
                for c in (csr, rep):
                    got = state(c), answers(c, ps, pd)
                    if first is None:
                        first = got
                        continue
                    (v0, e0, i0, t0, w0), a0 = first
                    (v, e, i, t, w), a = got
                    assert np.array_equal(v, v0) and np.array_equal(e, e0) and np.array_equal(i, i0), route
                    assert t == t0 and (w0 is None) == (w is None), route
                    assert w is None or np.array_equal(w, w0), route
                    for name in a0:
                        assert a[name] == a0[name], (route, name)
            finally:
                rep.free()
        finally:
            csr.free()
    return first


def expected_rows(gr):
    """The CSR of the rows by the restatement: (v, e, ids, weights)."""
    return orc.csr_build_weighted(gr.n, gr.src, gr.dst, gr.w, gr.eid)


# ---- the generated shapes ----------------------------------------------------------------------------------------------
def shapes():
    rng = np.random.default_rng(11)
    out = {}
    n = 40
    out["self_loops_parallel_i64"] = (n, np.r_[np.arange(n), rng.integers(0, n, 300), [3, 3, 3]],
                                      np.r_[np.arange(n), rng.integers(0, n, 300), [4, 4, 4]],
                                      np.r_[rng.integers(1, 9, n + 300), [5, 1, 9]])
    w = rng.random(n + 303) * 4.0
    w[[5, 17, 40]] = [-0.0, np.nan, 0.0]
    out["self_loops_parallel_f64"] = (n, out["self_loops_parallel_i64"][1], out["self_loops_parallel_i64"][2], w)
    out["n1_self_loops_i64"] = (1, np.zeros(3, np.int64), np.zeros(3, np.int64), np.array([4, 2, 7]))
    # a hub row of 9000 edges spans several create_csr_edge chunks and staging slots
    n = 300
    src = np.r_[np.full(9000, 7), rng.integers(0, n, 2000)]
    dst = np.r_[rng.integers(0, n, 9000), rng.integers(0, n, 2000)]
    out["hub_i64"] = (n, src, dst, rng.integers(0, 1 << 40, len(src)))
    out["hub_f64"] = (n, src, dst, rng.random(len(src)) + 0.25)
    # negative weights on a DAG (no negative cycle): cheapest_path_length relaxes from every vertex, cheapest_k_paths
    # refuses the CSR
    n = 200
    rank = rng.permutation(n)
    a, b = rng.integers(0, n, 900), rng.integers(0, n, 900)
    a, b = a[a != b], b[a != b]
    fwd = rank[a] < rank[b]
    s, d = np.where(fwd, a, b), np.where(fwd, b, a)
    out["dag_negative_i64"] = (n, s, d, rng.integers(-30, 31, len(s)))
    out["dag_negative_f64"] = (n, s, d, rng.integers(-(1 << 12), 1 << 12, len(s)) / 64.0)
    return out


SHAPES = shapes()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_generated_shape_every_route(gpu_ctx, other_ctx, name):
    n, src, dst, w = SHAPES[name]
    gr = graph_from_rows(n, src, dst, w)
    rng = np.random.default_rng(len(src))
    ps, pd = rng.integers(0, n, 200), rng.integers(0, n, 200)
    (v, e, ids, wt, wb), ans = check_routes(gr, gpu_ctx, other_ctx, ps, pd)
    ev, ee, eids, ew = expected_rows(gr)
    assert np.array_equal(v, ev) and np.array_equal(e, ee) and np.array_equal(ids, eids)
    assert wt == gr.wt and np.array_equal(wb, bits(ew))
    ocost, ovalid = orc.cheapest_path_length(n, ev, ee, ew, ps, pd)
    cost, valid = ans["cheapest_path_length"][1]
    keep = ovalid == 1
    assert valid == ovalid.astype(np.int64).tolist() and np.array_equal(np.array(cost)[keep], bits(ocost)[keep])
    if np.any(w < 0):
        assert ans["cheapest_k_paths"] == ("refused", pgq.PGQ_ERR_UNSUPPORTED)


@pytest.mark.parametrize("kind", ["i64", "f64"])
def test_no_edges_records_the_weight_type(gpu_ctx, other_ctx, kind):
    """m = 0: every one-shot route knows its weight type and answers as on a weighted graph without the path; the
    chunked protocol, which never sees a weight, stays at type 0."""
    n = 5
    w = np.zeros(0, np.float64 if kind == "f64" else np.int64)
    gr = graph_from_rows(n, [], [], w)
    ps, pd = np.array([0, 1, 4, 2]), np.array([0, 3, 4, 1])
    (v, e, ids, wt, wb), ans = check_routes(gr, gpu_ctx, other_ctx, ps, pd, routes=ROUTES[1:])
    assert wt == gr.wt and len(e) == 0 and len(wb) == 0 and np.array_equal(v, np.zeros(n + 2))
    cost, valid = ans["cheapest_path_length"][1]
    assert valid == [1, 0, 1, 0] and bits(np.zeros(1, w.dtype)).tolist() * 2 == [cost[0], cost[2]]
    chunked = make(gpu_ctx, gr, "chunked")
    assert chunked.weight_type() == 0
    chunked.free()


@pytest.mark.parametrize("name", KEY_FIXTURES)
def test_key_fixture_every_route(gpu_ctx, other_ctx, name):
    z = np.load(os.path.join(GOLDEN, f"refkw_{name}.npz"))
    g = {k: z[k] for k in z.files}
    gr, key_w = graph_from_fixture(g)
    n = gr.n
    ps, pd = g["psrc"], g["pdst"]
    (v, e, ids, wt, wb), ans = check_routes(gr, gpu_ctx, other_ctx, ps, pd, key_w=key_w)
    assert wt == int(g["w_type"])
    assert np.array_equal(v, g["csr_v"])
    row = np.repeat(np.arange(n), np.diff(v[:n + 1]))
    mine, ref = np.lexsort((wb, e, row)), np.lexsort((bits(g["csr_w"]), g["csr_e"], row))
    assert np.array_equal(e[mine], g["csr_e"][ref]) and np.array_equal(wb[mine], bits(g["csr_w"])[ref])
    cost, valid = ans["cheapest_path_length"][1]
    assert valid == g["cost_valid"].astype(np.int64).tolist()
    keep = g["cost_valid"] == 1
    assert np.array_equal(np.array(cost)[keep], bits(g["cost"])[keep])


# ---- argument errors ---------------------------------------------------------------------------------------------------
def test_exactly_one_weight_pointer(gpu_ctx):
    lib, h = gpu_ctx._lib, C.c_void_p()
    i64 = np.array([1, 2], np.int64)
    f64 = np.array([1.0, 2.0])
    src, dst, keys = np.array([0, 1], np.int64), np.array([1, 0], np.int64), np.array([10, 20], np.int64)
    pi, pf = i64.ctypes.data_as(C.POINTER(C.c_int64)), f64.ctypes.data_as(C.POINTER(C.c_double))
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
    v = np.array([0, 1, 2, 2], np.int64)
    d_src, d_dst, d_keys = cuda(src.astype(np.int32)), cuda(dst.astype(np.int32)), cuda(keys)
    d_i, d_f = cuda(i64), cuda(f64)
    for wi, wf, dwi, dwf in ((pi, pf, d_i.data_ptr(), d_f.data_ptr()), (None, None, None, None)):
        calls = [
            lambda: lib.pgq_csr_build_weighted(gpu_ctx._h, 2, 2, p(src), p(dst), None, wi, wf, C.byref(h)),
            lambda: lib.pgq_csr_build_device_weighted(gpu_ctx._h, 2, 2, d_src.data_ptr(), d_dst.data_ptr(), None,
                                                      dwi, dwf, C.byref(h)),
            lambda: lib.pgq_csr_upload_weighted(gpu_ctx._h, 2, 2, p(v), p(dst), None, wi, wf, C.byref(h)),
            lambda: lib.pgq_csr_build_keys_weighted(gpu_ctx._h, 2, p(keys), None, 2, p(keys), p(keys[::-1].copy()),
                                                    None, None, wi, wf, None, C.byref(h)),
            lambda: lib.pgq_csr_build_keys_weighted_device(gpu_ctx._h, 2, d_keys.data_ptr(), None, 2,
                                                           d_keys.data_ptr(), d_keys.data_ptr(), None, None, dwi, dwf,
                                                           None, C.byref(h)),
        ]
        for call in calls:
            assert call() == pgq.PGQ_ERR_INVALID_ARG
            assert b"exactly one" in lib.pgq_last_error()
            assert not h.value


@pytest.mark.parametrize("device", [False, True])
def test_null_weight_on_a_joined_edge(gpu_ctx, device):
    keys = np.array([5, 6, 7], np.int64)
    src, dst = np.array([5, 6, 9, 7], np.int64), np.array([6, 7, 5, 5], np.int64)  # edge 2 joins nothing (key 9)
    w = np.array([1.5, 2.5, np.nan, 4.0])

    def build(wv):
        if not device:
            return pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, src, dst, weight=w, weight_valid=wv)
        cols = [cuda(keys), cuda(src), cuda(dst), cuda(w), cuda(np.asarray(wv, np.uint8))]
        return pgq.DeviceCSR.build_from_keys_device(gpu_ctx, 3, 4, *(c.data_ptr() for c in cols[:3]),
                                                    d_weight=cols[3].data_ptr(), d_weight_valid=cols[4].data_ptr(),
                                                    weight_type=2)

    csr = build([1, 1, 0, 1])  # the NULL sits on the edge that joins nothing
    assert csr.weight_type() == 2 and np.array_equal(csr.download_weights(), [1.5, 2.5, 4.0])
    csr.free()
    with pytest.raises(pgq.InvalidInputException, match="edge row 1 joins but its weight is NULL") as ex:
        build([1, 0, 0, 0])
    assert ex.value.status == pgq.PGQ_ERR_INVALID_ARG


def test_undirected_with_a_weight_raises(gpu_ctx):
    keys = np.array([1, 2], np.int64)
    with pytest.raises(ValueError, match="undirected"):
        pgq.DeviceCSR.build_from_keys(gpu_ctx, keys, keys, keys[::-1], undirected=True, weight=[1, 2])
    d = cuda(keys)
    with pytest.raises(ValueError, match="undirected"):
        pgq.DeviceCSR.build_from_keys_device(gpu_ctx, 2, 2, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                                             undirected=True, d_weight=d.data_ptr(), weight_type=1)
