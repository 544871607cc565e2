#!/usr/bin/env python
"""Time pgq_cheapest_path_length and pgq_cheapest_path on R-MAT graphs, 1024 hashed pairs, BIGINT and DOUBLE weights,
with the card's name and power limit next to the numbers.

    python tools/cheapest_path_bench.py [--scales 20 22] [--pairs 1024] [--warm 2] [--out FILE]

Weights are drawn from a seeded generator: integers 1..100 (BIGINT) or k / 1024 for k in 1..2^20 (DOUBLE), and one
run with BIGINT weights in [-50, 50] on a DAG (every R-MAT edge oriented from the lower to the higher id, self-loops
dropped), where the sweeps start from every vertex.  Per function: the first call and the median of the warm calls
(CUDA events around calls that end in a stream synchronise), batches, Bellman-Ford sweeps and lanes; for cheapest_path
also the tight levels, their frontier vertices and out-edges.  Every call is checked: cheapest_path's rows are non-NULL
only where the cost is, and each path's weights sum to its row's cost."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from duckpgq_extension_b200 import datagen, pgq  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def timed(fn, warm):
    """-> (result of the last call, first call ms, median warm call ms)"""
    times = []
    res = None
    for _ in range(1 + warm):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return res, round(times[0], 3), round(float(np.median(times[1:])) if warm else times[0], 3)


def build(ctx, n, src, dst, w):
    m = len(src)
    csr = pgq.DeviceCSR.create(ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    step = 1 << 22
    for o in range(0, m, step):
        csr.add_edges(m, m, src[o:o + step], dst[o:o + step], np.arange(o, min(o + step, m)), w[o:o + step])
    csr.finalize()
    return csr


def check(w, cost, cvalid, paths):
    """paths only where costs are valid; sums equal costs (weights >= 0: d(s) = 0, and every valid cost has a path)"""
    eid_w = w  # edge id = input position
    neg = (w < 0).any()
    for i, path in enumerate(paths):
        if path is None:
            assert neg or not cvalid[i], f"row {i}: valid cost without a path"
            continue
        assert cvalid[i], f"row {i}: a path at a NULL cost"
        ws = eid_w[np.asarray(path[1::2], dtype=np.int64)]
        acc = ws.dtype.type(0)
        for x in ws:
            acc = acc + x
        assert acc == cost[i], f"row {i}: path sums to {acc}, cost {cost[i]}"


def run(ctx, label, n, src, dst, w, ps, pd, warm):
    csr = build(ctx, n, src, dst, w)
    (cost, cvalid, cst), c_first, c_warm = timed(lambda: csr.cheapest_path_length(ps, pd), warm)
    (paths, pst), p_first, p_warm = timed(lambda: csr.cheapest_path(ps, pd), warm)
    csr.free()
    check(w, cost, cvalid, paths)
    return {
        "graph": label, "n": int(n), "m": int(len(src)), "pairs": int(len(ps)), "weights": str(w.dtype),
        "cheapest_path_length": {"first_call_ms": c_first, "warm_call_ms_median": c_warm, "batches": cst["batches"],
                                 "sweeps": cst["levels"], "lanes": cst["lanes"], "valid_rows": int(cvalid.sum())},
        "cheapest_path": {"first_call_ms": p_first, "warm_call_ms_median": p_warm, "batches": pst["batches"],
                          "sweeps": pst["levels"], "lanes": pst["lanes"], "tight_levels": pst["push_levels"],
                          "tight_frontier_vertices": pst["frontier_vertices"],
                          "tight_edges": pst["edges_traversed"], "paths": sum(x is not None for x in paths),
                          "mean_hops": round(float(np.mean([(len(x) - 1) / 2 for x in paths if x is not None] or [0])), 2)},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--warm", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "runs": []}
    print(results["card"], flush=True)
    for scale in a.scales:
        n, src, dst = datagen.rmat_edges(scale)
        ps, pd = datagen.hashed_pairs(a.pairs, n)
        rng = np.random.default_rng(1000 + scale)
        for kind in ("i64", "f64"):
            w = rng.integers(1, 101, len(src)) if kind == "i64" else rng.integers(1, (1 << 20) + 1, len(src)) / 1024.0
            r = run(ctx, f"rmat{scale}", n, src, dst, w, ps, pd, a.warm)
            print(json.dumps(r), flush=True)
            results["runs"].append(r)
    scale = a.scales[0]
    n, src, dst = datagen.rmat_edges(scale)
    keep = src != dst
    lo, hi = np.minimum(src, dst)[keep], np.maximum(src, dst)[keep]
    w = np.random.default_rng(7).integers(-50, 51, len(lo))
    ps, pd = datagen.hashed_pairs(a.pairs, n)
    r = run(ctx, f"rmat{scale}_dag_negative", n, lo, hi, w, ps, pd, a.warm)
    print(json.dumps(r), flush=True)
    results["runs"].append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
