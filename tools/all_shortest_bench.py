#!/usr/bin/env python
"""Time pgq_shortestpath, pgq_shortest_path_count and pgq_all_shortest_paths (max_paths 1 and 64) on R-MAT graphs with
1024 hashed pairs, with the card's name and power limit read in the same run.

    python tools/all_shortest_bench.py [--scales 20 22] [--pairs 1024] [--warm 3] [--check 48] [--out FILE]

Per function: the first call and the median of the warm calls (host time around calls that end in a stream
synchronise), and the call's BFS counters.  A separate torch.profiler run of all_shortest_paths(64) splits the device
time between the BFS kernels and the path-count / step-list / unranking kernels (k_sigma_level, k_as_*, the radix
sort's k_rs_*).  Also: the distribution of the counts, the rows that saturate, and a check of `--check` sampled rows
(counts, validity and the 64 first lists) against oracle/pgq_oracle_allshortest.c over the downloaded CSR."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from duckpgq_extension_b200 import datagen, pgq  # noqa: E402
from oracle import pgq_oracle_allshortest as oas  # noqa: E402

INT64_MAX = (1 << 63) - 1
NEW_KERNELS = ("k_sigma_level", "k_as_", "k_rs_", "k_scan_")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def timed(fn, warm):
    """-> (result of the last call, first call ms, median warm call ms); each call ends in a stream synchronise"""
    times, res = [], None
    for _ in range(1 + warm):
        t0 = time.perf_counter()
        res = fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return res, round(times[0], 2), round(float(np.median(times[1:])), 2)


def kernel_split(fn):
    """device time of the kernels of one call, by torch.profiler: (BFS ms, path counts / lists ms)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    bfs = new = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = ev.cuda_time_total if t is None else t
        if not t:
            continue
        name = ev.key[5:] if ev.key.startswith("void ") else ev.key  # (templates print with their return type)
        if any(name.startswith(k) for k in NEW_KERNELS):
            new += t / 1e3
        elif name.startswith("k_"):
            bfs += t / 1e3
    return round(bfs, 2), round(new, 2)


def check_sample(csr, n, ps, pd, cnt, valid, paths, k):
    v, e, ids = csr.download()
    pick = np.linspace(0, len(ps) - 1, k).astype(np.int64)
    ocnt, ovalid = oas.shortest_path_count(n, v, e, ids, ps[pick], pd[pick])
    assert np.array_equal(ovalid, valid[pick]) and np.array_equal(ocnt, cnt[pick]), "counts differ from the oracle"
    opaths, _ = oas.all_shortest_paths(n, v, e, ids, ps[pick], pd[pick], 64)
    assert opaths == [paths[i] for i in pick], "lists differ from the oracle"
    return int(k)


def run(ctx, scale, pairs, warm, k):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(pairs, n)
    csr = pgq.DeviceCSR.build(ctx, n, src, dst)
    (sp, sst), sp_first, sp_warm = timed(lambda: csr.shortestpath(ps, pd), warm)
    (cnt, valid, cst), c_first, c_warm = timed(lambda: csr.shortest_path_count(ps, pd), warm)
    (p1, _, a1st), a1_first, a1_warm = timed(lambda: csr.all_shortest_paths(ps, pd, 1), warm)
    (p64, _, a64st), a64_first, a64_warm = timed(lambda: csr.all_shortest_paths(ps, pd, 64), warm)
    assert [None if x is None else x[0] for x in p1] == sp, "path 0 differs from shortestpath"
    checked = check_sample(csr, n, ps, pd, cnt, valid, p64, k)
    split_count = kernel_split(lambda: csr.shortest_path_count(ps, pd))
    split_64 = kernel_split(lambda: csr.all_shortest_paths(ps, pd, 64))
    csr.free()
    counts = cnt[valid == 1].astype(np.float64)
    q = np.percentile(counts, [50, 90, 99, 100]) if len(counts) else [0, 0, 0, 0]
    bfs = {k2: sst[k2] for k2 in ("batches", "levels", "lanes", "edges_traversed")}
    return {
        "graph": f"rmat{scale}", "n": int(n), "m": int(len(src)), "pairs": int(len(ps)), "bfs": bfs,
        "shortestpath": {"first_ms": sp_first, "warm_ms_median": sp_warm, "device_total_ms": round(sst["total_ms"], 2)},
        "shortest_path_count": {"first_ms": c_first, "warm_ms_median": c_warm,
                                "device_total_ms": round(cst["total_ms"], 2),
                                "kernel_ms_bfs_vs_counts": split_count},
        "all_shortest_paths_1": {"first_ms": a1_first, "warm_ms_median": a1_warm,
                                 "device_total_ms": round(a1st["total_ms"], 2)},
        "all_shortest_paths_64": {"first_ms": a64_first, "warm_ms_median": a64_warm,
                                  "device_total_ms": round(a64st["total_ms"], 2),
                                  "kernel_ms_bfs_vs_counts_lists": split_64,
                                  "lists": int(sum(len(x) for x in p64 if x is not None))},
        "counts": {"valid_rows": int(valid.sum()), "p50": float(q[0]), "p90": float(q[1]), "p99": float(q[2]),
                   "max": int(cnt.max()) if len(cnt) else 0, "rows_above_1": int((cnt > 1).sum()),
                   "saturated_rows": int((cnt == INT64_MAX).sum())},
        "oracle_checked_rows": checked,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--warm", type=int, default=3)
    ap.add_argument("--check", type=int, default=48)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "runs": []}
    print(results["card"], flush=True)
    for scale in a.scales:
        r = run(ctx, scale, a.pairs, a.warm, a.check)
        print(json.dumps(r), flush=True)
        results["runs"].append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
