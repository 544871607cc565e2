#!/usr/bin/env python
"""Time cheapest_path, cheapest_path_count and all_cheapest_paths(1 / 64) on R-MAT graphs, 1024 hashed pairs, with the
card's name and power limit next to the numbers.

    python tools/all_cheapest_bench.py [--scale 20] [--pairs 1024] [--warm 1] [--out FILE]

The workloads are tools/cheapest_path_bench.py's: BIGINT weights 1..100 and DOUBLE weights k / 1024 for k in 1..2^20,
plus BIGINT weights 0..3, where zero-cost cycles make some counts infinite and the |B(t)| bound is what ends those rows.
Per function: the first call and the median of the warm calls (CUDA events around calls that end in a stream
synchronise) and its counters.  Per workload: the distribution of the counts (NULL, 1, 2..63, 64 and more, infinite).
A separate torch.profiler run of one all_cheapest_paths(64) call splits its device time between the Bellman-Ford sweeps
(k_bf_*) and the tight walk search (the rest).  Every call is checked: the counts of the two calls agree, path 0 is
cheapest_path's, and (BIGINT) every listed path's weights sum to the row's cost."""
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

INT64_MAX = (1 << 63) - 1


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


def distribution(cnt, valid):
    c = np.asarray(cnt)
    return {"null": int((valid == 0).sum()), "one": int(((c == 1) & (valid == 1)).sum()),
            "2..63": int(((c >= 2) & (c < 64)).sum()), "64+": int(((c >= 64) & (c < INT64_MAX)).sum()),
            "infinite_or_saturated": int((c == INT64_MAX).sum())}


def profile_split(csr, ps, pd):
    """device time of one all_cheapest_paths(64) call: the sweeps (k_bf_*) against everything else"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        csr.all_cheapest_paths(ps, pd, 64)
        torch.cuda.synchronize()
    sweeps = other = 0.0
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        if not t or ev.key.startswith("cuda") or "Memset" in ev.key or "Memcpy" in ev.key:
            continue
        name = ev.key.split("(")[0].replace("void ", "")
        per[name] = per.get(name, 0.0) + t / 1000.0
        if "k_bf_" in ev.key:
            sweeps += t / 1000.0
        else:
            other += t / 1000.0
    top = dict(sorted(per.items(), key=lambda x: -x[1])[:8])
    return {"sweeps_ms": round(sweeps, 3), "tight_walks_ms": round(other, 3),
            "kernels_ms": {k: round(v, 3) for k, v in top.items()}}


def run(ctx, label, n, src, dst, w, ps, pd, warm):
    csr = build(ctx, n, src, dst, w)
    out = {"graph": label, "n": int(n), "m": int(len(src)), "pairs": int(len(ps)), "weights": label.split("_", 1)[1]}
    try:
        (paths, pst), f, wm = timed(lambda: csr.cheapest_path(ps, pd), warm)
        out["cheapest_path"] = {"first_call_ms": f, "warm_call_ms_median": wm, "sweeps": pst["levels"]}
        (cnt, valid, cst), f, wm = timed(lambda: csr.cheapest_path_count(ps, pd), warm)
        out["cheapest_path_count"] = {"first_call_ms": f, "warm_call_ms_median": wm, "batches": cst["batches"],
                                      "sweeps": cst["levels"], "lanes": cst["lanes"],
                                      "reach_levels": cst["push_levels"], "count_layers": cst["pull_levels"],
                                      "kernel_launches": cst["kernel_launches"]}
        out["counts"] = distribution(cnt, valid)
        for k in (1, 64):
            (lists, lcnt, lst), f, wm = timed(lambda: csr.all_cheapest_paths(ps, pd, k), warm)
            assert lcnt.tolist() == cnt.tolist()
            assert [x[0] if x else None for x in lists] == paths
            if w.dtype.kind == "i":
                cost, cvalid, _ = csr.cheapest_path_length(ps, pd)
                for i, rows in enumerate(lists):
                    for path in rows or []:
                        assert int(w[np.asarray(path[1::2], np.int64)].sum()) == cost[i]
            out[f"all_cheapest_paths_{k}"] = {
                "first_call_ms": f, "warm_call_ms_median": wm, "paths": int(sum(len(x) for x in lists if x)),
                "count_layers": lst["pull_levels"], "kernel_launches": lst["kernel_launches"],
                "mean_edges": round(float(np.mean([(len(p) - 1) / 2 for x in lists if x for p in x] or [0])), 2)}
        out["profile_all_cheapest_paths_64"] = profile_split(csr, ps, pd)
    finally:
        csr.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--warm", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "runs": []}
    print(results["card"], flush=True)
    n, src, dst = datagen.rmat_edges(a.scale)
    ps, pd = datagen.hashed_pairs(a.pairs, n)
    rng = np.random.default_rng(1000 + a.scale)
    for kind in ("i64_1_100", "f64", "i64_0_3"):
        if kind == "i64_1_100":
            w = rng.integers(1, 101, len(src))
        elif kind == "f64":
            w = rng.integers(1, (1 << 20) + 1, len(src)) / 1024.0
        else:
            w = rng.integers(0, 4, len(src))
        r = run(ctx, f"rmat{a.scale}_{kind}", n, src, dst, w, ps, pd, a.warm)
        print(json.dumps(r), flush=True)
        results["runs"].append(r)
    results["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
