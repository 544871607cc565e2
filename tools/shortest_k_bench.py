#!/usr/bin/env python
"""Time pgq_shortest_k_paths (k = 1, 16, 64) on R-MAT graphs with 1024 hashed pairs, with the card's name and power
limit read in the same run.

    python tools/shortest_k_bench.py [--scales 20 22] [--pairs 1024] [--ks 1 16 64] [--warm 2] [--check 4] [--out FILE]

Per k: the first call and the median of the warm calls (host time around calls that end in a stream synchronise), the
call's counters, the layers per batch, the storing groups and the peak layer memory (both from the rows' last walk
lengths by the header's packing rule), and a separate torch.profiler run that splits the device time between the
backward reach, the counting pass, the storing pass and the unranking (k_ks_omega is counted as counting or storing
by launch: the counting pass's launches come first).  `--check` sampled rows are checked against
oracle/pgq_oracle_kshortest.c over the downloaded CSR in the same run."""
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
from oracle import pgq_oracle_kshortest as oks  # noqa: E402

BUDGET = 4 << 30


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def timed(fn, warm):
    times, res = [], None
    for _ in range(1 + warm):
        t0 = time.perf_counter()
        res = fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return res, round(times[0], 2), round(float(np.median(times[1:])), 2)


def groups(paths, n_ab, lanes):
    """the storing groups and the largest group's layer bytes, by the header's greedy packing"""
    count, peak, rows, gh = 0, 0, 0, 0
    for p in paths:
        if not p:
            continue
        h = (len(p[-1]) - 1) // 2
        nh = max(gh, h)
        if rows and (rows == lanes or (nh + 1) * n_ab * (rows + 1) * 8 > BUDGET):
            count, peak, rows, gh = count + 1, max(peak, gh * n_ab * rows * 8), 0, 0
            nh = h
        rows, gh = rows + 1, nh
    if rows:
        count, peak = count + 1, max(peak, gh * n_ab * rows * 8)
    return count, peak


def split(fn):
    """device ms of one call by phase, from torch.profiler's kernel events in launch order"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"backward_reach": 0.0, "counting": 0.0, "storing": 0.0, "unranking": 0.0, "other": 0.0}
    events = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                    key=lambda e: e.time_range.start)
    storing = False
    for ev in events:
        name = ev.name[5:] if ev.name.startswith("void ") else ev.name
        ms = ev.time_range.elapsed_us() / 1e3
        if name.startswith("k_ks_reach"):
            out["backward_reach"] += ms
        elif name.startswith("k_ks_group_src"):
            storing = True
        elif name.startswith("k_ks_omega") or name.startswith("k_ks_step") or name.startswith("k_ks_start"):
            out["storing" if storing else "counting"] += ms
        elif name.startswith("k_ks_unrank"):
            out["unranking"] += ms
        else:
            out["other"] += ms
    return {k: round(v, 2) for k, v in out.items()}


def run(ctx, scale, pairs, ks, warm, check):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(pairs, n)
    csr = pgq.DeviceCSR.build(ctx, n, src, dst)
    n_ab = int(np.count_nonzero(np.bincount(dst, minlength=n)))
    v = e = ids = None
    res = {"graph": f"rmat{scale}", "n": int(n), "m": int(len(src)), "n_ab": n_ab, "pairs": int(len(ps)), "k": {}}
    for k in ks:
        (paths, npaths, st), first, warm_ms = timed(lambda: csr.shortest_k_paths(ps, pd, k), warm)
        g, peak = groups(paths, n_ab, st["lanes"])
        pick = np.linspace(0, len(ps) - 1, check).astype(np.int64)
        if v is None:
            v, e, ids = csr.download()
        opaths, _, _ = oks.shortest_k_paths(n, v, e, ids, ps[pick], pd[pick], k)
        assert opaths == [paths[i] for i in pick], f"k={k}: walks differ from the oracle"
        res["k"][k] = {
            "first_ms": first, "warm_ms_median": warm_ms, "device_total_ms": round(st["total_ms"], 2),
            "batches": st["batches"], "lanes": st["lanes"], "levels": st["levels"],
            "layers_per_batch": round(st["levels"] / max(st["batches"], 1), 2), "push_levels": st["push_levels"],
            "groups": g, "peak_layer_bytes": int(peak), "walks": int(npaths.sum()),
            "valid_rows": int(sum(p is not None for p in paths)), "kernel_launches": st["kernel_launches"],
            "device_ms_by_phase": split(lambda: csr.shortest_k_paths(ps, pd, k)), "oracle_checked_rows": int(check),
        }
        print(json.dumps({res["graph"]: {k: res["k"][k]}}), flush=True)
    csr.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--warm", type=int, default=2)
    ap.add_argument("--check", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "runs": []}
    print(results["card"], flush=True)
    for scale in a.scales:
        results["runs"].append(run(ctx, scale, a.pairs, a.ks, a.warm, a.check))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
