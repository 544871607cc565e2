#!/usr/bin/env python
"""Time pgq_cheapest_k_paths (WALK, ACYCLIC and TRAIL) for k = 1, 4, 16 on R-MAT graphs with hashed BIGINT weights
1..16 and 1024 hashed pairs, with the card's name and power limit read in the same run.

    python tools/cheapest_k_bench.py [--scales 18 20] [--pairs 1024] [--ks 1 4 16] [--modes WALK ACYCLIC TRAIL]
                                     [--warm 2] [--check 2] [--check-k 1] [--out FILE]

Per (mode, k): the first call and the median of the warm calls (host time around calls that end in a stream
synchronise), the call's counters, and a separate torch.profiler run that splits the call between seeding (the seed
checks and the seeds), sweeps (k_bf_sweep), tight levels (tight seed, level and finish kernels), walk-back, other device
work (the step-list sort, the distance fill) and the host's share (the call's wall time minus its device kernels).
`--check` sampled rows are checked against oracle/pgq_oracle_cheapest_k.c over the downloaded CSR in the same run, for
k <= --check-k (the oracle runs a sequential Bellman-Ford per spur search)."""
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
from oracle import pgq_oracle_cheapest_k as ock  # noqa: E402


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
    return res, round(times[0], 2), round(float(np.median(times[1:])) if warm else times[0], 2)


def split(fn):
    """ms of one call by phase, from torch.profiler's kernel events; host = wall time minus the kernels"""
    from torch.profiler import ProfilerActivity, profile
    out = {"seeding": 0.0, "sweeps": 0.0, "tight_levels": 0.0, "walk_back": 0.0, "other_device": 0.0}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name[5:] if ev.name.startswith("void ") else ev.name
        ms = ev.time_range.elapsed_us() / 1e3
        if name.startswith(("k_ck_has_seed", "k_ck_seed")):
            out["seeding"] += ms
        elif name.startswith("k_bf_sweep"):
            out["sweeps"] += ms
        elif name.startswith(("k_ck_tight_seed", "k_ck_tight_level", "k_ck_finish")):
            out["tight_levels"] += ms
        elif name.startswith("k_ck_walk"):
            out["walk_back"] += ms
        else:
            out["other_device"] += ms
    out["host"] = wall - sum(out.values())
    return {k: round(v, 2) for k, v in out.items()}


def hashed_weights(m):
    """BIGINT weights 1..16 from a multiplicative hash of the edge's position"""
    x = (np.arange(m, dtype=np.uint64) * np.uint64(2654435761)) >> np.uint64(7)
    return (x % np.uint64(16)).astype(np.int64) + 1


def build(ctx, n, src, dst, w):
    m = len(src)
    csr = pgq.DeviceCSR.create(ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    step = 1 << 22
    for o in range(0, m, step):
        csr.add_edges(m, m, src[o:o + step], dst[o:o + step], np.arange(o, min(o + step, m)), w[o:o + step])
    csr.finalize()
    return csr


def run(ctx, scale, pairs, ks, modes, warm, check, check_k):
    n, src, dst = datagen.rmat_edges(scale)
    w = hashed_weights(len(src))
    ps, pd = datagen.hashed_pairs(pairs, n)
    csr = build(ctx, n, src, dst, w)
    ref = None
    res = {"graph": f"rmat{scale}", "n": int(n), "m": int(len(src)), "pairs": int(len(ps)), "weights": "bigint 1..16",
           "runs": {}}
    for mode in modes:
        for k in ks:
            call = lambda: csr.cheapest_k_paths(ps, pd, k, mode=mode)  # noqa: E731
            (paths, costs, npaths, st), first, warm_ms = timed(call, warm)
            checked = 0
            if k <= check_k and check > 0:
                pick = np.linspace(0, len(ps) - 1, check).astype(np.int64)
                if ref is None:
                    v, e, ids = csr.download()
                    ref = (v, e, ids, csr.download_weights())
                opaths, ocosts, _, _ = ock.cheapest_k_paths(n, *ref, ps[pick], pd[pick], k, mode)
                assert opaths == [paths[i] for i in pick], f"{mode} k={k}: paths differ from the oracle"
                assert ocosts == [costs[i] for i in pick], f"{mode} k={k}: costs differ from the oracle"
                checked = check
            r = {"first_ms": first, "warm_ms_median": warm_ms, "device_total_ms": round(st["total_ms"], 2),
                 "batches": st["batches"], "lanes": st["lanes"], "searches": st["searches"], "sweeps": st["levels"],
                 "tight_levels": st["push_levels"], "paths": int(npaths.sum()),
                 "valid_rows": int(sum(p is not None for p in paths)), "kernel_launches": st["kernel_launches"],
                 "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"], "ms_by_phase": split(call),
                 "oracle_checked_rows": checked}
            res["runs"][f"{mode} k={k}"] = r
            print(json.dumps({res["graph"]: {f"{mode} k={k}": r}}), flush=True)
    csr.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[18, 20])
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--modes", nargs="+", default=["WALK", "ACYCLIC", "TRAIL"])
    ap.add_argument("--warm", type=int, default=2)
    ap.add_argument("--check", type=int, default=2)
    ap.add_argument("--check-k", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "graphs": []}
    print(results["card"], flush=True)
    for scale in a.scales:
        results["graphs"].append(run(ctx, scale, a.pairs, a.ks, a.modes, a.warm, a.check, a.check_k))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
