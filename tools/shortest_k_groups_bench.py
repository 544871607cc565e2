#!/usr/bin/env python
"""Time pgq_shortest_k_groups (WALK at k = 1, 2, 4 with max_paths 64 and count-only; ACYCLIC and TRAIL at k = 1, 2 with
max_paths 64) on R-MAT graphs with 1024 hashed pairs, with the card's name and power limit read in the same run.

    python tools/shortest_k_groups_bench.py [--scales 20 22] [--pairs 1024] [--max-paths 64] [--warm 2] [--check 2]
                                            [--only NAME ...] [--out FILE]

Per run: the first call and the median of the warm calls (host time around calls that end in a stream synchronise),
the call's counters, and a separate torch.profiler run that splits the call by kernel family (WALK: backward reach,
counting, storing, unranking; the modes: seeding, forward levels, walk-back), other device work (the step-list sort,
memsets, scans) and the host's share (the call's wall time minus its device kernels).  `--check` sampled rows are
checked against oracle/pgq_oracle_kgroups.c over the downloaded CSR in the same run.  `--only` keeps the runs whose
name (e.g. "TRAIL k=2 max_paths=64") contains one of the given strings."""
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
from oracle import pgq_oracle_kgroups as okg  # noqa: E402

PHASES = (("backward_reach", ("k_ks_reach",)), ("counting", ("k_ks_start", "k_ks_omega", "k_kg_step")),
          ("unranking", ("k_ks_unrank", "k_ks_group_src")), ("seeding", ("k_km_has_seed", "k_km_seed")),
          ("forward_levels", ("k_km_level", "k_km_fold", "k_km_finish")), ("walk_back", ("k_km_walk",)))


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


def split(fn):
    """ms of one call by kernel family, from torch.profiler's kernel events; host = wall time minus the kernels.  (The
    storing pass runs k_ks_omega too, so WALK's counting includes the layers it recomputes.)"""
    from torch.profiler import ProfilerActivity, profile
    out = {name: 0.0 for name, _ in PHASES}
    out["other_device"] = 0.0
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
        out[next((p for p, pre in PHASES if name.startswith(pre)), "other_device")] += ms
    out["host"] = wall - sum(out.values())
    return {k: round(v, 2) for k, v in out.items() if v or k == "host"}


def run(ctx, scale, pairs, max_paths, warm, check, only):
    n, src, dst = datagen.rmat_edges(scale)
    ps, pd = datagen.hashed_pairs(pairs, n)
    csr = pgq.DeviceCSR.build(ctx, n, src, dst)
    v, e, ids = csr.download()
    pick = np.linspace(0, len(ps) - 1, check).astype(np.int64) if check > 0 else np.zeros(0, np.int64)
    res = {"graph": f"rmat{scale}", "n": int(n), "m": int(len(src)), "pairs": int(len(ps)), "runs": {}}
    plan = [("WALK", k, max_paths, False) for k in (1, 2, 4)] + [("WALK", k, 0, True) for k in (1, 2, 4)]
    plan += [(m, k, max_paths, False) for m in ("ACYCLIC", "TRAIL") for k in (1, 2)]
    for mode, k, mp, count_only in plan:
        name = f"{mode} k={k} " + ("count" if count_only else f"max_paths={mp}")
        if only and not any(o in name for o in only):
            continue
        if count_only:
            call = lambda: csr.shortest_k_groups_count(ps, pd, k)  # noqa: E731
        else:
            call = lambda: csr.shortest_k_groups(ps, pd, k, mp, mode=mode)  # noqa: E731
        out, first, warm_ms = timed(call, warm)
        st = out[-1]
        cnt = out[0] if count_only else out[1]
        _, orows, _ = okg.shortest_k_groups(n, v, e, ids, ps[pick], pd[pick], k, mp, mode, count_only=count_only)
        assert np.array_equal(orows["count"], cnt[pick]), f"{mode} k={k}: counts differ from the oracle"
        r = {"first_ms": first, "warm_ms_median": warm_ms, "device_total_ms": round(st["total_ms"], 2),
             "batches": st["batches"], "lanes": st["lanes"], "searches": st["searches"], "levels": st["levels"],
             "kernel_launches": st["kernel_launches"], "valid_rows": int((cnt > 0).sum()),
             "ms_by_phase": split(call), "oracle_checked_rows": int(len(pick))}
        if not count_only:
            opaths = okg.shortest_k_groups(n, v, e, ids, ps[pick], pd[pick], k, mp, mode)[0]
            assert opaths == [out[0][i] for i in pick], f"{mode} k={k}: paths differ from the oracle"
            r["paths"] = int(sum(len(p) for p in out[0] if p))
            r["complete_rows"] = int(out[4].sum())
        res["runs"][name] = r
        print(json.dumps({res["graph"]: {name: r}}), flush=True)
    csr.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--max-paths", type=int, default=64)
    ap.add_argument("--warm", type=int, default=2)
    ap.add_argument("--check", type=int, default=2)
    ap.add_argument("--only", nargs="+", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    results = {"card": card(), "graphs": []}
    print(results["card"], flush=True)
    for scale in a.scales:
        results["graphs"].append(run(ctx, scale, a.pairs, a.max_paths, a.warm, a.check, a.only))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
