#!/usr/bin/env python
"""Times the CSR build from key columns (pgq_csr_build_keys) against mapping the keys to rowids on the host first.

    python tools/keys_build_bench.py [--scale 22] [--reps 5] [--host-reps 1] [--out DIR]

Input: R-MAT at --scale (directed, duplicates kept); the vertex table's key column is a random permutation of the
rowids, the edge table's src / dst columns are the keys of the R-MAT endpoints.  Phases, each the median of --reps
runs after one warm-up run of the device phases (the host route, whose searchsorted takes minutes at scale 22, runs
--host-reps times):
    keys_host_call_ms      pgq_csr_build_keys from host columns (the call ends synchronised: host clock)
    keys_h2d_ms            the three key columns to HBM with torch (CUDA events)
    keys_device_call_ms    pgq_csr_build_keys_device on those columns (CUDA events around the call)
    rowids_device_call_ms  pgq_csr_build_device on int32 rowid columns already in HBM: the build pipeline that the
                           key build shares, so keys_device_call_ms - rowids_device_call_ms is the device join
    host_map_ms            numpy: argsort of the vertex keys + searchsorted of src and dst + the match checks
    host_build_call_ms     pgq_csr_build on the mapped rowids (host clock)
The CSRs of the three routes are downloaded once and compared.  Prints one JSON object (and writes
DIR/keys_build_bench.json with --out), with the GPU's name and power limit.

    python tools/keys_build_bench.py --undirected [--scale 22] [--reps 5] [--out DIR]

times the directed and the undirected build (pgq_csr_build_keys_undirected) on the same columns instead:
    {dir,undir}_host_call_ms    from host columns (host clock)
    {dir,undir}_device_call_ms  from the columns in HBM (CUDA events around the call)
    {dir,undir}_rows_call_ms    pgq_csr_build_device on the rows the key build hands on (the directed edge rows; the
                                distinct pairs of both directions), already in HBM: the difference to the device call
                                is the join (and the de-duplication) on the device
The oracle's restatements run once each, for scale (oracle_{dir,undir}_ms); all CSRs are compared with them.
Writes DIR/keys_build_bench_undirected_<scale>.json with --out.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from duckpgq_extension_b200 import datagen, pgq  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": f"unknown ({ex})"}


def host_map(vkey, src_key, dst_key):
    """key -> rowid on the host for unique vertex keys; every edge key must match"""
    order = np.argsort(vkey, kind="stable")
    sk = vkey[order]
    rows = []
    for col in (src_key, dst_key):
        pos = np.searchsorted(sk, col)
        pos_c = np.minimum(pos, len(sk) - 1)
        if not np.all(sk[pos_c] == col):
            raise ValueError("an edge key matches no vertex")
        rows.append(order[pos_c])
    if np.any(sk[1:] == sk[:-1]):
        raise ValueError("duplicate vertex keys")
    return rows[0], rows[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=1, help="timed runs of the host route (minutes each at scale 22)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--undirected", action="store_true", help="time the directed and the undirected key builds")
    args = ap.parse_args()
    if args.undirected:
        return main_undirected(args)

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    n, src, dst = datagen.rmat_edges(args.scale)
    m = len(src)
    vkey = np.random.default_rng(args.scale).permutation(n).astype(np.int64)
    skey, dkey = vkey[src], vkey[dst]
    ctx = pgq.default_context(0)
    d_src32 = torch.from_numpy(src.astype(np.int32)).cuda()
    d_dst32 = torch.from_numpy(dst.astype(np.int32)).cuda()

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    phases = {k: [] for k in ("keys_host_call_ms", "keys_h2d_ms", "keys_device_call_ms", "rowids_device_call_ms",
                              "host_map_ms", "host_build_call_ms")}
    results = {}
    for rep in range(args.reps + 1):
        t = {}
        t0 = time.perf_counter()
        a = pgq.DeviceCSR.build_from_keys(ctx, vkey, skey, dkey)
        t["keys_host_call_ms"] = (time.perf_counter() - t0) * 1e3

        torch.cuda.synchronize()
        e0 = ev()
        cols = [torch.from_numpy(c).cuda(non_blocking=False) for c in (vkey, skey, dkey)]
        e1 = ev()
        b = pgq.DeviceCSR.build_from_keys_device(ctx, n, m, *(c.data_ptr() for c in cols))
        e2 = ev()
        c = pgq.DeviceCSR.build_device(ctx, n, m, d_src32.data_ptr(), d_dst32.data_ptr())
        e3 = ev()
        torch.cuda.synchronize()
        t["keys_h2d_ms"] = e0.elapsed_time(e1)
        t["keys_device_call_ms"] = e1.elapsed_time(e2)
        t["rowids_device_call_ms"] = e2.elapsed_time(e3)

        d = None
        if 1 <= rep <= args.host_reps:  # (pgq_csr_build shares the pipeline the warm-up pass ran)
            t0 = time.perf_counter()
            ms, md = host_map(vkey, skey, dkey)
            t1 = time.perf_counter()
            d = pgq.DeviceCSR.build(ctx, n, ms, md)
            t2 = time.perf_counter()
            t["host_map_ms"] = (t1 - t0) * 1e3
            t["host_build_call_ms"] = (t2 - t1) * 1e3
        if rep == 1:  # check the routes once
            ref = d.download()
            results["keys_host_equals_host_map"] = all(np.array_equal(x, y) for x, y in zip(a.download(), ref))
            results["keys_device_equals_host_map"] = all(np.array_equal(x, y) for x, y in zip(b.download(), ref))
            results["rowids_device_equals_host_map"] = all(np.array_equal(x, y) for x, y in zip(c.download(), ref))
        if rep >= 1:
            for k, x in t.items():
                phases[k].append(x)
        for csr in (a, b, c, d):
            if csr is not None:
                csr.free()
        del cols
        print(f"rep {rep}: " + ", ".join(f"{k} {x:.1f}" for k, x in t.items()), file=sys.stderr, flush=True)
    med = {k: round(float(np.median(v)), 2) for k, v in phases.items()}
    out = {"scale": args.scale, "n": n, "m": m, "reps": args.reps, **gpu_info(), **results, "median_ms": med,
           "device_join_ms": round(med["keys_device_call_ms"] - med["rowids_device_call_ms"], 2),
           "host_route_ms": round(med["host_map_ms"] + med["host_build_call_ms"], 2),
           "all_ms": {k: [round(x, 2) for x in v] for k, v in phases.items()}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "keys_build_bench.json"), "w") as f:
            f.write(line + "\n")


def main_undirected(args):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    from oracle import pgq_oracle_keys as orck
    from oracle import pgq_oracle_keys_undirected as orcu
    info = gpu_info()
    n, src, dst = datagen.rmat_edges(args.scale)
    m = len(src)
    vkey = np.random.default_rng(args.scale).permutation(n).astype(np.int64)
    skey, dkey = vkey[src], vkey[dst]
    ctx = pgq.default_context(0)
    # the rows each build hands to the common pipeline: the edges as they are; the distinct pairs of both directions
    pairs = np.unique(np.concatenate([src.astype(np.int64) * n + dst, dst.astype(np.int64) * n + src]))
    rows = {"dir": (torch.from_numpy(src.astype(np.int32)).cuda(), torch.from_numpy(dst.astype(np.int32)).cuda()),
            "undir": (torch.from_numpy((pairs // n).astype(np.int32)).cuda(),
                      torch.from_numpy((pairs % n).astype(np.int32)).cuda())}
    cols = [torch.from_numpy(c).cuda() for c in (vkey, skey, dkey)]

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    phases = {f"{d}_{k}": [] for d in ("dir", "undir") for k in ("host_call_ms", "device_call_ms", "rows_call_ms")}
    got = {}
    for rep in range(args.reps + 1):
        t = {}
        for d, und in (("dir", False), ("undir", True)):
            t0 = time.perf_counter()
            a = pgq.DeviceCSR.build_from_keys(ctx, vkey, skey, dkey, undirected=und)
            t[f"{d}_host_call_ms"] = (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            e0 = ev()
            b = pgq.DeviceCSR.build_from_keys_device(ctx, n, m, *(c.data_ptr() for c in cols), undirected=und)
            e1 = ev()
            r = pgq.DeviceCSR.build_device(ctx, n, rows[d][0].shape[0], rows[d][0].data_ptr(), rows[d][1].data_ptr())
            e2 = ev()
            torch.cuda.synchronize()
            t[f"{d}_device_call_ms"] = e0.elapsed_time(e1)
            t[f"{d}_rows_call_ms"] = e1.elapsed_time(e2)
            if rep == 0:
                got[d] = (a.download(), b.download())
            for csr in (a, b, r):
                csr.free()
        if rep >= 1:
            for k, x in t.items():
                phases[k].append(x)
        print(f"rep {rep}: " + ", ".join(f"{k} {x:.1f}" for k, x in t.items()), file=sys.stderr, flush=True)
    results = {}
    for d, fn in (("dir", orck.csr_build_keys), ("undir", orcu.csr_build_keys_undirected)):
        t0 = time.perf_counter()
        ref = fn(vkey, skey, dkey)
        results[f"oracle_{d}_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        results[f"{d}_equals_oracle"] = all(all(np.array_equal(x, y) for x, y in zip(g, ref)) for g in got[d])
    med = {k: round(float(np.median(v)), 2) for k, v in phases.items()}
    join = {d: round(med[f"{d}_device_call_ms"] - med[f"{d}_rows_call_ms"], 2) for d in ("dir", "undir")}
    out = {"scale": args.scale, "n": n, "m": m, "undirected_rows": int(pairs.shape[0]), "reps": args.reps, **info,
           **results, "median_ms": med, "join_ms": join,
           "join_share": {d: round(join[d] / med[f"{d}_device_call_ms"], 3) for d in join},
           "all_ms": {k: [round(x, 2) for x in v] for k, v in phases.items()}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"keys_build_bench_undirected_{args.scale}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
