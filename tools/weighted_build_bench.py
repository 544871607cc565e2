#!/usr/bin/env python
"""Times the weighted device CSR builds against the chunked create_csr_edge protocol.

    python tools/weighted_build_bench.py [--scale 22] [--reps 3] [--out DIR]

Input: R-MAT at --scale (directed, duplicates kept) with random weights, once BIGINT (1 .. 2^20) and once DOUBLE
((0, 100)); the vertex table's key column is a random permutation of the rowids, the edge table's src / dst columns
are the keys of the R-MAT endpoints.  Phases per weight type, each the median of --reps runs after one warm-up run:
    chunked_2048_ms          pgq_csr_create + add_vertex_counts + add_edges_weighted in 2048-row chunks + finalize
                             (host clock: the protocol a DuckDB DataChunk stream drives)
    build_host_call_ms       pgq_csr_build_weighted from host columns (host clock; the call ends synchronised)
    build_device_call_ms     pgq_csr_build_device_weighted on int32 rowids and the weights in HBM (CUDA events)
    keys_device_call_ms      pgq_csr_build_keys_weighted_device on the key and weight columns in HBM (CUDA events)
    keys_device_unweighted_call_ms   pgq_csr_build_keys_device on the same key columns: keys_device_call_ms minus this
                             is what the weights cost the key build
The CSRs and weight columns of the four weighted routes are downloaded once and compared.  Prints one JSON object
(and writes DIR/weighted_build_bench_<scale>.json with --out), with the GPU's name and power limit.
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

CHUNK = 2048


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": f"unknown ({ex})"}


def chunked(ctx, n, src, dst, eid, w):
    csr = pgq.DeviceCSR.create(ctx, n)
    csr.add_vertex_counts(np.arange(n), np.bincount(src, minlength=n))
    m = len(src)
    for o in range(0, m, CHUNK):
        csr.add_edges(m, m, src[o:o + CHUNK], dst[o:o + CHUNK], eid[o:o + CHUNK], w[o:o + CHUNK])
    csr.finalize()
    return csr


def snapshot(csr):
    v, e, ids = csr.download()
    w = csr.download_weights()
    return v, e, ids, w.view(np.int64), csr.weight_type()


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def run(ctx, torch, n, src, dst, vkey, w, reps):
    m = len(src)
    wt = 2 if w.dtype.kind == "f" else 1
    eid = np.arange(m, dtype=np.int64)
    skey, dkey = vkey[src], vkey[dst]
    d_src, d_dst = (torch.from_numpy(x.astype(np.int32)).cuda() for x in (src, dst))
    d_vkey, d_skey, d_dkey, d_w = (torch.from_numpy(x).cuda() for x in (vkey, skey, dkey, w))

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    phases = {k: [] for k in ("chunked_2048_ms", "build_host_call_ms", "build_device_call_ms", "keys_device_call_ms",
                              "keys_device_unweighted_call_ms")}
    equal = None
    for rep in range(reps + 1):
        t = {}
        t0 = time.perf_counter()
        a = chunked(ctx, n, src, dst, eid, w)
        t1 = time.perf_counter()
        b = pgq.DeviceCSR.build(ctx, n, src, dst, eid, weight=w)
        t2 = time.perf_counter()
        t["chunked_2048_ms"] = (t1 - t0) * 1e3
        t["build_host_call_ms"] = (t2 - t1) * 1e3
        torch.cuda.synchronize()
        e0 = ev()
        c = pgq.DeviceCSR.build_device(ctx, n, m, d_src.data_ptr(), d_dst.data_ptr(), 0, d_weight=d_w.data_ptr(),
                                       weight_type=wt)
        e1 = ev()
        d = pgq.DeviceCSR.build_from_keys_device(ctx, n, m, d_vkey.data_ptr(), d_skey.data_ptr(), d_dkey.data_ptr(),
                                                 d_weight=d_w.data_ptr(), weight_type=wt)
        e2 = ev()
        u = pgq.DeviceCSR.build_from_keys_device(ctx, n, m, d_vkey.data_ptr(), d_skey.data_ptr(), d_dkey.data_ptr())
        e3 = ev()
        torch.cuda.synchronize()
        t["build_device_call_ms"] = e0.elapsed_time(e1)
        t["keys_device_call_ms"] = e1.elapsed_time(e2)
        t["keys_device_unweighted_call_ms"] = e2.elapsed_time(e3)
        if rep == 0:  # every route holds the rows in the same order within a source row: compare position by position
            ref = snapshot(a)
            equal = {"build": same(snapshot(b), ref), "build_device": same(snapshot(c), ref),
                     "keys_device": same(snapshot(d), ref),
                     "keys_device_unweighted": same(u.download(), ref[:3])}
        else:
            for k, x in t.items():
                phases[k].append(x)
        for csr in (a, b, c, d, u):
            csr.free()
        print(f"w_type {wt} rep {rep}: " + ", ".join(f"{k} {x:.1f}" for k, x in t.items()), file=sys.stderr,
              flush=True)
    med = {k: round(float(np.median(v)), 2) for k, v in phases.items()}
    return {"w_type": wt, "routes_equal": equal, "all_routes_equal": all(equal.values()), "median_ms": med,
            "weights_cost_keys_ms": round(med["keys_device_call_ms"] - med["keys_device_unweighted_call_ms"], 2),
            "all_ms": {k: [round(x, 2) for x in v] for k, v in phases.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs the GPU")
    info = gpu_info()
    n, src, dst = datagen.rmat_edges(args.scale)
    src, dst = src.astype(np.int64), dst.astype(np.int64)
    m = len(src)
    rng = np.random.default_rng(args.scale)
    vkey = rng.permutation(n).astype(np.int64)
    ctx = pgq.default_context(0)
    results = [run(ctx, torch, n, src, dst, vkey, rng.integers(1, 1 << 20, m), args.reps),
               run(ctx, torch, n, src, dst, vkey, rng.random(m) * 100.0, args.reps)]
    out = {"scale": args.scale, "n": n, "m": m, "reps": args.reps, **info,
           "all_routes_equal": all(r["all_routes_equal"] for r in results), "bigint": results[0],
           "double": results[1]}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"weighted_build_bench_{args.scale}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
