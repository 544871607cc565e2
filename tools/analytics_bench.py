#!/usr/bin/env python
"""Times local_clustering_coefficient, pagerank and weakly_connected_component on the device CSR and checks them
against the CPU restatement of the reference (oracle/pgq_oracle.c, single-threaded, as the reference runs them).

    python tools/analytics_bench.py [--scales 20,22] [--lcc-rows 65536] [--oracle-lcc-rows 1024] [--out DIR]

Workloads, per R-MAT scale: PageRank on the directed graph, WCC on the undirected graph (both directions of every
distinct non-loop edge), LCC on a fixed sample of --lcc-rows vertices of the undirected graph.  For PageRank and WCC
the first call computes the whole vector (device time from CUDA events, call time from the host clock around the
call, which returns after a device synchronise); a second call is answered from the cached host copy.  The oracle
runs on the full vectors for PageRank and WCC; its LCC resets a bitmap of n + 2 bytes per row, as the reference does,
so it is timed and checked on the first --oracle-lcc-rows rows of the sample only.  Prints one JSON object (and
writes DIR/analytics_bench.json with --out), with the GPU's name and power limit.
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
from oracle import pgq_oracle as orc  # noqa: E402


def undirected(n, src, dst):
    """both directions of every distinct non-loop edge (as tests/golden/make_golden_next4.undirected)"""
    keep = src != dst
    a, b = np.minimum(src[keep], dst[keep]), np.maximum(src[keep], dst[keep])
    key = np.unique(a.astype(np.int64) * n + b)
    a, b = key // n, key % n
    return np.concatenate([a, b]), np.concatenate([b, a])


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": f"unknown ({ex})"}


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t0) * 1e3


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def run_scale(ctx, scale: int, lcc_rows: int, oracle_lcc_rows: int) -> dict:
    n, s, d = datagen.rmat_edges(scale)
    s, d = s.astype(np.int64), d.astype(np.int64)
    us, ud = undirected(n, s, d)
    res = {"scale": scale, "n": n, "m_directed": int(len(s)), "m_undirected": int(len(us))}
    ids = np.arange(n + 2, dtype=np.int64)

    # ---- PageRank, directed
    csr = pgq.DeviceCSR.build(ctx, n, s, d)
    (pr, _, iters, st), ms = timed(lambda: csr.pagerank(ids))
    (_, _, _, st2), ms2 = timed(lambda: csr.pagerank(ids))
    csr.free()
    v, e, _ = orc.csr_build(n, s, d)
    (opr, _, oiters), oms = timed(lambda: orc.pagerank(n, v, e, ids))
    del v, e
    res["pagerank"] = {
        "iterations": iters, "first_call_device_ms": st["total_ms"], "first_call_ms": ms,
        "dangling_fold_ms_per_iteration": st["expand_ms"] / max(iters, 1), "cached_call_ms": ms2,
        "cached_call_device_ms": st2["total_ms"], "oracle_ms": oms,
        "equal": bool(iters == oiters and np.array_equal(bits(pr), bits(opr)))}

    # ---- WCC and LCC, undirected
    csr = pgq.DeviceCSR.build(ctx, n, us, ud)
    (w, _, st), ms = timed(lambda: csr.weakly_connected_component(ids))
    (_, _, st2), ms2 = timed(lambda: csr.weakly_connected_component(ids))
    sample = np.sort(np.random.default_rng(scale).choice(n, size=min(lcc_rows, n), replace=False))
    csr.local_clustering_coefficient(sample[:256])  # warm-up of the LCC kernels
    (lcc, _, lst), lms = timed(lambda: csr.local_clustering_coefficient(sample))
    csr.free()
    v, e, _ = orc.csr_build(n, us, ud)
    (ow, _), oms = timed(lambda: orc.weakly_connected_component(n, v, e, ids))
    (olcc, _), olms = timed(lambda: orc.local_clustering_coefficient(n, v, e, sample[:oracle_lcc_rows]))
    res["wcc"] = {
        "rounds": st["levels"], "first_call_device_ms": st["total_ms"], "first_call_ms": ms, "cached_call_ms": ms2,
        "cached_call_device_ms": st2["total_ms"], "components": int(len(np.unique(w))), "oracle_ms": oms,
        "equal": bool(np.array_equal(w, ow))}
    res["lcc"] = {
        "rows": int(len(sample)), "call_device_ms": lst["total_ms"], "call_ms": lms,
        "oracle_rows": int(min(oracle_lcc_rows, len(sample))), "oracle_ms": olms,
        "equal_on_oracle_rows": bool(np.array_equal(bits(lcc[:oracle_lcc_rows]), bits(olcc)))}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="20,22")
    ap.add_argument("--lcc-rows", type=int, default=65536)
    ap.add_argument("--oracle-lcc-rows", type=int, default=1024)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if pgq.device_count() < 1:
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    ctx = pgq.default_context(0)
    out = dict(gpu_info())
    out["results"] = [run_scale(ctx, int(x), a.lcc_rows, a.oracle_lcc_rows) for x in a.scales.split(",")]
    txt = json.dumps(out, indent=1)
    print(txt)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "analytics_bench.json"), "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
