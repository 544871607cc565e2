#!/usr/bin/env python
"""Time pgq_reachability on R-MAT graphs, 2048 hashed pairs, in its default mode (iterativelength's rows) and with the
reference's 512-lane batches, with the card's name and power limit next to the numbers.

    python tools/reach_bench.py [--scales 20 22] [--warm 5] [--no-oracle]

Per mode: the first call (cold workspace, host clock), the median of warm calls (host clock) and the device time of the
last call (CUDA events, stats total_ms).  For comparison, the path the DuckDB shim took before reachability ran on the
device: download the CSR into the reference's host layout (pgq_csr_download) and run the reference's single-threaded
search, here its loop-for-loop restatement (oracle/pgq_oracle_reach.c).  Every call is checked: both modes give the
same rows, and the restatement's rows and counters equal the reference-batching call's."""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def timed(csr, ps, pd, options, warm):
    t0 = time.perf_counter()
    out, valid, st = csr.reachability(ps, pd, options=options)
    first = (time.perf_counter() - t0) * 1e3
    times = []
    for _ in range(warm):
        t0 = time.perf_counter()
        o2, v2, st = csr.reachability(ps, pd, options=options)
        times.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(o2, out) and np.array_equal(v2, valid)
    return out, st, {"first_call_ms": round(first, 3), "warm_call_ms_median": round(float(np.median(times)), 3),
                     "device_call_ms": round(st["total_ms"], 3), "batches": st["batches"], "levels": st["levels"],
                     "edges_traversed": st["edges_traversed"], "searches": st["searches"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=2048)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    result = {"card": card(), "pairs": a.pairs, "runs": []}
    for scale in a.scales:
        n, s, d = datagen.rmat_edges(scale)
        ps, pd = datagen.hashed_pairs(a.pairs, n)
        csr = pgq.DeviceCSR.build(ctx, n, s, d)
        run = {"scale": scale, "n": n, "m": len(s)}
        out, _, run["default"] = timed(csr, ps, pd, None, a.warm)
        ref_out, st, run["reference_batching"] = timed(csr, ps, pd, pgq.Options(reference_batching=True), a.warm)
        assert np.array_equal(out, ref_out), "the two modes differ"
        run["reachable"] = int(out.sum())
        if not a.no_oracle:
            from oracle import pgq_oracle_reach as orr
            t0 = time.perf_counter()
            v, e, _ = csr.download_ve()
            run["host_download_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            t0 = time.perf_counter()
            eo, ew, ost = orr.reachability(n, v, e, ps, pd)
            run["host_oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            assert np.array_equal(eo, out) and ew.all()
            assert (ost.batches, ost.levels, ost.edges_traversed) == (st["batches"], st["levels"], st["edges_traversed"])
            del v, e
        csr.free()
        result["runs"].append(run)
        print(json.dumps(run), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
