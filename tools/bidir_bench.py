#!/usr/bin/env python
"""Time pgq_iterativelength_bidirectional: the first call (cold workspace) and the median of warm calls, 2048 hashed pairs
on R-MAT graphs, directed and undirected, with the card's name and power limit next to the numbers.

    python tools/bidir_bench.py [--scales 20 22] [--warm 5] [--oracle]

Checks every call: on undirected graphs the rows must equal iterativelength's; --oracle also runs the restatement
(oracle/pgq_oracle_bidir.c, single-threaded CPU: minutes at these sizes) and compares rows and counters.  Also reported:
the time of clearing the two mask sets a batch starts with (6 x n x 64 B, the same memset on a torch buffer)."""
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


def clear_ms(n, reps=10):
    buf = torch.empty(6 * n * 64, dtype=torch.uint8, device="cuda:0")
    buf.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        buf.zero_()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--pairs", type=int, default=2048)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing to measure")
    ctx = pgq.default_context(0)
    result = {"card": card(), "pairs": a.pairs, "runs": []}
    for scale in a.scales:
        n, s, d = datagen.rmat_edges(scale)
        ps, pd = datagen.hashed_pairs(a.pairs, n)
        for undirected in (False, True):
            es, ed = (np.concatenate([s, d]), np.concatenate([d, s])) if undirected else (s, d)
            csr = pgq.DeviceCSR.build(ctx, n, es, ed)
            t0 = time.perf_counter()
            out, valid, st = csr.iterativelengthbidirectional(ps, pd)
            first = (time.perf_counter() - t0) * 1e3
            warm = []
            for _ in range(a.warm):
                t0 = time.perf_counter()
                o2, v2, _ = csr.iterativelengthbidirectional(ps, pd)
                warm.append((time.perf_counter() - t0) * 1e3)
                assert np.array_equal(o2, out) and np.array_equal(v2, valid)
            run = {"scale": scale, "undirected": undirected, "n": n, "m": len(es), "first_call_ms": round(first, 3),
                   "warm_call_ms_median": round(float(np.median(warm)), 3), "device_call_ms": round(st["total_ms"], 3),
                   "batches": st["batches"], "iterations": st["levels"], "edges_traversed": st["edges_traversed"],
                   "met": int(valid.sum()), "mask_clear_ms_per_batch": round(clear_ms(n), 3)}
            if undirected:
                lo, lv, _ = csr.iterativelength(ps, pd)
                assert np.array_equal(lo, out) and np.array_equal(lv, valid), "undirected: differs from iterativelength"
            if a.oracle:
                from oracle import pgq_oracle_bidir as orb
                v, e, _ = csr.download()
                t0 = time.perf_counter()
                eo, ev, ost = orb.iterativelengthbidirectional(n, v, e, ps, pd)
                run["oracle_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                assert np.array_equal(eo, out) and np.array_equal(ev, valid)
                assert (ost.batches, ost.iterations, ost.edges_traversed) == (st["batches"], st["levels"],
                                                                              st["edges_traversed"])
            csr.free()
            result["runs"].append(run)
            print(json.dumps(run), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
