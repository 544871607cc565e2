#!/usr/bin/env python
"""Where the time of a bench step goes (development aid): the bench's workload -- R-MAT-22, 1024 hashed pairs per
step, steps 3..22 of its pair stream, iterativelength_device on the current stream with default options -- run under
torch.profiler with CUDA activities.  Per step it reports the call time, the device time of every kernel by name and
of the memsets / copies, and the idle time of the device between them (the step's span minus the union of its busy
intervals over both batch streams).

    python tools/step_breakdown.py [--out DIR] [--scale 22] [--pairs 1024] [--warmup 3] [--steps 20]

Prints one table (milliseconds per step, averaged over the steps); with --out it also writes DIR/step_breakdown.json
with the per-step numbers.  Run it on its own: tracing slows the host, so its call times are not the bench's.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from duckpgq_extension_b200 import datagen  # noqa: E402

# kernels that expand a frontier; everything else on the device is the level loop's overhead
EXPANSION = ("k_pull_fused", "k_expand_push", "k_tail")


def short_name(name: str) -> str:
    """'void k_pull_fused<4, false>(PullArgs<4>)' -> 'k_pull_fused<4, false>'"""
    name = re.sub(r"^void\s+", "", name)
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def base_name(name: str) -> str:
    return short_name(name).split("<")[0]


def union_length(intervals) -> float:
    total, end = 0.0, -np.inf
    for a, b in sorted(intervals):
        if b <= end:
            continue
        total += b - max(a, end)
        end = b
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--pairs", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    from duckpgq_extension_b200 import pgq

    if not torch.cuda.is_available():
        raise SystemExit("step_breakdown.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    n, src, dst = datagen.rmat_edges_cached(args.scale)
    ctx = pgq.Context(0)
    csr = pgq.DeviceCSR.build(ctx, n, src, dst)
    P, nsteps = args.pairs, args.warmup + args.steps
    ps_all, pd_all = datagen.hashed_pairs(P * nsteps, n)
    ps_all, pd_all = ps_all.reshape(nsteps, P), pd_all.reshape(nsteps, P)
    d_src = torch.from_numpy(ps_all).to(dev)
    d_dst = torch.from_numpy(pd_all).to(dev)
    d_len = torch.empty(P, dtype=torch.int64, device=dev)
    d_val = torch.empty(P, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream()
    opts = pgq.Options()

    def step(i):
        return csr.iterativelength_device(d_src[i].data_ptr(), d_dst[i].data_ptr(), P, d_len.data_ptr(),
                                          d_val.data_ptr(), 0, stream.cuda_stream, opts)

    # as bench.py: a call with more searches than one batch holds creates the second workspace before the window
    csr.iterativelength(ps_all[0], pd_all[0], None, pgq.Options(256, 0, 0, True))
    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()

    stats = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(args.warmup, nsteps):
            with record_function(f"step_{i}"):  # (the synchronize inside: work queued after the call's last wait counts)
                stats.append(step(i))
                torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    events = trace["traceEvents"] if isinstance(trace, dict) else trace
    windows = {}
    for e in events:
        if e.get("ph") == "X" and e.get("cat") == "user_annotation" and str(e.get("name", "")).startswith("step_"):
            windows[int(e["name"][5:])] = (float(e["ts"]), float(e["ts"]) + float(e["dur"]))
    device = [e for e in events if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]

    rows = []
    for k, i in enumerate(range(args.warmup, nsteps)):
        lo, hi = windows[i]
        mine = [e for e in device if lo <= float(e["ts"]) <= hi]
        per = {}
        busy = []
        for e in mine:
            a, d = float(e["ts"]), float(e["dur"])
            busy.append((a, a + d))
            name = short_name(e["name"]) if e["cat"] == "kernel" else e["cat"]
            t = per.setdefault(name, [0, 0.0])
            t[0] += 1
            t[1] += d / 1e3
        span = (max(b for _, b in busy) - min(a for a, _ in busy)) / 1e3 if busy else 0.0
        st = stats[k]
        expansion = sum(v[1] for nm, v in per.items() if base_name(nm) in EXPANSION)
        rows.append({"step": i, "call_ms": st["total_ms"], "device_span_ms": span,
                     "busy_ms": union_length(busy) / 1e3, "idle_ms": span - union_length(busy) / 1e3,
                     "expansion_ms": expansion, "kernels": {nm: {"count": c, "ms": ms} for nm, (c, ms) in per.items()},
                     "searches": st["searches"], "batches": st["batches"], "levels": st["levels"],
                     "pull_levels": st["pull_levels"], "push_levels": st["push_levels"],
                     "kernel_launches": st["kernel_launches"]})

    props = torch.cuda.get_device_properties(0)
    steps = len(rows)
    mean = lambda key: sum(r[key] for r in rows) / steps  # noqa: E731
    names = sorted({nm for r in rows for nm in r["kernels"]},
                   key=lambda nm: -sum(r["kernels"].get(nm, {"ms": 0})["ms"] for r in rows))
    print(f"device: {props.name}; {steps} steps (R-MAT-{args.scale}, {P} pairs per step, steps "
          f"{args.warmup}..{nsteps - 1}); milliseconds per step, mean over the steps")
    print(f"  call (CUDA events inside the call) {mean('call_ms'):8.4f}")
    print(f"  device span of the step            {mean('device_span_ms'):8.4f}")
    print(f"  device busy (union, both streams)   {mean('busy_ms'):8.4f}")
    print(f"  device idle between kernels         {mean('idle_ms'):8.4f}")
    print(f"  expansion kernels ({', '.join(EXPANSION)}) {mean('expansion_ms'):8.4f}")
    print(f"  searches {mean('searches'):.1f}, batches {mean('batches'):.2f}, levels {mean('levels'):.2f} "
          f"(pull {mean('pull_levels'):.2f}, push {mean('push_levels'):.2f}), launches {mean('kernel_launches'):.1f}")
    print(f"  {'kernel / activity':<60s} {'count':>7s} {'ms':>8s} {'share':>7s}")
    call = mean("call_ms")
    for nm in names:
        c = sum(r["kernels"].get(nm, {"count": 0})["count"] for r in rows) / steps
        ms = sum(r["kernels"].get(nm, {"ms": 0.0})["ms"] for r in rows) / steps
        print(f"  {nm[:60]:<60s} {c:7.2f} {ms:8.4f} {100 * ms / call:6.1f}%")
    outside = call - mean("expansion_ms")
    print(f"  outside the expansion kernels: {outside:.4f} ms = {100 * outside / call:.1f}% of the call")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_breakdown.json"), "w") as f:
            json.dump({"device": props.name, "scale": args.scale, "pairs": P, "steps": rows}, f, indent=1)


if __name__ == "__main__":
    main()
