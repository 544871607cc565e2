#!/usr/bin/env python
"""Turn Nsight Compute artefacts into small text summaries.

  python tools/profile_summary.py launches <launches.csv> <out.md> [which]   per-kernel totals of ONE path-function
        call of a launch list (which = index of the call, default -1 = last; bench.py ends with two calls in the
        reference's batch composition, so the last timed step is which = -3)
  python tools/profile_summary.py full <report.ncu-rep> <out.md> [<traffic.json>]   key metrics of a --set full capture
"""
import collections
import csv
import json
import subprocess
import sys


def launches(path, out, which=-1):
    lines = [l for l in open(path) if not l.startswith("==")]
    rows = list(csv.DictReader(lines))
    names = [r["Kernel Name"] for r in rows]
    # one path-function call = from its k_assign to the next one (or the end)
    starts = [i for i, n in enumerate(names) if "k_assign" in n]
    lo = starts[which] if starts else 0
    hi = starts[which + 1] if (starts and which < -1) else len(rows)
    agg = collections.OrderedDict()
    for r in rows[lo:hi]:
        v = float(r["Metric Value"].replace(",", "")) * {"ns": 1e-3, "us": 1.0, "ms": 1e3}.get(r["Metric Unit"], 1.0)
        a = agg.setdefault(r["Kernel Name"].split("(")[0], [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(a[1] for a in agg.values())
    with open(out, "w") as f:
        f.write(f"# ncu launch list ({path}), path-function call #{which} of the run: {hi - lo} launches, {tot:.1f} us in kernels\n\n")
        f.write("(gpu__time_duration.sum, --clock-control none; cold-cache, serialised: compare SHARES)\n\n")
        f.write("| kernel | launches | total us | avg us | share |\n|---|---|---|---|---|\n")
        for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{k}` | {c} | {t:.1f} | {t / c:.1f} | {100 * t / tot:.1f}% |\n")


WANT = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__registers_per_thread",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sectors.sum", "lts__t_sector_hit_rate.pct",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__t_sector_hit_rate.pct",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
]


def full(rep, out, traffic=None):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    name_i = hdr.index("Kernel Name")
    with open(out, "w") as f:
        f.write(f"# ncu --set full --clock-control none: {rep}\n\n")
        f.write("kernel: " + data[0][name_i].split("(")[0] + f"   ({len(data)} launches captured)\n\n| metric | unit | " +
                " | ".join(f"launch {i}" for i in range(len(data))) + " |\n|---|---|" + "---|" * len(data) + "\n")
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                f.write(f"| {w} | {units[i]} | " + " | ".join(d[i] for d in data) + " |\n")
    if traffic:
        ir, iw = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        per = [float(d[ir]) * scale[units[ir]] + float(d[iw]) * scale[units[iw]] for d in data]
        json.dump({"kernel": data[0][name_i].split("(")[0], "dram_bytes_per_launch": sum(per) / len(per),
                   "launches": len(per), "source": rep}, open(traffic, "w"), indent=1)


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3], int(sys.argv[4]) if len(sys.argv) > 4 else -1)
    else:
        full(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else None)
