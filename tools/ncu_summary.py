#!/usr/bin/env python
"""Turn ncu outputs into small text summaries.

    python tools/ncu_summary.py launches launches.csv            # per-kernel totals and shares
    python tools/ncu_summary.py sass prof.ncu-rep [kernel-index] # instruction counts per 40-instruction block
    python tools/ncu_summary.py metrics prof.ncu-rep             # a handful of headline metrics

`launches.csv` comes from  ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file ... ;
`prof.ncu-rep` from         ncu --set full --clock-control none --import-source on -k regex:<kernel> ...
The sass view needs the code to be compiled with -lineinfo (build.py does)."""
import collections
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__grid_size",
        "launch__registers_per_thread", "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "l1tex__t_sector_hit_rate.pct",
        "lts__t_sector_hit_rate.pct", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def launches(path):
    lines = open(path).read().splitlines()
    start = next(i for i, ln in enumerate(lines) if ln.startswith('"ID"'))
    agg = collections.OrderedDict()
    rows = list(csv.DictReader(lines[start:]))
    for r in rows:
        name = r["Kernel Name"].split("(")[0]
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += float(r["Metric Value"]) / 1e6
    total = sum(a[1] for a in agg.values())
    print("kernel,launches,total_ms,share_pct")
    for name, (c, t) in sorted(agg.items(), key=lambda x: -x[1][1]):
        print("%s,%d,%.3f,%.1f" % (name, c, t, 100 * t / total))
    print("TOTAL,%d,%.3f,100.0" % (len(rows), total))


def _ncu(rep, *extra):
    return subprocess.run(["ncu", "-i", rep] + list(extra), capture_output=True, text=True).stdout


def metrics(rep):
    rows = list(csv.reader(_ncu(rep, "--page", "raw", "--csv").splitlines()))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        print("---", r[hdr.index("Kernel Name")][:80])
        for k in KEYS:
            if k in hdr:
                print("%-72s %s %s" % (k, r[hdr.index(k)], units[hdr.index(k)]))


def sass(rep, which=0):
    rows = list(csv.reader(_ncu(rep, "--page", "source", "--csv", "--print-source", "sass").splitlines()))
    kernels, cur = [], None
    for r in rows:
        if r and r[0] == "Kernel Name":
            cur = {"name": r[1], "rows": []}
            kernels.append(cur)
        elif cur is not None and r and r[0] == "Address":
            cur["hdr"] = r
        elif cur is not None and r and r[0].startswith("0x"):
            cur["rows"].append(r)
    k = kernels[which]
    h = k["hdr"]
    ii, it = h.index("Instructions Executed"), h.index("Avg. Threads Executed")
    total = sum(int(r[ii]) for r in k["rows"])
    print(k["name"][:100], "warp instructions:", total)
    for a in range(0, len(k["rows"]), 40):
        seg = k["rows"][a:a + 40]
        n = sum(int(r[ii]) for r in seg)
        if n < 0.004 * total:
            continue
        thr = sum(int(r[ii]) * float(r[it]) for r in seg) / max(1, n)
        ops = collections.Counter()
        for r in seg:
            t = r[1].split()
            ops[t[1] if t[0].startswith("@") else t[0]] += int(r[ii])
        print("%5d %5.1f%% threads/instr %4.1f  %s" % (a, 100 * n / total, thr, ops.most_common(5)))


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "launches":
        launches(sys.argv[2])
    elif cmd == "metrics":
        metrics(sys.argv[2])
    elif cmd == "sass":
        sass(sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else 0)
