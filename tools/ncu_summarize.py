#!/usr/bin/env python
"""Summarise Nsight Compute artefacts into small text/JSON files.

  python tools/ncu_summarize.py launches launches.csv launches.txt
  python tools/ncu_summarize.py full prof_k3.ncu-rep k3_k4_full.txt [traffic.json kernel-substr]
"""
import collections
import csv
import json
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__bytes_read.sum.per_second",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__cycles_active.avg",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_bytes.sum", "l1tex__t_bytes.sum",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__shared_mem_per_block_dynamic", "smsp__cycles_active.avg", "sm__cycles_elapsed.max"]


def launches(src, dst):
    with open(src) as f:
        lines = [l for l in f if not l.startswith("==")]
    agg = collections.OrderedDict()
    for row in csv.DictReader(lines):
        try:
            v = float(row["Metric Value"].replace(",", ""))
        except Exception:
            continue
        agg.setdefault((row["Kernel Name"].split("(")[0][:70], row["Grid Size"], row["Block Size"]), []).append(v)
    tot = sum(sum(v) for v in agg.values())
    with open(dst, "w") as out:
        out.write("# ncu --metrics gpu__time_duration.sum --clock-control none (cold-cache, serialised: compare SHARES)\n")
        out.write(f"# {'kernel':70s} {'grid':>12s} {'block':>12s} {'n':>5s} {'avg_ns':>12s} {'share%':>7s}\n")
        for (n, g, b), v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
            out.write(f"{n:72s} {g:>12s} {b:>12s} {len(v):5d} {sum(v)/len(v):12.1f} {100*sum(v)/tot:7.2f}\n")
    print(open(dst).read())


def full(src, dst, traffic_json=None, kernel_sub=None):
    raw = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(dst, "w") as out:
        out.write(f"# ncu --set full --clock-control none, from {src}\n")
        for r in rows[2:]:
            out.write(f"\n== {r[hdr.index('Kernel Name')][:110]}\n")
            for k in KEYS:
                if k in hdr:
                    out.write(f"{k:72s} {r[hdr.index(k)]:>18s} {units[hdr.index(k)]}\n")
    if traffic_json and kernel_sub:
        vals = []
        for r in rows[2:]:
            if kernel_sub in r[hdr.index("Kernel Name")]:
                def val(k):
                    i = hdr.index(k)
                    u = units[i].lower()
                    mul = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)
                    return float(r[i].replace(",", "")) * mul
                vals.append(val("dram__bytes_read.sum") + val("dram__bytes_write.sum"))
        with open(traffic_json, "w") as f:
            json.dump({"kernel": kernel_sub, "launches": len(vals), "traffic_bytes_per_launch": sum(vals) / len(vals),
                       "source": src}, f)
    print(open(dst).read())


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3])
    else:
        full(*sys.argv[2:])
