"""Condense `ncu --metrics ... --csv` (tools/gpu_kernel_table.sh) into one row per kernel: the LAST captured launch of each
(steady state), with its share of the step.  usage: python tools/kernel_table.py kernel_table_C2.csv out.csv"""
import collections
import csv
import re
import sys

src, dst = sys.argv[1], sys.argv[2]
rows = list(csv.reader(open(src)))
hi = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
H = {n: i for i, n in enumerate(rows[hi])}
launch = collections.OrderedDict()
for r in rows[hi + 1:]:
    if len(r) < len(H):
        continue
    d = launch.setdefault(int(r[H["ID"]]), {"kernel": r[H["Kernel Name"]], "grid": r[H["Grid Size"]], "block": r[H["Block Size"]]})
    d[r[H["Metric Name"]]] = float(r[H["Metric Value"]].replace(",", "")) * {"usecond": 1e3, "msecond": 1e6, "second": 1e9, "Kbyte": 1e3,
                                                                             "Mbyte": 1e6, "Gbyte": 1e9}.get(r[H["Metric Unit"]], 1.0)
last = collections.OrderedDict()
for d in launch.values():
    head = d["kernel"].split("(")[0] if not d["kernel"].startswith("(") else d["kernel"]
    name = re.sub(r"(void |rgs::|<?unnamed>::|\(anonymous namespace\)::)", "", head)
    d["name"] = name
    last[name] = d
total = sum(d["gpu__time_duration.sum"] for d in last.values())
cols = ["kernel", "grid", "block", "regs", "time_us", "share_pct", "dram_read_MB", "dram_write_MB", "dram_GBps", "dram_pct_peak", "sm_pct_peak",
        "warps_active_pct", "warp_inst_M"]
with open(dst, "w", newline="") as f:
    w = csv.writer(f)
    w.writerow(cols)
    for d in last.values():
        t = d["gpu__time_duration.sum"]
        rd, wr = d.get("dram__bytes_read.sum", 0.0), d.get("dram__bytes_write.sum", 0.0)
        w.writerow([d["name"], d["grid"], d["block"], int(d.get("launch__registers_per_thread", 0)), round(t / 1e3, 2), round(100 * t / total, 1),
                    round(rd / 1e6, 1), round(wr / 1e6, 1), round((rd + wr) / t, 1), round(d.get("dram__throughput.avg.pct_of_peak_sustained_elapsed", 0), 1),
                    round(d.get("sm__throughput.avg.pct_of_peak_sustained_elapsed", 0), 1),
                    round(d.get("sm__warps_active.avg.pct_of_peak_sustained_active", 0), 1), round(d.get("sm__inst_executed.sum", 0) / 1e6, 1)])
print(open(dst).read())
