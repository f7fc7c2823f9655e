"""Per-N achieved HBM GB/s from ncu counters (north_star: "throughput ... at 1, 2, 4 and 8 GPUs ... as achieved HBM GB/s from ncu
counters"): reads the `ncu --csv` launch lists tools/gpu_r2_ncu.sh wrote for one rank's share of the step at each N and prints,
per N, kernel time, DRAM bytes (dram__bytes_read.sum + dram__bytes_write.sum) and GB/s, and the step totals.

    python tools/per_n_hbm.py ncu_slab_C2_n{1,2,4,8}.csv > hbm_per_n_C2.txt"""
import collections
import csv
import re
import sys


def load(path):
    rows = list(csv.reader(open(path)))
    hi = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
    H = {n: i for i, n in enumerate(rows[hi])}
    launches = collections.OrderedDict()
    for r in rows[hi + 1:]:
        if len(r) < len(H):
            continue
        d = launches.setdefault(int(r[H["ID"]]), {"kernel": r[H["Kernel Name"]]})
        d[r[H["Metric Name"]]] = float(r[H["Metric Value"]].replace(",", "")) * {"usecond": 1e3, "msecond": 1e6, "second": 1e9, "nsecond": 1.0, "Kbyte": 1e3,
                                                                                 "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0}.get(r[H["Metric Unit"]], 1.0)
    return list(launches.values())


for path in sys.argv[1:]:
    L = load(path)
    names = [re.sub(r"(void |rgs::|\(anonymous namespace\)::)", "", d["kernel"].split("(")[0]) for d in L]
    # the last step's launches: from the last preprocess_forward_kernel on
    start = max(i for i, n in enumerate(names) if n.startswith("preprocess_forward_kernel"))
    tot_t = tot_b = 0.0
    print(f"== {path}")
    print(f"{'kernel':42s} {'time_us':>9s} {'dram_MB':>9s} {'GB/s':>8s}")
    for d, n in list(zip(L, names))[start:]:
        t = d.get("gpu__time_duration.sum", 0.0)
        b = d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
        tot_t += t
        tot_b += b
        print(f"{n[:42]:42s} {t / 1e3:9.1f} {b / 1e6:9.1f} {b / max(t, 1):8.1f}")
    print(f"{'step (kernels of one rank, ncu-serialised)':42s} {tot_t / 1e3:9.1f} {tot_b / 1e6:9.1f} {tot_b / max(tot_t, 1):8.1f}")
