"""Summarise an ncu report's SASS page: instructions executed grouped by opcode and the hottest SASS regions.
usage: python tools/ncu_hot.py prof_bwd.ncu-rep [top]"""
import collections
import csv
import subprocess
import sys

rep = sys.argv[1]
top = int(sys.argv[2]) if len(sys.argv) > 2 else 25
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hi = next(i for i, r in enumerate(rows) if r and r[0] == "Address")
hdr = rows[hi]
ci, si, ni, sti = hdr.index("Instructions Executed"), hdr.index("Source"), hdr.index("# Samples"), hdr.index("Warp Stall Sampling (All Samples)")
ti = hdr.index("Avg. Predicated-On Threads Executed")
by_op = collections.Counter()
samples_op = collections.Counter()
total = 0
tot_samples = 0
data = []
for r in rows[hi + 1:]:
    if len(r) <= ci:
        continue
    n = int(r[ci] or 0)
    s = int(r[sti] or 0)
    op = r[si].strip().split()[0]
    if op.startswith("@"):
        op = r[si].strip().split()[1]
    op = op.split(".")[0]
    by_op[op] += n
    samples_op[op] += s
    total += n
    tot_samples += s
    data.append((n, s, r[si].strip(), r[ti]))
print(f"total warp instructions {total/1e6:.1f} M, stall samples {tot_samples}")
print("by opcode (instr M, % instr, % samples):")
for op, n in by_op.most_common(top):
    print(f"  {op:10s} {n/1e6:9.1f}  {100*n/total:5.1f}%  {100*samples_op[op]/max(tot_samples,1):5.1f}%")
print("hottest single instructions by stall samples:")
for n, s, src, thr in sorted(data, key=lambda x: -x[1])[:top]:
    print(f"  {s:7d} samples  {n/1e6:8.2f} M  thr {thr:>5s}  {src[:90]}")
