"""SASS evidence: opcode histogram per kernel of librgs_b200.so (cuobjdump -sass).

    python tools/sass_histogram.py > sass_opcodes.txt

Columns: the opcodes the design claims (LDGSTS = cp.async staging, RED/ATOM = gradient scatter, SHFL = warp reduce-scatter,
MUFU = exp / rcp, BAR = CTA barriers) and ones it must NOT contain: FFMA2/FMUL2/FADD2 (packed fp32x2) and UTCMMA / LDTM
(tcgen05), which sm_90a does not have; UTMALDG (TMA), which Hopper has but this path does not use (records are staged with
cp.async); HMMA (the north star rules tensor cores out)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so")
COLS = ["total", "LDGSTS", "LDG", "STG", "LDS", "STS", "FFMA2", "FMUL2", "FADD2", "FFMA", "MUFU", "SHFL", "SEL", "REDG", "ATOMG", "ATOMS", "BAR", "VOTE",
        "UTMALDG", "UTCMMA", "LDTM", "HMMA"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            name = re.sub(r"\(.*", "", name).replace("void ", "")
            cur = kernels.setdefault(name, collections.Counter())
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur is not None:
            op = m.group(1)
            cur["total"] += 1
            cur[op] += 1
    print("SASS opcode histogram of librgs_b200.so (sm_90a), one row per kernel; static instruction counts")
    print(f"{'kernel':78s}" + "".join(f"{c:>8s}" for c in COLS))
    for name, c in kernels.items():
        if not name.startswith("rgs::"):
            continue
        print(f"{name[:78]:78s}" + "".join(f"{c.get(k, 0):8d}" for k in COLS))


if __name__ == "__main__":
    main()
