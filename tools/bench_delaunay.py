"""Time tetra.delaunay on the tetra points of seeded synthetic Gaussians, with scipy.spatial.Delaunay beside it.

    python tools/bench_delaunay.py [--gaussians 100000,1000000,3000000] [--scipy 50000,150000] [--check]

Per size: the median of 3 timed calls after one warm-up, the rounds, the cells, the largest slot cavity, the overflowed
cavities and the peak device memory.  --check runs the validity checker `check_gpu` of tests/delaunay_exact.py on the
1 M Gaussian size (or the nearest below): every cell positive and every interior face locally Delaunay in torch fp64
with a filter bound, the exact model on what the bound cannot decide, and each face in at most two cells.  One JSON line per
size; the GPU name and power limit come first.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")]

from rade_gs_b200 import tetra  # noqa: E402


def gaussians(P, seed=0):
    g = np.random.default_rng(seed)
    xyz = g.normal(size=(P, 3)) * 2
    s = np.exp(g.normal(-4.0, 0.6, size=(P, 3))) * 3
    q = g.normal(size=(P, 4))
    t = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda")  # noqa: E731
    pts, _ = tetra.tetra_points(t(xyz), t(np.log(s)).exp(), t(q))
    return pts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", default="100000,1000000,3000000")
    ap.add_argument("--scipy", default="50000,150000")
    ap.add_argument("--check", action="store_true")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": q}), flush=True)
    sizes = [int(x) for x in a.gaussians.split(",") if x]
    check_at = max([s for s in sizes if s <= 1_000_000] or sizes[:1])
    for P in sizes:
        pts = gaussians(P)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        tetra.delaunay(pts)
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            cells, st = tetra.delaunay(pts, return_stats=True)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        row = {"gaussians": P, "points": int(pts.shape[0]), "seconds": sorted(times)[1], "cells": int(cells.shape[0]),
               "cells_per_point": cells.shape[0] / pts.shape[0], "peak_gb": torch.cuda.max_memory_allocated() / 1e9, **st}
        print(json.dumps(row), flush=True)
        if a.check and P == check_at:
            import delaunay_exact as dx
            print(json.dumps({"gaussians": P, "check": dx.check_gpu(pts, cells)}), flush=True)
        del cells, pts
        torch.cuda.empty_cache()
    for P in [int(x) for x in a.scipy.split(",") if x]:
        from scipy.spatial import Delaunay
        pts = gaussians(P).cpu().double().numpy()
        t0 = time.perf_counter()
        d = Delaunay(pts)
        print(json.dumps({"scipy_gaussians": P, "points": len(pts), "seconds": time.perf_counter() - t0, "cells": int(len(d.simplices))}), flush=True)


if __name__ == "__main__":
    main()
