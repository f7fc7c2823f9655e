"""Time simple_knn's distCUDA2 (rgs_knn.cu) on the point clouds the reference initialises from.

Workloads (all seeded):
  blender_100k      scene/dataset_readers.py:303-307: 100 000 uniform points in [-1.3, 1.3]^3
  trimesh_1.2m      dataset_readers.py:233: 1 200 000 draws WITH replacement from a 300 000-point surface cloud (duplicates)
  clustered_1m      a COLMAP-like cloud: Gaussian mixture on 8 centres plus 1 % far outliers
  uniform_10m       the largest bench scenes' splat count

Each output is first checked against scipy.spatial.cKDTree in fp64 (k = 4): |ours - fp64| <= 2e-6 fp64 elementwise and exact
zeros.  Then the median of --reps CUDA-event-timed calls after --warmup calls.  The torch stand-in the fixture generators use
(tests/ref_stubs/simple_knn, cdist + topk in fp64) is timed on the 100 k cloud only: it is O(P^2), so larger clouds are reported
as not run.  Prints one JSON line per workload and one with the card name and power limit, read in the same run.

Usage: python tools/bench_knn.py [--reps 20] [--warmup 3] [--only NAME ...]
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from scipy.spatial import cKDTree  # noqa: E402


def surface_cloud(n, rng):
    """points on three planes and a sphere shell"""
    pick = rng.integers(0, 4, n)
    uv = rng.uniform(-1, 1, (n, 2))
    pts = np.empty((n, 3))
    for axis in range(3):
        m = pick == axis
        pts[m] = np.insert(uv[m], axis, 0.25 * axis - 0.5, axis=1)
    m = pick == 3
    v = rng.normal(size=(m.sum(), 3))
    pts[m] = 0.8 * v / np.linalg.norm(v, axis=1, keepdims=True)
    return pts


def workload(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "blender_100k":
        pts = rng.random((100_000, 3)) * 2.6 - 1.3
    elif name == "trimesh_1.2m":
        verts = surface_cloud(300_000, rng)
        pts = verts[rng.choice(np.arange(len(verts)), 1_200_000)]
    elif name == "clustered_1m":
        P = 1_000_000
        centers = rng.uniform(-2, 2, (8, 3))
        pts = centers[rng.integers(0, 8, P)] + rng.normal(scale=0.03, size=(P, 3))
        out = rng.random(P) < 0.01
        pts[out] = rng.uniform(-60, 60, (out.sum(), 3))
    elif name == "uniform_10m":
        pts = rng.uniform(-1.3, 1.3, (10_000_000, 3))
    else:
        raise ValueError(name)
    return pts.astype(np.float32)


WORKLOADS = ["blender_100k", "trimesh_1.2m", "clustered_1m", "uniform_10m"]


def verify(pts, ours):
    p = pts.astype(np.float64)
    d, _ = cKDTree(p).query(p, k=4, workers=-1)
    ref = (d[:, 1:] ** 2).mean(axis=1)
    err = np.abs(ours.astype(np.float64) - ref)
    ok = bool(np.all(err <= 2e-6 * ref) and np.all(ours[ref == 0.0] == 0.0))
    rel = float(np.max(err / np.where(ref > 0, ref, 1.0)))
    return {"ok": ok, "worst_rel_err": rel, "zeros": int((ref == 0.0).sum())}


def time_calls(fn, x, warmup, reps):
    for _ in range(warmup):
        fn(x)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(x)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "reps": reps}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", nargs="*", choices=WORKLOADS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_knn needs a CUDA device: distCUDA2 has no CPU path")
    from simple_knn._C import distCUDA2

    import bench
    dev = torch.cuda.current_device()
    vis = os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",")
    nvml_index = int(vis[dev]) if dev < len(vis) and vis[dev].strip().isdigit() else dev
    print(json.dumps({"device": bench.device_info(dev, nvml_index)}), flush=True)

    spec = importlib.util.spec_from_file_location("standin_knn", os.path.join(ROOT, "tests", "ref_stubs", "simple_knn", "_C.py"))
    standin = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(standin)

    for name in args.only or WORKLOADS:
        pts = workload(name)
        x = torch.from_numpy(pts).cuda()
        rec = {"workload": name, "points": len(pts), "verify_vs_ckdtree_fp64": verify(pts, distCUDA2(x).cpu().numpy())}
        rec["distCUDA2"] = time_calls(distCUDA2, x, args.warmup, args.reps)
        if name == "blender_100k":
            rec["torch_standin"] = time_calls(standin.distCUDA2, x, 1, args.reps)
        else:
            rec["torch_standin"] = "not run: O(P^2)"
        print(json.dumps(rec), flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
