"""Per-stage timing of the unbounded-scene mesh (rade_gs_b200.unbounded) on the GPU, with the reference's eager torch
expressions (tests/unbounded_scenes.torch_tsdf, chunks of 256^3 samples as the reference splits them) as the comparison.
Prints the card's name and power limit, then one JSON line per workload.

Workloads: --views (default 50 and 300) analytic views at --width x --height (default 1240x820) of a unit sphere, a ground
plane and a far background sphere, at --resolution (default 512 and 1024).  Per stage, the median of CUDA-event times:
normalisation (host, including the one norm kernel and numpy's quantile), SDF per crop, marching cubes per crop, merge,
colours and cleanup (post_process_mesh).  Also sample-view evaluations per second of the SDF and its algorithmic bytes
over time (each sample writes 4 bytes and reads 4 bilinear corners of every view it projects into; the bytes count the
depth-map reads at 16 per in-view sample-view, an upper bound on DRAM traffic since most hit L1/L2).  The eager
comparison runs at 512 and the smallest view count only (--eager-views); other sizes print "not run".

Usage:  python tools/bench_unbounded.py [--views 50 300] [--resolution 512 1024] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

DEV = "cuda:0"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


class Timer:
    def __init__(self):
        self.t = {}

    def run(self, name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        self.t.setdefault(name, []).append(a.elapsed_time(b))
        return out

    def median(self, name):
        return float(np.median(self.t[name])) if name in self.t else None


def one_run(tm, U, ub, d, c, wv, fp, xyz, resolution):
    t0 = time.perf_counter()
    center, radius = ub.normalization(wv)
    R = ub.scene_bound(xyz, center, radius)
    torch.cuda.synchronize()
    tm.t.setdefault("normalisation", []).append(1e3 * (time.perf_counter() - t0))
    cl = [float(x) for x in center]
    trunc = float(np.float32(5 * (radius * 2 / resolution)))
    verts, tris, base = [], [], 0
    for lo, sp, axes in ub.crop_axes(R, resolution, ub.CROP):
        xs, ys, zs = (torch.from_numpy(a).to(DEV) for a in axes)
        sdf = tm.run("sdf_per_crop", lambda: U.sdf(xs, ys, zs, fp, d, cl, radius, trunc))
        v, t = tm.run("mcubes_per_crop", lambda: U.mcubes(sdf, [float(x) for x in lo], [float(x) for x in sp]))
        del sdf
        if t.shape[0]:
            verts.append(v)
            tris.append(t + base)
            base += v.shape[0]
    mv, mt = tm.run("merge", lambda: U.merge(torch.cat(verts), torch.cat(tris)))
    world, _ = U.contract(mv, cl, radius, True, ub.MAX_RANGE)
    col = tm.run("colors", lambda: U.colors(world, fp, d, c, trunc))
    from rade_gs_b200.tsdf import TriangleMesh
    mesh = TriangleMesh(world, mt, col)
    clean = tm.run("cleanup", lambda: ub.post_process_mesh(mesh, 1000))
    return center, radius, R, mesh, clean


def in_view_fraction(U, ub, fp, d, center, radius, R, n=64):
    """Fraction of (sample, view) pairs that project into the view, on an n^3 grid over [-R, R]^3 (the bytes estimate)."""
    x = np.linspace(-R, R, n).astype(np.float32)
    s = torch.from_numpy(np.stack(np.meshgrid(x, x, x, indexing="ij"), -1).reshape(-1, 3)).to(DEV)
    y = ub.uncontract(s) * float(np.float32(radius)) + torch.tensor(np.asarray(center, np.float32), device=DEV)
    h = torch.cat([y, torch.ones_like(y[:, :1])], 1) @ fp        # [V, N, 4]
    pix = h[..., :2] / h[..., 3:]
    return float(((pix > -1) & (pix < 1)).all(-1).logical_and(h[..., 3] > 0).float().mean())


def eager(d, fp, center, radius, R, resolution, S):
    from rade_gs_b200 import unbounded as ub
    vs = radius * 2 / resolution
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for lo, sp, axes in ub.crop_axes(R, resolution, ub.CROP):
        pts = torch.from_numpy(np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)).to(DEV)
        for chunk in torch.split(pts, 256 ** 3):
            S.torch_tsdf(chunk, np.asarray(center, np.float32), float(radius), vs, d, fp, torch.float32)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[50, 300])
    ap.add_argument("--resolution", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--width", type=int, default=1240)
    ap.add_argument("--height", type=int, default=820)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--eager-views", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark measures the GPU: no CUDA device"
    import unbounded_scenes as S
    from diff_gaussian_rasterization import _C
    from rade_gs_b200 import unbounded as ub
    U = _C._unbounded
    print("card:", card(), flush=True)
    xyz = S.sphere_xyz(200_000).to(DEV)
    for V in args.views:
        d, c, wv, fp = S.views(V, W=args.width, H=args.height, seed=V)
        d, c, fp = d.to(DEV), c.to(DEV), fp.to(DEV)
        wv = list(wv)
        for res in args.resolution:
            tm = Timer()
            one_run(tm, U, ub, d, c, wv, fp, xyz, res)               # warm-up
            tm = Timer()
            for _ in range(args.reps):
                center, radius, R, mesh, clean = one_run(tm, U, ub, d, c, wv, fp, xyz, res)
            frac = in_view_fraction(U, ub, fp, d, center, radius, R)
            crop_samples = ub.CROP ** 3
            sdf_ms = tm.median("sdf_per_crop")
            evals = crop_samples * V / (sdf_ms * 1e-3)
            bytes_ = crop_samples * 4 + crop_samples * V * frac * 16
            row = {"views": V, "size": f"{args.width}x{args.height}", "resolution": res, "crops": (res // ub.CROP) ** 3,
                   **{f"{k}_ms": round(tm.median(k), 3) for k in ("normalisation", "sdf_per_crop", "mcubes_per_crop", "merge", "colors", "cleanup")},
                   "sample_view_evals_per_s": float(f"{evals:.4g}"), "in_view_fraction": round(frac, 4),
                   "sdf_bytes_per_s_upper": float(f"{bytes_ / (sdf_ms * 1e-3):.4g}"),
                   "vertices": int(mesh.vertices.shape[0]), "triangles": int(mesh.triangles.shape[0]),
                   "triangles_after_cleanup": int(clean.triangles.shape[0])}
            if res == 512 and V == args.eager_views:
                row["eager_sdf_s"] = round(eager(d, fp, center, radius, R, res, S), 3)
                row["ours_sdf_s"] = round(sdf_ms * row["crops"] * 1e-3, 4)
            else:
                row["eager_sdf_s"] = "not run"
            print(json.dumps(row), flush=True)
        del d, c, fp
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
