"""Time the Tanks and Temples evaluation (rade_gs_b200.tnt_eval) on a TNT-sized synthetic scene: a bumpy surface about
4 m across meshed with a few million triangles (vertices plus centroids: several million source points), about 10^7
ground-truth points and tau = 0.005 (Caterpillar / Truck).

Prints CUDA-event times per stage (crop, voxel downsample, each ICP stage with its iteration count, distances,
histogram), the host time of the RANSAC, the point counts, and the card's name and power limit from the same run.  With
Open3D importable it would also time Open3D; it is not installed here, so no comparison is made and no speed-up is
claimed.  Real TNT scenes are not available here: their sizes and times are not measured.

Usage:  python tools/bench_tnt_eval.py [--grid 1200] [--gt 10000000] [--out DIR]
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
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def height(x, y):
    return 0.15 * np.sin(1.3 * x) * np.cos(0.9 * y) + 0.05 * np.cos(4.0 * x + 1.0)


class Timer:
    def __init__(self):
        self.ms = {}

    def __call__(self, name, fn, *a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        out = fn(*a, **k)
        e.record()
        torch.cuda.synchronize()
        self.ms[name] = self.ms.get(name, 0.0) + s.elapsed_time(e)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=1200, help="mesh grid side: 2 (grid - 1)^2 triangles")
    ap.add_argument("--gt", type=int, default=10_000_000)
    ap.add_argument("--extent", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tnt_eval needs a CUDA device")
    from diff_gaussian_rasterization import _C
    from rade_gs_b200 import tnt_eval as te

    tau, e, dev = 0.005, a.extent, "cuda"
    rng = np.random.default_rng(0)
    g = a.grid
    xs = np.linspace(-e, e, g)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    verts = np.column_stack([X.ravel(), Y.ravel(), height(X.ravel(), Y.ravel())]) + rng.normal(0, tau / 3, (g * g, 3))
    i, j = np.meshgrid(np.arange(g - 1), np.arange(g - 1), indexing="ij")
    A, B, C, D = i * g + j, (i + 1) * g + j, i * g + j + 1, (i + 1) * g + j + 1
    faces = np.concatenate([np.stack([A, B, C], -1).reshape(-1, 3), np.stack([B, D, C], -1).reshape(-1, 3)])
    xy = rng.uniform(-e, e, (a.gt, 2))
    gt = np.column_stack([xy, height(xy[:, 0], xy[:, 1])])
    poly = np.array([[-0.9, -0.9], [0.9, -0.9], [0.9, 0.9], [0.0, 0.3], [-0.9, 0.9]]) * e
    vol = te.CropVolume(2, -1.0, 1.0, poly)
    P = np.eye(4)
    c, s = np.cos(0.002), np.sin(0.002)
    P[:3, :3] = 1.001 * np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    P[:3, 3] = [0.003, -0.002, 0.001]
    verts = te.apply_transform(np.linalg.inv(P), verts)
    n_cams = 300
    ang = np.linspace(0, 2 * np.pi, n_cams, endpoint=False)
    centres = np.column_stack([1.5 * e * np.cos(ang), 1.5 * e * np.sin(ang), np.full(n_cams, 1.0)])
    gt_traj = np.tile(np.eye(4), (n_cams, 1, 1))
    gt_traj[:, :3, 3] = centres
    traj = gt_traj.copy()
    traj[:, :3, 3] = te.apply_transform(np.linalg.inv(P), centres) + rng.normal(0, 1e-4, (n_cams, 3))

    t = Timer()
    src_all = t("mesh_points_with_upload", te.mesh_points, verts, faces)   # includes the host -> device copy of the mesh
    gt_d = torch.as_tensor(gt, device=dev)
    h0 = time.perf_counter()
    T0 = te.trajectory_alignment(traj, gt_traj, np.eye(4), seed=0)
    ransac_s = time.perf_counter() - h0
    gt_crop = t("crop_gt", te.crop, gt_d, vol)[0]
    gt_tau = t("voxel_gt_tau", te.voxel_down_sample, gt_crop, tau)[0]
    gt_half = t("voxel_gt_tau/2", te.voxel_down_sample, gt_crop, tau / 2)[0]
    stages, T = [], T0
    for k, (voxel, thr, target) in enumerate(((tau, 80 * tau, gt_tau), (tau / 2, 20 * tau, gt_half), (None, 2 * tau, te.uniform_for_registration(gt_crop)))):
        sc = t(f"stage{k + 1}_crop", te.crop, src_all, vol, T)[0]
        if voxel is not None:
            sc = t(f"stage{k + 1}_voxel", te.voxel_down_sample, sc, voxel)[0]
        r = t(f"stage{k + 1}_icp", te.icp, sc, target, thr, None, 20)
        T = r.transformation @ T
        stages.append(dict(source=int(sc.shape[0]), target=int(target.shape[0]), iterations=r.iterations, fitness=r.fitness, rmse=r.inlier_rmse,
                           ms=round(t.ms[f"stage{k + 1}_icp"], 2), ms_per_iteration=round(t.ms[f"stage{k + 1}_icp"] / (r.iterations + 1), 2)))
    s = t("eval_crop", te.crop, src_all, vol, T)[0]
    s = t("eval_voxel", te.voxel_down_sample, s, tau / 2)[0]
    d1 = t("distance_precision", lambda: _C.dtu_nearest(gt_half, s)[0])
    d2 = t("distance_recall", lambda: _C.dtu_nearest(s, gt_half)[0])
    edges = te.histogram_edges(tau)
    t("histogram_first_call", lambda: (te.cumulative_histogram(d1, edges), te.cumulative_histogram(d2, edges)))   # includes one-time setup
    t("histogram", lambda: (te.cumulative_histogram(d1, edges), te.cumulative_histogram(d2, edges)))
    p, r_, f = te.f_score(d1, d2, tau)
    res = {"card": card(), "tau": tau, "triangles": int(len(faces)), "source_points": int(src_all.shape[0]), "gt_points": int(gt.shape[0]),
           "gt_cropped": int(gt_crop.shape[0]), "gt_voxel_tau": int(gt_tau.shape[0]), "gt_voxel_tau/2": int(gt_half.shape[0]),
           "eval_source": int(s.shape[0]), "ransac_host_s": round(ransac_s, 3), "stages": stages,
           "stage_ms": {k: round(v, 2) for k, v in t.ms.items()}, "total_gpu_ms": round(sum(t.ms.values()), 2),
           "precision": p, "recall": r_, "fscore": f, "final_error_vs_planted": float(np.abs(T - P).max())}
    try:
        import open3d  # noqa: F401
        res["open3d"] = "importable, but not timed by this tool"
    except ImportError:
        res["open3d"] = "not installed: not measured"
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_tnt_eval.json"), "w") as fp:
            json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
