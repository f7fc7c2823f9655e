"""Time the DTU evaluation (rade_gs_b200.dtu_eval) on a DTU-sized synthetic scan: a closed bumpy object about 300 mm
across with more than a million triangles, sampled at 0.2 mm, and a few million ground-truth (STL) points.

Prints CUDA-event times per stage, the point counts, and the card's name and power limit.  With scikit-learn installed it
also times, once, the numpy / scikit-learn calls eval.py makes on the same inputs (eval.py samples in a multiprocessing
pool; here the sampling is the same numpy per triangle, in one process, so that stage is not compared).  Real DTU scans
are not available here: their sizes are not measured, and no speed-up on them is claimed.

Usage:  python tools/bench_dtu_eval.py [--rings 700] [--stl 3000000] [--skip-cpu] [--out DIR]
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


def object_mesh(rings: int, radius: float = 150.0, centre=(500.0, 500.0, 500.0)):
    """A bumpy closed surface (UV sphere with radial ripples): 2 * rings * (2 * rings) triangles."""
    th = np.linspace(0, np.pi, rings + 1)
    ph = np.linspace(0, 2 * np.pi, 2 * rings, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    R = radius * (1 + 0.05 * np.sin(5 * T) * np.cos(7 * P))
    v = np.stack([R * np.sin(T) * np.cos(P), R * np.sin(T) * np.sin(P), R * np.cos(T)], -1).reshape(-1, 3) + np.asarray(centre)
    n = 2 * rings
    i, j = np.meshgrid(np.arange(rings), np.arange(n), indexing="ij")
    a, b, c, d = i * n + j, i * n + (j + 1) % n, (i + 1) * n + j, (i + 1) * n + (j + 1) % n
    f = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)])
    return v, f


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rings", type=int, default=700)
    ap.add_argument("--stl", type=int, default=3_000_000)
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dtu_eval needs a CUDA device")
    from rade_gs_b200 import dtu_eval as de

    v, f = object_mesh(a.rings)
    rng = np.random.default_rng(0)
    vs = v[rng.integers(0, len(v), a.stl)]
    stl = vs + rng.normal(0, 0.3, vs.shape)
    bb = np.array([[330.0, 330.0, 330.0], [670.0, 670.0, 670.0]])
    res = np.array([[2.0]])
    obs = np.ones((171, 171, 171), np.uint8)
    plane = np.array([0.0, 0.0, 1.0, -380.0])
    dev = torch.device("cuda")
    vt, ft = torch.as_tensor(v, device=dev), torch.as_tensor(f, device=dev)
    stl_t = torch.as_tensor(stl, device=dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1)

    # warm-up of every shape's kernels on a small copy
    de.evaluate((v[:5000], f[(f < 5000).all(1)]), stl[:10000], obs, bb, res, plane, seed=0)
    torch.cuda.synchronize()
    pcd, t_sample = timed(lambda: de.sample_mesh_points(vt, ft, 0.2))
    ds, t_down = timed(lambda: de.radius_downsample(pcd, 0.2, seed=0))
    r, t_total = timed(lambda: de.evaluate((vt, ft), stl_t, obs, bb, res, plane, seed=0))
    down = ds.points
    _, t_d2s = timed(lambda: de.nearest_distances(stl_t, down))
    _, t_s2d = timed(lambda: de.nearest_distances(down, stl_t))
    result = {"card": card(), "triangles": len(f), "vertices": len(v), "sampled_points": int(pcd.shape[0]), "kept_points": int(down.shape[0]),
              "downsample_rounds": ds.rounds, "stl_points": len(stl), "ms": {"sample": t_sample, "downsample": t_down, "nearest_data_to_stl": t_d2s,
                                                                               "nearest_stl_to_data": t_s2d, "evaluate_total": t_total},
              "means": [r.mean_d2s, r.mean_s2d, r.overall]}

    if not a.skip_cpu:
        try:
            import sklearn.neighbors as skln
        except ImportError:
            skln = None
        if skln is not None:
            data_pcd = pcd.cpu().numpy()[ds.perm.cpu().numpy()]
            t = time.perf_counter()
            nn = skln.NearestNeighbors(n_neighbors=1, radius=0.2, algorithm="kd_tree", n_jobs=-1)
            nn.fit(data_pcd)
            idxs = nn.radius_neighbors(data_pcd, radius=0.2, return_distance=False)
            mask = np.ones(len(data_pcd), bool)
            for cur, ix in enumerate(idxs):
                if mask[cur]:
                    mask[ix] = 0
                    mask[cur] = 1
            t_cpu_down = time.perf_counter() - t
            assert np.array_equal(mask, ds.kept.cpu().numpy()), "scikit-learn's kept set differs"
            dd = data_pcd[mask]
            t = time.perf_counter()
            nn.fit(stl)
            nn.kneighbors(dd, n_neighbors=1, return_distance=True)
            t_cpu_d2s = time.perf_counter() - t
            t = time.perf_counter()
            nn.fit(dd)
            nn.kneighbors(stl, n_neighbors=1, return_distance=True)
            t_cpu_s2d = time.perf_counter() - t
            result["cpu_reference_s"] = {"cores": os.cpu_count(), "downsample": t_cpu_down, "nearest_data_to_stl": t_cpu_d2s,
                                         "nearest_stl_to_data": t_cpu_s2d}
    print(json.dumps(result))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_dtu_eval.json"), "w") as fp:
            json.dump(result, fp, indent=1)


if __name__ == "__main__":
    main()
