"""Tanks and Temples mesh cull on a synthetic TNT-sized case: a room with objects (about 20 M triangles, 10 M vertices) and
300 cameras at 1920x1080 with the TNT intrinsics.

Reports CUDA-event medians of the rasterizer and of the visibility count per view and the time of the whole ``cull_mesh``;
the share of faces on each side of the rasterizer's work split (the numpy model on a seeded 1 M-face sample, for one
view); the algorithmic bytes per view over the per-view time against the 3.35 TB/s data sheet; a torch restatement of
the reference's ``point_masks`` expressions (matmul, ``grid_sample``) on the same GPU with the maps given, over a subset of
views; and the card's name and power limit.  pyrender is not installed, so there is no rasterizer baseline.

Usage:  python tools/bench_tnt_cull.py [--views 300] [--timed 30] [--out FILE.json]
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
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from rade_gs_b200 import tnt_cull  # noqa: E402

H, W = tnt_cull.H, tnt_cull.W
K = dict(fx=tnt_cull.FX, fy=tnt_cull.FY, cx=tnt_cull.CX, cy=tnt_cull.CY)


def grid(o, du, dv, n):
    s = np.linspace(0.0, 1.0, n + 1, dtype=np.float32)
    a, b = np.meshgrid(s, s, indexing="ij")
    v = o + a.reshape(-1, 1) * du + b.reshape(-1, 1) * dv
    i = np.arange((n + 1) ** 2, dtype=np.int32).reshape(n + 1, n + 1)
    q = np.stack([i[:-1, :-1], i[1:, :-1], i[1:, 1:], i[:-1, 1:]], -1).reshape(-1, 4)
    return v.astype(np.float32), np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])


def box(lo, hi, n):
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    out = []
    for ax in range(3):
        u, w = [k for k in range(3) if k != ax]
        for side in (lo[ax], hi[ax]):
            o = lo.copy()
            o[ax] = side
            du, dv = np.zeros(3, np.float32), np.zeros(3, np.float32)
            du[u], dv[w] = hi[u] - lo[u], hi[w] - lo[w]
            out.append(grid(o, du, dv, n))
    return out


def scene(seed=0):
    rng = np.random.default_rng(seed)
    parts = box([-6, -2, -6], [6, 2, 6], 900)
    for _ in range(10):
        c = rng.uniform([-4, -1.2, -4], [4, 0.5, 4])
        s = rng.uniform(0.3, 0.8, 3)
        parts += box(c - s, c + s, 300)
    vs, fs, off = [], [], 0
    for v, f in parts:
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    return np.concatenate(vs), np.concatenate(fs).astype(np.int32)


def cameras(n, seed=1):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        eye = rng.uniform([-5, -1.5, -5], [5, 1.5, 5])
        t = rng.uniform([-3, -1, -3], [3, 1, 3])
        z = t - eye
        z /= np.linalg.norm(z)
        x = np.cross(z, [0.0, -1.0, 0.0])
        x /= np.linalg.norm(x)
        T = np.eye(4)
        T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, np.cross(z, x), z, eye
        out.append(T)
    return np.stack(out)


def reference_point_masks(points, depths, c2w, fx, fy, cx, cy, eps=0.005):
    """The reference's per-view torch expressions (one batch, maps given), restated: fp32 inverse, K @ (w2c @ p), z + 1e-8,
    frustum, grid_sample(border, align_corners=True), the occlusion test; returns the count per point."""
    import torch.nn.functional as F
    n = points.shape[0]
    cnt = torch.zeros(n, dtype=torch.int32, device=points.device)
    Kt = torch.tensor([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], device=points.device).float()
    homo = torch.cat([points, torch.ones_like(points[:, :1])], 1).reshape(-1, 4, 1)
    for D, c in zip(depths, c2w):
        w2c = torch.inverse(c)
        cam = (w2c @ homo)[:, :3, :]
        uv = Kt @ cam
        z = uv[:, -1:] + 1e-8
        uv = uv[:, :2] / z
        u, v, z = uv[:, 0, 0], uv[:, 1, 0], z[:, 0, 0]
        fr = (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1) & (z > 0)
        g = uv.reshape(1, 1, -1, 2).clone()
        g[..., 0] = g[..., 0] / (W - 1) * 2.0 - 1.0
        g[..., 1] = g[..., 1] / (H - 1) * 2.0 - 1.0
        s = F.grid_sample(D.reshape(1, 1, H, W), g, padding_mode="border", align_corners=True).reshape(-1)
        cnt += (fr & torch.where(s > 0, z < s + eps, torch.ones_like(fr))).int()
    return cnt


def median_ms(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--timed", type=int, default=30, help="views timed one by one (and for the reference's expressions)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tnt_cull needs a CUDA device")
    from diff_gaussian_rasterization import _C
    C = _C._tnt_cull
    t0 = time.time()
    v, f = scene()
    poses = cameras(a.views)
    V, F_ = len(v), len(f)
    print(f"scene: {F_} faces, {V} vertices, {a.views} views at {W}x{H} (built in {time.time() - t0:.1f} s)", flush=True)
    vt, ft = torch.as_tensor(v, device="cuda"), torch.as_tensor(f, device="cuda")
    ms = tnt_cull._w2c(poses)

    import tnt_cull_model as M
    sample = np.random.default_rng(2).choice(F_, 1_000_000, replace=False)
    shares = [M.split(v, f[sample], np.array(ms[k], np.float32), K["fx"], K["fy"], K["cx"], K["cy"], H, W) for k in range(2)]
    drawn = [sum(s) for s in shares]

    depth = C.mesh_depth(vt, ft, ms[0], *K.values(), H, W, 0.01, 20.0)   # warm-up
    counts = torch.zeros(V, dtype=torch.int32, device="cuda")
    C.visibility_count(vt, depth, ms[0], *K.values(), 0.005, counts)
    torch.cuda.synchronize()
    k = 0
    raster = []
    count = []
    for k in range(a.timed):
        m = ms[k % len(ms)]
        raster.append(median_ms(lambda: C.mesh_depth(vt, ft, m, *K.values(), H, W, 0.01, 20.0), 1))
        depth = C.mesh_depth(vt, ft, m, *K.values(), H, W, 0.01, 20.0)
        count.append(median_ms(lambda: C.visibility_count(vt, depth, m, *K.values(), 0.005, counts), 3))
    r_ms, c_ms = float(np.median(raster)), float(np.median(count))

    torch.cuda.synchronize()
    t = time.time()
    _, cf, valid, _ = tnt_cull.cull_mesh(vt, ft, poses)
    torch.cuda.synchronize()
    whole = time.time() - t

    # algorithmic bytes per view: faces (12 B) and their vertices (12 B per face corner, L2-resident mostly: counted once
    # per vertex), the depth memset, drawing (one 4 B atomic per covered pixel, counted once) and finish (read + write);
    # the count reads every point (12 B), four depth corners at most (counted as one 4 B read) and updates the count (8 B)
    px = H * W
    raster_bytes = 12 * F_ + 12 * V + 4 * px * 4
    count_bytes = V * (12 + 4 + 8)
    gbs = (raster_bytes + count_bytes) / ((r_ms + c_ms) * 1e-3) / 1e9

    sub = min(a.timed, 20)
    pts = vt
    depths = torch.stack([C.mesh_depth(vt, ft, ms[i], *K.values(), H, W, 0.01, 20.0) for i in range(sub)])
    c2w32 = torch.as_tensor(poses[:sub], device="cuda").float()
    reference_point_masks(pts, depths[:2], c2w32[:2], **K)
    ref_ms = median_ms(lambda: reference_point_masks(pts, depths, c2w32, **K), 3) / sub
    ours = torch.zeros(V, dtype=torch.int32, device="cuda")
    ours_ms = median_ms(lambda: [C.visibility_count(vt, depths[i], ms[i], *K.values(), 0.005, ours) for i in range(sub)], 3) / sub

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=smi, faces=F_, vertices=V, views=a.views, H=H, W=W,
               split_sample_faces=1_000_000, split_small_medium_large=[list(s) for s in shares],
               split_share_small=[s[0] / max(d, 1) for s, d in zip(shares, drawn)],
               raster_ms_per_view_median=r_ms, count_ms_per_view_median=c_ms,
               algorithmic_bytes_per_view=raster_bytes + count_bytes, achieved_GBps=gbs, fraction_of_3p35TBps=gbs / 3350.0,
               cull_mesh_total_s=whole, cull_mesh_ms_per_view=1e3 * whole / a.views, valid_vertices=int(valid.sum()), kept_faces=len(cf),
               reference_point_masks_ms_per_view=ref_ms, our_count_ms_per_view_same_maps=ours_ms, reference_views_timed=sub)
    print(json.dumps(res, indent=1), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
