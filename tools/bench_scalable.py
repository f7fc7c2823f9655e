"""Times the bounded TSDF (rade_gs_b200.tsdf.ScalableTSDFVolume, the volume of GaussianExtractor.extract_mesh_bounded) on a
DTU-sized case: 64 views at 800x600 (DTU at -r 2), voxel 0.004, sdf_trunc 0.02, depth_trunc 3.  The maps are analytic (a
sphere of radius 0.3 before a plane, cameras on an orbit of radius 1.2), so unit counts are those of this synthetic scene,
not of a trained DTU model.  Open3D is not installed, so there is no CPU baseline here.  Prints a table, then one JSON line.

    python tools/bench_scalable.py [--views 64] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_tsdf import HBM_DATASHEET, card  # noqa: E402

W, H = 800, 600


def views(n):
    import tsdf_scenes as ts
    out = []
    for eye in ts.orbit(n, 1.2, seed=0.7):
        K = ts.intrinsic(W, H, 50.0)
        E = ts.look_at(eye, (0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0))
        d, c = ts.render(K, E, H, W, spheres=[((0.0, 0.0, 0.0), 0.3)], planes=[(tuple(-eye / np.linalg.norm(eye)), 0.6)], max_depth=8.0)
        rgb = torch.from_numpy(np.ascontiguousarray(np.transpose(c, (2, 0, 1)))).cuda()
        out.append((rgb, torch.from_numpy(d[None]).cuda(), K, E))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_scalable needs a CUDA device")
    from rade_gs_b200.tsdf import ScalableTSDFVolume, rgbd_from_color_and_depth
    vl, trunc, depth_trunc = 0.004, 0.02, 3.0
    vw = views(a.views)

    def fuse(timed):
        vol = ScalableTSDFVolume(vl, trunc)
        per_view, units = [], []
        for rgb, d, K, E in vw:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            color, depth = rgbd_from_color_and_depth(rgb, d, depth_trunc)
            vol.integrate(color, depth, K, E)
            e1.record()
            if timed:
                torch.cuda.synchronize()
                per_view.append(e0.elapsed_time(e1))
                units.append(int(vol.counters[1].item()))
        return vol, per_view, units

    fuse(False)                                   # module load, allocator and CUB warm-up, the volume's growth
    view_ms = []
    for _ in range(a.reps):
        vol = None                                # one volume alive at a time
        vol, per_view, units = fuse(True)
        view_ms += per_view
    ms = float(np.median(view_ms))
    ext = []
    for _ in range(a.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        mesh = vol.extract_triangle_mesh()
        e1.record()
        torch.cuda.synchronize()
        ext.append(e0.elapsed_time(e1))
    ext_ms = float(np.median(ext[1:]))
    med_units = float(np.median(units))
    # algorithmic bytes of one view: the RGBD conversion reads 12 B of colour and 4 B of depth and writes 3 B and 4 B per
    # pixel; touch reads every 16th depth value; integrate reads and writes tsdf, weight and 3 colours (40 B) of every voxel
    # of the touched units and reads one depth value and 3 colour bytes (7 B)
    view_bytes = W * H * (12 + 4 + 3 + 4) + W * H // 16 * 4 + med_units * 4096 * 47
    name, power = card()
    rows = [("integrate per view (rgbd + touch + integrate), ms, median", f"{ms:.3f}"),
            ("touched units per view, median", f"{med_units:.0f}"),
            ("allocated units", f"{int(vol.active_blocks()[0].shape[0])}"),
            ("algorithmic bytes per view, MB", f"{view_bytes / 1e6:.1f}"),
            ("achieved, GB/s (share of the 3.35 TB/s data sheet)", f"{view_bytes / (ms * 1e-3) / 1e9:.1f} ({view_bytes / (ms * 1e-3) / HBM_DATASHEET:.3f})"),
            ("extract, ms, median", f"{ext_ms:.3f}"),
            ("mesh vertices / triangles", f"{mesh.vertices.shape[0]} / {mesh.triangles.shape[0]}"),
            ("CPU baseline (Open3D)", "not installed: not measured"),
            ("card", f"{name}, power limit {power}")]
    for k, v in rows:
        print(f"{k:<60} {v}")
    print(json.dumps({
        "bench": "scalable_tsdf", "views": a.views, "image": f"{W}x{H}", "voxel_length": vl, "sdf_trunc": trunc, "depth_trunc": depth_trunc,
        "integrate_ms_per_view_median": round(ms, 4), "units_per_view_median": med_units, "extract_ms_median": round(ext_ms, 3),
        "bytes_per_view": int(view_bytes), "achieved_GBps": round(view_bytes / (ms * 1e-3) / 1e9, 1),
        "vertices": int(mesh.vertices.shape[0]), "triangles": int(mesh.triangles.shape[0]), "gpu": name, "power_limit": power,
    }))


if __name__ == "__main__":
    main()
