"""Times TSDF fusion and mesh extraction (rade_gs_b200.tsdf) at mesh_extract.py's settings: 49 views at 800x600, voxel 2 mm,
16^3 blocks, depth_max 8, truncation 8 voxels, weight threshold 3.  The depth and colour maps are analytic (a sphere of radius
0.3, cameras on an orbit of radius 1.2; like mesh_extract.py with DTU's object masks, only the object has depth), so the
block counts are those of this synthetic scene, not of a trained DTU model.  Prints one JSON line.

    python tools/bench_tsdf.py [--views 49] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_DATASHEET = 3.35e12   # H100 SXM data sheet, bytes/s


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "not read"
    except (OSError, subprocess.SubprocessError):
        power = "not read"
    return name, power


def views(n, W=800, H=600):
    import tsdf_scenes as ts
    out = []
    for eye in ts.orbit(n, 1.2, seed=0.7):
        K = ts.intrinsic(W, H, 50.0)
        E = ts.look_at(eye, (0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0))
        d, c = ts.render(K, E, H, W, spheres=[((0.0, 0.0, 0.0), 0.3)], max_depth=8.0)
        out.append((torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), K, E))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tsdf needs a CUDA device")
    from rade_gs_b200.tsdf import VoxelBlockGrid
    vs = 0.002
    vw = views(a.views)

    def fuse(timed):
        vbg = VoxelBlockGrid(vs, 16, 50000)
        per_view, per_int, nblk = [], [], []
        for d, c, K, E in vw:
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            coords = vbg.compute_unique_block_coordinates(d, K, E, 1.0, 8.0)
            e1.record()
            vbg.integrate(coords, d, c, K, E, 1.0, 8.0)
            e2.record()
            if timed:
                torch.cuda.synchronize()
                per_view.append(e0.elapsed_time(e2))
                per_int.append(e1.elapsed_time(e2))
                nblk.append(coords.shape[0])
        return vbg, per_view, per_int, nblk

    fuse(False)                                   # module load, allocator and CUB warm-up
    views_ms, int_ms = [], []
    for _ in range(a.reps):
        vbg = None                                # one grid alive at a time
        vbg, per_view, per_int, nblk = fuse(True)
        views_ms += per_view
        int_ms += per_int
    view_ms, int_ms = float(np.median(views_ms)), float(np.median(int_ms))
    ext = []
    for _ in range(a.reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        mesh = vbg.extract_triangle_mesh().compute_vertex_normals()
        e1.record()
        torch.cuda.synchronize()
        ext.append(e0.elapsed_time(e1))
    ext_ms = float(np.median(ext[1:]))
    blocks = int(vbg.active_blocks()[0].shape[0])
    # integrate's algorithmic bytes, counted from the block count of each view: every voxel of the given blocks reads and
    # writes tsdf, weight and 3 colours once (40 B) and reads one depth value (4 B); plus the colour image once
    med_blocks = float(np.median(nblk))
    int_bytes = med_blocks * 4096 * 44 + 800 * 600 * 12
    name, power = card()
    print(json.dumps({
        "bench": "tsdf", "views": a.views, "image": "800x600", "voxel_size": vs, "depth_max": 8.0,
        "touch_integrate_ms_per_view_median": round(view_ms, 4), "integrate_ms_per_view_median": round(int_ms, 4),
        "extract_normals_ms_median": round(ext_ms, 3),
        "blocks_per_view_median": med_blocks, "active_blocks": blocks, "voxels": blocks * 4096,
        "vertices": int(mesh.vertices.shape[0]), "triangles": int(mesh.triangles.shape[0]),
        "integrate_algorithmic_GBps": round(int_bytes / (int_ms * 1e-3) / 1e9, 1),
        "integrate_share_of_datasheet_3.35TBps": round(int_bytes / (int_ms * 1e-3) / HBM_DATASHEET, 3),
        "dtu_model_blocks": "not measured",
        "gpu": name, "power_limit": power,
    }))


if __name__ == "__main__":
    main()
