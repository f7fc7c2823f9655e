"""Per-stage timing of the tetrahedra mesh extraction (rade_gs_b200.tetra) on the GPU, next to the reference's eager torch
expressions for the same stage on the same GPU.  Prints the card's name and power limit, then one line per stage.

Stages at --gaussians (default 0.1 M and 1 M synthetic Gaussians): tetra points; CullSDF.add per view on synthetic integrate
outputs (1600x1200 render, all 9P points), apart from integrate.  Marching tetrahedra, one bisection step and the filter run
on Kuhn-subdivided lattices (--lattice, default 100 and 180 cubes a side: 6.0 M and 35.0 M tets), because a host Delaunay of
0.9 M or 9 M points takes minutes.  The whole extraction, integrate included, runs on a sphere of --e2e-gaussians disc
Gaussians seen from 20 views (host triangulation reported apart).

Usage:  python tools/bench_tetra.py [--gaussians 100000 1000000] [--lattice 100 180] [--e2e-gaussians 10000] [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

DEV = "cuda:0"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


# ---- the reference's eager expressions (restated) ---------------------------------------------------------------------------

def eager_tetra_points(xyz, s, rot):
    q = rot / rot.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z), 1 - 2 * (x * x + z * z),
                     2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    box = torch.tensor([[(k >> 2) & 1, (k >> 1) & 1, k & 1] for k in range(8)], dtype=torch.float32, device=xyz.device).T * 2 - 1
    s3 = s * 3.0
    v = torch.bmm(R, box[None].repeat(xyz.shape[0], 1, 1) * s3[..., None]) + xyz[..., None]
    pts = torch.cat([v.permute(0, 2, 1).reshape(-1, 3), xyz])
    m = s3.max(dim=-1, keepdim=True)[0]
    return pts, torch.cat([m.repeat(1, 8).reshape(-1, 1), m])


def eager_cull(final, weight, alpha, coord, render7, W, H):
    pc = coord.clone()
    pc[:, 0] = (pc[:, 0] * 2 + 1) / (W - 1) - 1
    pc[:, 1] = (pc[:, 1] * 2 + 1) / (H - 1) - 1
    prob = torch.nn.functional.grid_sample(render7[None, None], pc[None, None], padding_mode="zeros", align_corners=False)[0, 0, 0]
    valid = prob > 0.5
    return torch.where(valid, torch.min(alpha, final), final), torch.where(valid, weight + 1, weight)


def eager_marching(vertices, tets, sdf):
    occ = sdf > 0
    occ4 = occ[tets.reshape(-1)].reshape(-1, 4)
    s = occ4.sum(-1)
    valid = (s > 0) & (s < 4)
    edges = tets[valid][:, [0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3]].reshape(-1, 2)
    edges = torch.sort(edges, dim=1)[0]
    uniq, inv = torch.unique(edges, dim=0, return_inverse=True)
    cross = occ[uniq.reshape(-1)].reshape(-1, 2).sum(-1) == 1
    return vertices[uniq[cross].reshape(-1)].reshape(-1, 2, 3), inv


def eager_bisect(left, right, ls, mid_sdf):
    mid = (left + right) / 2
    low = ((mid_sdf < 0) & (ls < 0)) | ((mid_sdf > 0) & (ls > 0))
    left[low] = mid[low]
    right[~low] = mid[~low]
    return (left + right) / 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, nargs="*", default=[100_000, 1_000_000])
    ap.add_argument("--lattice", type=int, nargs="*", default=[100, 180])
    ap.add_argument("--e2e-gaussians", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_tetra needs a CUDA device"
    from diff_gaussian_rasterization import _C
    from rade_gs_b200 import tetra
    import test_gpu_tetra as g

    rows = []

    def report(stage, size, ours, eager=None):
        rows.append({"stage": stage, "size": size, "ours_ms": ours, "eager_ms": eager})
        e = f"   eager {eager:9.3f} ms   x{eager / ours:6.1f}" if eager else ""
        print(f"{stage:28s} {size:>26s}   ours {ours:9.3f} ms{e}", flush=True)

    print(f"card: {card()}", flush=True)
    gen = torch.Generator(DEV).manual_seed(0)
    for P in args.gaussians:
        xyz = torch.randn(P, 3, device=DEV, generator=gen)
        s = torch.rand(P, 3, device=DEV, generator=gen) * 0.05
        rot = torch.randn(P, 4, device=DEV, generator=gen)
        report("tetra_points", f"{P} Gaussians", timed(lambda: _C.tetra_points(xyz, s, rot), args.reps),
               timed(lambda: eager_tetra_points(xyz, s, rot), args.reps))
        N, W, H = 9 * P, 1600, 1200
        alpha = torch.rand(N, device=DEV, generator=gen)
        coord = torch.rand(N, 2, device=DEV, generator=gen) * torch.tensor([W * 1.2, H * 1.2], device=DEV) - 0.1 * torch.tensor([W, H], device=DEV)
        r7 = torch.rand(H, W, device=DEV, generator=gen)
        cull = tetra.CullSDF(N, DEV)
        fin, wt = torch.ones(N, device=DEV), torch.zeros(N, dtype=torch.int32, device=DEV)
        report("CullSDF.add (per view)", f"{N} points", timed(lambda: cull.add(alpha, coord, r7), args.reps),
               timed(lambda: eager_cull(fin, wt, alpha, coord, r7, W, H), args.reps))
        del xyz, s, rot, alpha, coord, cull, fin, wt
        torch.cuda.empty_cache()

    for n in args.lattice:
        pts, tets = g.kuhn_lattice(n, DEV)
        c = n * 0.5 + 0.37
        o = pts - torch.tensor([c, c - 0.21, c + 0.13], device=DEV)
        sdf = (o * o).sum(-1) - (n * 0.4) ** 2
        scl = torch.rand(pts.shape[0], device=DEV, generator=gen)
        T = tets.shape[0]
        out = _C.tetra_marching(pts, sdf, scl, tets)
        try:
            eager = timed(lambda: eager_marching(pts, tets, sdf), max(1, args.reps // 5))
        except torch.OutOfMemoryError:
            eager = None
        report("marching_tetrahedra", f"{T / 1e6:.1f} M tets", timed(lambda: _C.tetra_marching(pts, sdf, scl, tets), max(1, args.reps // 2)), eager)
        ends, esdf, escl, faces, _ = out
        M = ends.shape[0]
        left, right = ends[:, 0].contiguous(), ends[:, 1].contiguous()
        ls, rs = esdf[:, 0, 0].contiguous(), esdf[:, 1, 0].contiguous()
        mid = torch.empty_like(left)
        msdf = torch.randn(M, device=DEV, generator=gen)
        report("bisection step", f"{M} vertices", timed(lambda: _C.tetra_bisect(msdf, left, right, ls, rs, mid), args.reps),
               timed(lambda: eager_bisect(left, right, ls, msdf), args.reps))
        report("filter", f"{M} v / {faces.shape[0]} f", timed(lambda: _C.tetra_filter(mid, ends, escl, faces), args.reps))
        del pts, tets, sdf, scl, out, ends, esdf, escl, faces, left, right, mid
        torch.cuda.empty_cache()

    # whole extraction with integrate, 20 views
    import diff_gaussian_rasterization as dgr
    P, W, H, fov = args.e2e_gaussians, 800, 800, math.radians(50)
    xyz, scales, rot = (t.to(DEV) for t in g._disc_sphere(P, 7))
    opac = torch.full((P, 1), 0.95, device=DEV)
    shs = torch.zeros((P, 1, 3), device=DEV)
    rasts = []
    for k in range(20):
        d = torch.randn(3, generator=torch.Generator().manual_seed(100 + k)).double()
        view, proj, campos = g._camera(tuple((3.5 * d / d.norm()).tolist()), W, H, fov)
        st = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=math.tan(fov / 2), tanfovy=math.tan(fov / 2), kernel_size=0.0,
                                               bg=torch.zeros(3, device=DEV), scale_modifier=1.0, viewmatrix=view.to(DEV), projmatrix=proj.to(DEV),
                                               sh_degree=0, campos=campos.to(DEV), prefiltered=False, require_depth=True, require_coord=True, debug=False)
        rasts.append(dgr.GaussianRasterizer(st))

    def evaluate(points):
        cull = tetra.CullSDF(points.shape[0], points.device)
        for r in rasts:
            color, alpha, _, coord, _, _ = r.integrate(points3D=points, means3D=xyz, means2D=None, opacities=opac, shs=shs, scales=scales, rotations=rot)
            cull.add(alpha, coord, color[7])
        return cull.sdf()

    pts, pscl = tetra.tetra_points(xyz, scales, rot)
    t0 = time.perf_counter()
    cells = tetra.triangulate(pts)
    tri = time.perf_counter() - t0
    tetra.extract_mesh(pts, pscl, cells, evaluate)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    v, f = tetra.extract_mesh(pts, pscl, cells, evaluate)
    torch.cuda.synchronize()
    whole = (time.perf_counter() - t0) * 1e3
    print(f"host triangulation: {tri:.2f} s for {pts.shape[0]} points -> {cells.shape[0]} tets", flush=True)
    report("extract_mesh (20 views)", f"{P} Gaussians, {v.shape[0]} v", whole)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": card(), "rows": rows, "triangulation_s": tri}, fh, indent=1)


if __name__ == "__main__":
    main()
