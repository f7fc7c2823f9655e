"""Fixtures of the DTU evaluation, made by the reference's own code on the CPU: tests/golden/dtu_eval/*.npz.

Runs the UNMODIFIED dtu_eval/eval.py with runpy on synthetic scans (mm-scale coordinates offset by about 500, synthetic
ObsMask / Plane .mat files, both modes) and calls the reference's ``cull_mesh`` from evaluate_dtu_mesh.py.  Stand-ins:

* ``open3d``: an in-process module whose readers return the arrays registered here and whose ``write_point_cloud`` is
  captured;
* the shuffle: ``np.random.default_rng`` is seeded; the permutation is recorded by drawing it from an identically seeded
  generator, and the shuffled array is checked to equal ``original[perm]``;
* ``cull_mesh`` is compiled from its source alone (the script's other imports need a training checkout), with ``.cuda()``
  meaning the CPU (as in gen_golden_fused.py), scikit-image's ``binary_dilation`` / ``disk`` replaced by
  ``scipy.ndimage.binary_dilation`` with the disk footprint, and the trimesh mesh by an object with trimesh's
  ``update_vertices`` / ``update_faces``.

Usage:  python tools/gen_golden_dtu_eval.py [--reference /path/to/RaDe-GS] [--out DIR]   (needs scikit-learn, tqdm)
Copy the files to tests/golden/dtu_eval/ (a subdirectory: tests/golden/*.npz are rasterizer cases).
"""
from __future__ import annotations

import argparse
import ast
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import scipy.io
from scipy import ndimage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- scenes ---------------------------------------------------------------------------------------------------------------

def _mesh_scene(rng, n_tri=120, scale=2.5):
    """A bumpy sheet of triangles near (500, 500, 500) plus the degenerate families."""
    g = 12
    xs, ys = np.meshgrid(np.arange(g) * scale, np.arange(g) * scale, indexing="ij")
    zs = 0.8 * np.sin(xs / 3.0) * np.cos(ys / 4.0) + rng.normal(0, 0.2, xs.shape)
    verts = np.stack([xs, ys, zs], -1).reshape(-1, 3) + np.array([488.0, 489.5, 500.25])
    faces = []
    for i in range(g - 1):
        for j in range(g - 1):
            a, b, c, d = i * g + j, (i + 1) * g + j, i * g + j + 1, (i + 1) * g + j + 1
            faces += [(a, b, c), (b, d, c)]
    faces = [faces[k] for k in rng.choice(len(faces), n_tri, replace=False)]
    V = len(verts)
    extra = np.array([
        [500.0, 500.0, 503.0], [500.0, 500.0, 503.0],          # duplicate vertices
        [501.0, 500.0, 503.0], [502.0, 500.0, 503.0],          # collinear with the first: zero area
        [495.0, 495.0, 506.0], [495.0 + 1e-9, 495.0, 506.0], [510.0, 495.0, 506.0],   # a sliver
        [480.0, 480.0, 510.0], [492.0, 480.0, 510.0], [480.0, 491.0, 511.0],          # one large triangle
        [400.0, 400.0, 400.0], [400.5, 400.0, 400.0], [400.0, 400.5, 400.0],          # outside the box and the grid
    ])
    verts = np.concatenate([verts, extra])
    faces += [(V, V + 1, V + 2), (V, V + 2, V + 3), (V + 1, V + 1, V + 2),            # zero area, repeated index
              (V + 4, V + 5, V + 6), (V + 7, V + 8, V + 9), (V + 10, V + 11, V + 12)]
    return verts, np.array(faces, np.int64)


def _ground_truth(rng, n_stl, plane_z=499.0):
    bb = np.array([[484.0, 484.0, 494.0], [520.0, 520.0, 514.0]])
    res = np.array([[1.0]])
    shape = tuple(((bb[1] - bb[0]) / res[0, 0]).astype(int) + 1)
    obs = (rng.random(shape) < 0.85).astype(np.uint8)
    stl = np.concatenate([
        rng.uniform([486, 486, 497], [518, 518, 503], (n_stl, 3)),
        rng.uniform([486, 486, 490], [518, 518, 498.5], (n_stl // 4, 3)),             # below the plane
        np.array([[600.0, 600.0, 600.0]]),
    ])
    plane = np.array([[0.0], [0.0], [1.0], [-plane_z]])                           # z > plane_z is above
    return obs, bb, res, plane, stl


def _pcd_scene(rng, n=6000):
    p = rng.uniform([486, 486, 498], [518, 518, 502], (n, 3))
    p = np.concatenate([p, p[:300], np.full((50, 3), 505.125), rng.uniform(300, 700, (200, 3))])  # duplicates and far points
    return p


# ---- running eval.py ----------------------------------------------------------------------------------------------------

def _open3d_standin(registry, written):
    o3d = types.ModuleType("open3d")

    class _Cloud:
        def __init__(self, points=None):
            self.points = points
            self.colors = None

    class _Mesh:
        def __init__(self, v, f):
            self.vertices, self.triangles = v, f

    def read_point_cloud(path):
        return _Cloud(registry[os.path.basename(path)].copy())

    def read_triangle_mesh(path):
        v, f = registry[os.path.basename(path)]
        return _Mesh(v.copy(), f.copy())

    def write_point_cloud(path, pcd):
        written[os.path.basename(path)] = (np.asarray(pcd.points).copy(), np.asarray(pcd.colors).copy())
        return True

    o3d.geometry = types.SimpleNamespace(PointCloud=_Cloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    o3d.io = types.SimpleNamespace(read_point_cloud=read_point_cloud, read_triangle_mesh=read_triangle_mesh, write_point_cloud=write_point_cloud)
    return o3d


def run_eval(reference, data, mode, gt, scan, seed, extra_args):
    import sklearn.neighbors  # noqa: F401  imported before the rng is replaced: scipy.stats draws examples at import time
    import tqdm  # noqa: F401
    obs, bb, res, plane, stl = gt
    registry, written, rec = {"data.ply": data, f"stl{scan:03}_total.ply": stl}, {}, {}
    real_rng = np.random.default_rng

    class _RecordingRng:
        def __init__(self, *a, **k):
            self.g = real_rng(seed)

        def shuffle(self, x, axis=0):
            rec["original"] = x.copy()
            rec["perm"] = real_rng(seed).permutation(len(x))
            self.g.shuffle(x, axis=axis)
            assert np.array_equal(x, rec["original"][rec["perm"]]), "the shuffle is not original[perm]"

    with tempfile.TemporaryDirectory() as d:
        os.makedirs(f"{d}/ObsMask")
        scipy.io.savemat(f"{d}/ObsMask/ObsMask{scan}_10.mat", {"ObsMask": obs, "BB": bb, "Res": res})
        scipy.io.savemat(f"{d}/ObsMask/Plane{scan}.mat", {"P": plane})
        saved = sys.argv, sys.modules.get("open3d"), np.random.default_rng
        sys.argv = ["eval.py", "--data", f"{d}/data.ply", "--scan", str(scan), "--mode", mode, "--dataset_dir", d, "--vis_out_dir", d] + extra_args
        sys.modules["open3d"] = _open3d_standin(registry, written)
        np.random.default_rng = _RecordingRng
        try:
            g = runpy.run_path(os.path.join(reference, "dtu_eval", "eval.py"), run_name="__main__")
        finally:
            sys.argv, np.random.default_rng = saved[0], saved[2]
            if saved[1] is None:
                sys.modules.pop("open3d", None)
            else:
                sys.modules["open3d"] = saved[1]
    return g, rec, written


# ---- running cull_mesh --------------------------------------------------------------------------------------------------

class _Mesh:
    """trimesh's update_vertices(mask) / update_faces(mask) on plain arrays."""

    def __init__(self, vertices, faces):
        self.vertices, self.faces = vertices, faces

    def update_vertices(self, mask):
        idx = np.nonzero(mask)[0]
        inverse = np.zeros(len(self.vertices), np.int64)
        inverse[idx] = np.arange(len(idx))
        self.faces = inverse[self.faces.reshape(-1)].reshape(-1, 3)
        self.vertices = self.vertices[idx]

    def update_faces(self, mask):
        self.faces = self.faces[mask]


def reference_cull(reference, cameras, vertices, faces):
    import torch
    import torch.nn.functional as F
    src = open(os.path.join(reference, "evaluate_dtu_mesh.py")).read()
    tree = ast.parse(src)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("fov2focal", "cull_mesh")]
    ns = {"torch": torch, "F": F, "np": np, "math": __import__("math"),
          "binary_dilation": lambda img, fp: ndimage.binary_dilation(img, structure=fp, border_value=0),
          "disk": lambda r: (np.add.outer(np.arange(-r, r + 1) ** 2, np.arange(-r, r + 1) ** 2) <= r * r).astype(np.uint8)}
    exec(compile(ast.Module(body=fns, type_ignores=[]), "evaluate_dtu_mesh.py", "exec"), ns)
    saved = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        mesh = ns["cull_mesh"](cameras, _Mesh(vertices.copy(), faces.copy()))
    finally:
        torch.Tensor.cuda = saved
    return mesh.vertices, mesh.faces


def cull_scene(rng, n_views=5, W=64, H=48, n_vert=3000):
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from tsdf_scenes import look_at
    ctr = np.array([500.0, 500.0, 500.0])
    verts = ctr + rng.normal(0, 40, (n_vert, 3))
    faces = rng.integers(0, n_vert, (2 * n_vert, 3))
    cams = []
    for k in range(n_views):
        ang = 2 * np.pi * k / n_views
        eye = ctr + np.array([300 * np.cos(ang), 300 * np.sin(ang), 120.0])
        E = look_at(eye, ctr + rng.normal(0, 5, 3))
        mask = np.zeros((1, H, W), np.float32)
        yy, xx = np.mgrid[0:H, 0:W]
        mask[0][(xx - W / 2 - 4 * k) ** 2 / (W / 4) ** 2 + (yy - H / 2) ** 2 / (H / 4) ** 2 < 1] = 1.0
        mask[0][rng.random((H, W)) < 0.01] = 1.0
        cams.append(types.SimpleNamespace(world_view_transform=torch.tensor(E.T, dtype=torch.float32), FoVx=0.9, FoVy=0.9 * H / W,
                                          image_width=W, image_height=H, gt_mask=torch.tensor(mask)))
    return cams, verts, faces


# ---- main -----------------------------------------------------------------------------------------------------------------

SCANS = [  # name, mode, scan id, seed, density, extra eval.py arguments
    ("mesh_a", "mesh", 1, 11, 0.2, ["--patch_size", "3", "--max_dist", "1.5"]),
    ("mesh_b", "mesh", 2, 12, 0.35, ["--downsample_density", "0.35", "--patch_size", "60"]),
    ("pcd", "pcd", 3, 13, 0.2, ["--patch_size", "2", "--max_dist", "4", "--visualize_threshold", "2"]),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference")))
    ap.add_argument("--out", default=os.path.join(ROOT, "golden_out"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    for name, mode, scan, seed, density, extra in SCANS:
        rng = np.random.default_rng(seed)
        if mode == "mesh":
            v, f = _mesh_scene(rng)
            data = (v, f)
        else:
            data = _pcd_scene(rng)
        gt = _ground_truth(rng, 4000)
        g, rec, written = run_eval(a.reference, data, mode, gt, scan, seed, extra)
        args = g["args"]
        obs, bb, res, plane, stl = gt
        out = dict(mode=np.array(mode), scan=np.array(scan), density=np.array(args.downsample_density), patch=np.array(args.patch_size),
                   max_dist=np.array(args.max_dist), vis=np.array(args.visualize_threshold), obs_mask=obs, bb=bb, res=res, plane=plane, stl=stl,
                   original=rec["original"], perm=rec["perm"], kept=g["mask"],
                   in_obs=np.where(g["inbound"])[0][g["grid_inbound"]][g["in_obs"]], dist_d2s=g["dist_d2s"][:, 0], dist_s2d=g["dist_s2d"][:, 0],
                   means=np.array([g["mean_d2s"], g["mean_s2d"], g["over_all"]]),
                   data_color=written[f"vis_{scan:03}_d2s.ply"][1], stl_color=written[f"vis_{scan:03}_s2d.ply"][1])
        if mode == "mesh":
            out.update(vertices=data[0], faces=data[1])
        else:
            out.update(points=data)
        np.savez_compressed(os.path.join(a.out, name + ".npz"), **out)
        print(name, len(rec["original"]), "points,", int(g["mask"].sum()), "kept, means", out["means"], flush=True)

    rng = np.random.default_rng(21)
    cams, verts, faces = cull_scene(rng)
    cv, cf = reference_cull(a.reference, cams, verts, faces)
    np.savez_compressed(os.path.join(a.out, "cull.npz"), vertices=verts, faces=faces,
                        w2c_t=np.stack([c.world_view_transform.numpy() for c in cams]), fov=np.array([[c.FoVx, c.FoVy] for c in cams]),
                        size=np.array([cams[0].image_width, cams[0].image_height]), masks=np.stack([c.gt_mask.numpy() for c in cams]),
                        culled_vertices=cv, culled_faces=cf)
    print("cull", len(verts), "->", len(cv), "vertices,", len(faces), "->", len(cf), "faces", flush=True)


if __name__ == "__main__":
    main()
