"""Fixtures of the tetrahedra mesh extraction, made by the reference's own code on the CPU: tests/golden/tetra/*.npz.

Imports the UNMODIFIED ``mesh_extract_tetrahedra.py``, ``utils/tetmesh.py`` and ``scene/gaussian_model.py`` from the reference
checkout (beside the repository, or $RADE_GS_REFERENCE, or --reference) and runs ``marching_tetrahedra_with_binary_search``
as written.  The reference says ``.cuda()`` and ``device="cuda"``; for the run those mean the CPU (the shim of
gen_golden_fused.py, extended to ``torch.ones`` / ``torch.zeros``).  In-process stand-ins replace what is not installed:

* ``trimesh``: ``creation.box`` (its unit cube, vertex order 000, 001, 010, ..., 111, minus 0.5) and a ``Trimesh`` that applies
  ``update_vertices`` / ``update_faces`` as trimesh does and records what ``export`` would write;
* ``tetranerf``: ``cpp.triangulate`` returns the cells the generator fixed (scipy's Delaunay of the tetra points);
* ``diff_gaussian_rasterization``: names only; ``integrate`` is replaced by the analytic stand-in of tests/tetra_scenes.py,
  which gives the same bits on the CPU and the GPU.

Every evaluation is checked for two margins, in fp64, and the case is re-seeded if one fails: no sampled mask value within
1e-5 of 0.5, and no |distance - scale| within 1e-6 of the scale.  Within them, decisions cannot depend on how grid_sample or
torch.norm round.  The second cannot hold everywhere: adjacent box corners along a Gaussian's longest axis are exactly
s_left + s_right apart.  For those ties (counted in ``filter_ties``) the case is re-seeded unless torch.norm, as the script
runs it here, and the contract's fp32 formula decide alike.

Usage:  python tools/gen_golden_tetra.py [--reference /path/to/RaDe-GS] [--out DIR]
"""
from __future__ import annotations

import argparse
import io
import os
import sys
import tempfile
import types
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tetra_model as model  # noqa: E402
import tetra_scenes as scenes  # noqa: E402

CASES = {
    # name: (seed, Gaussians, views, H, W, gt_mask on every n-th view (None: never), blank masks)
    "sphere_gt": (11, 160, 3, 48, 64, 2, False),
    "sphere_nogt": (23, 120, 2, 40, 56, None, False),
    "empty": (37, 40, 2, 24, 32, 1, True),
}


# ---- stand-ins ------------------------------------------------------------------------------------------------------------

class _Trimesh:
    """trimesh.Trimesh(process=False) as far as the script uses it: update_vertices(mask) renumbers the faces through the
    inverse of the mask and keeps the masked vertices, update_faces(mask) keeps the masked faces, export records the result."""
    exported = []

    def __init__(self, vertices=None, faces=None, process=True):
        self.vertices = np.asarray(vertices)
        self.faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)

    def update_vertices(self, mask):
        mask = np.asanyarray(mask)
        if (mask.dtype.name == "bool" and mask.all()) or len(mask) == 0 or len(self.vertices) == 0:
            return
        inverse = np.zeros(len(self.vertices), dtype=np.int64)
        inverse[mask] = np.arange(mask.sum())
        self.faces = inverse[self.faces.reshape(-1)].reshape((-1, 3))
        self.vertices = self.vertices[mask]

    def update_faces(self, mask):
        self.faces = self.faces[np.asanyarray(mask)]

    def export(self, path):
        _Trimesh.exported.append((self.vertices.copy(), self.faces.copy()))


def _box():
    v = np.array([0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 1, 1, 1, 0, 0, 1, 0, 1, 1, 1, 0, 1, 1, 1], dtype=np.float64).reshape(-1, 3) - 0.5
    return types.SimpleNamespace(vertices=v)


_CELLS = {"cells": None}


def install_stubs(ref):
    tm = types.ModuleType("trimesh")
    tm.creation = types.SimpleNamespace(box=_box)
    tm.Trimesh = _Trimesh
    sys.modules["trimesh"] = tm
    ext = types.ModuleType("tetranerf.utils.extension")
    ext.cpp = types.SimpleNamespace(triangulate=lambda points: torch.from_numpy(_CELLS["cells"]))
    sys.modules["tetranerf"] = types.ModuleType("tetranerf")
    sys.modules["tetranerf.utils"] = types.ModuleType("tetranerf.utils")
    sys.modules["tetranerf.utils.extension"] = ext
    dgr = types.ModuleType("diff_gaussian_rasterization")
    dgr.GaussianRasterizationSettings = dgr.GaussianRasterizer = None
    sys.modules["diff_gaussian_rasterization"] = dgr
    sys.path[:0] = [os.path.join(ROOT, "tests", "ref_stubs"), ref]

    torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
    torch.nn.Module.cuda = lambda self, *a, **k: self         # noqa: E731
    for name in ("tensor", "ones", "zeros"):
        orig = getattr(torch, name)

        def on_cpu(*a, _orig=orig, **k):
            if str(k.get("device", "")).startswith("cuda"):
                k["device"] = "cpu"
            return _orig(*a, **k)
        setattr(torch, name, on_cpu)


# ---- one case -------------------------------------------------------------------------------------------------------------

class MarginError(Exception):
    pass


def run_case(mt, GaussianModel, seed, P, n_views, H, W, gt_every, blank):
    xyz, log_scale, rot, filt = scenes.make_gaussians(seed, P)
    views = scenes.make_views(seed + 1, n_views, H, W, gt_every, blank)
    g = GaussianModel(0)
    g._xyz = torch.from_numpy(xyz)
    g._scaling = torch.from_numpy(log_scale)
    g._rotation = torch.from_numpy(rot)
    g.filter_3D = torch.from_numpy(filt)
    s3d = g.get_scaling_with_3D_filter.numpy().copy()

    rec = {"tetra": None, "evals": [], "march": None}
    orig_tp = GaussianModel.get_tetra_points

    def get_tetra_points(self):
        pts, sc = orig_tp(self)
        rec["tetra"] = (pts.numpy().copy(), sc.numpy().copy())
        from scipy.spatial import Delaunay
        _CELLS["cells"] = np.ascontiguousarray(Delaunay(pts.numpy().astype(np.float64)).simplices, dtype=np.int32)
        return pts, sc

    def integrate(points, view, gaussians, pipeline, background, kernel_size):
        ret = scenes.integrate(points, view)
        v = scenes.sample_mask_f64(view, ret["point_coordinate"].numpy())
        if np.any(np.abs(v - 0.5) < 1e-5):
            raise MarginError("a sampled mask value lies within 1e-5 of 0.5")
        return ret

    orig_eval = mt.evaluage_cull_alpha

    def evaluage_cull_alpha(points, views_, masks, *a):
        sdf = orig_eval(points, views_, masks, *a)
        rec["evals"].append((points.numpy().copy(), sdf.numpy().copy()))
        return sdf

    orig_march = mt.marching_tetrahedra

    def marching_tetrahedra(*a):
        out = orig_march(*a)
        (ends, esdf), escl, faces, interp = out[0][0], out[1][0], out[2][0], out[3][0]
        rec["march"] = tuple(t.numpy().copy() for t in (ends, esdf, escl, faces, interp))
        d = ends[:, 0].double() - ends[:, 1].double()
        dist = d.norm(dim=-1).numpy()
        s = escl[:, 0, 0].double().numpy() + escl[:, 1, 0].double().numpy()
        near = np.abs(dist - s) <= 1e-6 * np.abs(s)
        # Adjacent box corners along a Gaussian's longest axis are exactly s_left + s_right apart, so such ties exist by
        # construction.  There the fixture is usable only when the reference's torch.norm and the contract's fp32 formula agree.
        ref_keep = (torch.norm(ends[:, 0] - ends[:, 1], dim=-1) <= escl[:, 0, 0] + escl[:, 1, 0]).numpy()
        e = ends.numpy()
        dd = e[:, 0] - e[:, 1]
        f32 = np.sqrt(model.fma32(dd[:, 2], dd[:, 2], model.fma32(dd[:, 1], dd[:, 1], dd[:, 0] * dd[:, 0])))
        model_keep = f32 <= escl[:, 0, 0].numpy() + escl[:, 1, 0].numpy()
        if np.any(near & (ref_keep != model_keep)):
            raise MarginError("an edge length within 1e-6 of its scale is decided differently by torch.norm and the contract")
        rec["ties"] = int(near.sum())
        return out

    GaussianModel.get_tetra_points = get_tetra_points
    mt.integrate = integrate
    mt.evaluage_cull_alpha = evaluage_cull_alpha
    mt.marching_tetrahedra = marching_tetrahedra
    mt.tqdm = lambda it, **k: it
    _Trimesh.exported.clear()
    try:
        with tempfile.TemporaryDirectory() as tmp, torch.no_grad():
            mt.marching_tetrahedra_with_binary_search(tmp, "test", 0, views, g, None, None, 0.0)
    finally:
        GaussianModel.get_tetra_points = orig_tp
        mt.evaluage_cull_alpha = orig_eval
        mt.marching_tetrahedra = orig_march

    pts, sc = rec["tetra"]
    ends, esdf, escl, faces, interp = rec["march"]
    verts, fout = _Trimesh.exported[-1]
    out = {
        "xyz": xyz, "scaling": s3d, "rotation": rot, "points": pts, "scales": sc, "points_f64": tetra_points_f64(xyz, s3d, rot),
        "cells": _CELLS["cells"], "sdf": rec["evals"][0][1],
        "ends": ends, "end_sdf": esdf, "end_scales": escl, "faces": faces, "interp_v": interp,
        "n_steps": np.int64(len(rec["evals"]) - 1), "filter_ties": np.int64(rec.get("ties", 0)), "vertices": verts.astype(np.float32), "out_faces": fout.astype(np.int64),
    }
    for k, (p, s) in enumerate(rec["evals"][1:]):
        out[f"mid_{k}"], out[f"mid_sdf_{k}"] = p, s
    for i, v in enumerate(views):
        out[f"view{i}_axes"] = np.array(v.axes, np.int64)
        out[f"view{i}_signs"] = np.array(v.signs, np.float32)
        out[f"view{i}_center"] = v.center
        out[f"view{i}_focal_k"] = np.array([v.focal, v.k], np.float64)
        out[f"view{i}_mask"] = v.mask
        if v.gt_mask is not None:
            out[f"view{i}_gt"] = v.gt_mask
    out["n_views"] = np.int64(len(views))
    return out


def tetra_points_f64(xyz, s, rot):
    """get_tetra_points evaluated in fp64 from the fp32 inputs: the arbiter of the stage-1 tolerance."""
    q = rot.astype(np.float64)
    q = q / np.sqrt((q * q).sum(1, keepdims=True))
    r, x, y, z = q.T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                  2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    corners = (_box().vertices * 2)                                         # [8, 3]
    s3 = s.astype(np.float64) * 3
    v = np.einsum("prc,pkc->pkr", R, corners[None] * s3[:, None, :]) + xyz.astype(np.float64)[:, None, :]
    return np.concatenate([v.reshape(-1, 3), xyz.astype(np.float64)])


def _write_npz(path, arrays):
    """np.savez_compressed with fixed timestamps, so the bytes depend on the arrays only."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.save(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference"))
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "tetra"))
    args = ap.parse_args()
    install_stubs(args.reference)
    torch.set_num_threads(4)
    import mesh_extract_tetrahedra as mt
    from scene.gaussian_model import GaussianModel
    os.makedirs(args.out, exist_ok=True)
    for name, (seed, P, n_views, H, W, gt_every, blank) in CASES.items():
        for attempt in range(50):
            try:
                out = run_case(mt, GaussianModel, seed + 1000 * attempt, P, n_views, H, W, gt_every, blank)
                break
            except MarginError as e:
                print(f"[{name}] seed {seed + 1000 * attempt}: {e}; re-seeding", flush=True)
        else:
            raise SystemExit(f"{name}: no seed met the margins")
        out["seed"] = np.int64(seed + 1000 * attempt)
        _write_npz(os.path.join(args.out, name + ".npz"), out)
        print(f"[{name}] {out['points'].shape[0]} points, {out['cells'].shape[0]} tets, {out['ends'].shape[0]} crossing edges, "
              f"{out['faces'].shape[0]} faces -> {out['vertices'].shape[0]} vertices, {out['out_faces'].shape[0]} faces", flush=True)


if __name__ == "__main__":
    main()
