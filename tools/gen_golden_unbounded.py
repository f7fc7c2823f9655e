"""Fixtures of the unbounded-scene mesh, made by the reference's own code on the CPU: tests/golden/unbounded/unbounded.npz.

Imports the UNMODIFIED ``utils/mesh_utils.py``, ``utils/mcube_utils.py`` and ``utils/render_utils.py`` from the reference
checkout (beside the repository, or $RADE_GS_REFERENCE, or --reference) with in-process stand-ins for ``open3d``,
``trimesh``, ``skimage``, ``mediapy`` and ``matplotlib``; ``.cuda()`` and ``device="cuda"`` mean the CPU for the run.  Its
``GaussianExtractor.reconstruction`` cannot run (it calls ``render`` without ``kernel_size`` and reads ``middepth``), so
the extractor's ``depthmaps``, ``rgbmaps``, ``depth_normals`` and ``viewpoint_stack`` are set to the analytic views of
tests/unbounded_scenes.py.  Then ``extract_mesh_unbounded(resolution=512)`` runs as written: 134 M samples on the CPU.

The ``skimage.measure.marching_cubes`` stand-in records the 512^3 volume and returns planted vertices (lattice points
advanced by t along one axis, in the spacing units skimage returns), so the fixture also pins the uncontraction and clip
and the colouring of vertices.  The ``trimesh`` stand-in concatenates and merges by this repository's rule (the planted
vertices are far apart, so the merge changes nothing).

The fp64 SDF is stored as its difference from the fp32 one, the decision marks as bits, and the three planes' voxel
indices implicitly (``plane_voxels``), which keeps the file small.  Stored: the inputs (depth, RGB, cameras, xyz); center, radius, voxel_size and R as the reference computed them; the SDF
at three full planes, random voxels and near-surface voxels of the volume; the planted vertex positions, the world
vertices and their colours; and for each of these the same expressions in fp64 (tests/unbounded_scenes.torch_tsdf, inputs
as the fixture holds them, centre and radius unrounded), whose difference from the fp32 reference gives the tests' bound.
A sample or vertex whose fp64 distance to a discrete decision (|pix| = 1, w = 0, sdf = -trunc, |s| = 1, |p| = 1) is below
1e-5 is marked and counted.  The SHA-256 of the full volume is stored for the record.

Usage:  python tools/gen_golden_unbounded.py [--reference /path/to/RaDe-GS] [--out DIR]
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import unbounded_scenes as S  # noqa: E402

RES = 512
MARGIN = 1e-5
_REC = {}


class _Trimesh:
    def __init__(self, vertices=None, faces=None, vertex_normals=None, **_):
        self.vertices = np.asarray(vertices, np.float64)
        self.faces = np.asarray(faces, np.int64).reshape(-1, 3)

    def merge_vertices(self, digits_vertex=6):
        keys = np.rint(self.vertices * 10.0 ** digits_vertex).astype(np.int64)
        _, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
        rep = first[inv.reshape(-1)]
        surv = rep == np.arange(len(self.vertices))
        newid = np.cumsum(surv) - surv
        self.faces = newid[rep[self.faces]]
        self.vertices = self.vertices[surv]

    @property
    def as_open3d(self):
        return types.SimpleNamespace(vertices=self.vertices, triangles=self.faces, vertex_colors=None)


def _concatenate(meshes):
    v, f, base = [], [], 0
    for m in meshes:
        v.append(m.vertices)
        f.append(m.faces + base)
        base += len(m.vertices)
    return _Trimesh(np.concatenate(v), np.concatenate(f))


def _marching_cubes(volume, level=0, spacing=(1.0, 1.0, 1.0), **_):
    _REC["volume"] = np.array(volume, np.float32, copy=True)
    _REC["level"] = level
    _REC["spacing"] = tuple(float(s) for s in spacing)
    idx = _REC["planted"]
    verts = idx * np.asarray(spacing, np.float64)
    faces = np.arange(len(idx) - len(idx) % 3).reshape(-1, 3)
    return verts, faces, np.zeros_like(verts), np.zeros(len(verts))


def install_stubs(ref):
    tm = types.ModuleType("trimesh")
    tm.Trimesh = _Trimesh
    tm.util = types.SimpleNamespace(concatenate=_concatenate)
    sys.modules["trimesh"] = tm
    o3d = types.ModuleType("open3d")
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    sys.modules["open3d"] = o3d
    sk = types.ModuleType("skimage")
    sk.measure = types.SimpleNamespace(marching_cubes=_marching_cubes)
    sys.modules["skimage"] = sk
    sys.modules["skimage.measure"] = sk.measure
    sys.modules["mediapy"] = types.ModuleType("mediapy")
    mpl = types.ModuleType("matplotlib")
    mpl.cm = types.SimpleNamespace()
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.cm"] = mpl.cm
    sys.path[:0] = [ref]
    torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
    torch.cuda.empty_cache = lambda: None
    for name in ("tensor", "ones", "zeros"):
        orig = getattr(torch, name)

        def on_cpu(*a, _orig=orig, **k):
            if str(k.get("device", "")).startswith("cuda"):
                k["device"] = "cpu"
            return _orig(*a, **k)
        setattr(torch, name, on_cpu)


def scene():
    d, c, wv, fp = S.views(6, W=64, H=48, seed=0)
    g = np.random.default_rng(5)
    far = g.normal(size=(1500, 3))
    far = S.SKY_R * far / np.linalg.norm(far, axis=1, keepdims=True)
    xyz = torch.cat([S.sphere_xyz(4000), torch.from_numpy(far.astype(np.float32))])
    return d, c, wv, fp, xyz


def planted(n):
    """Lattice points advanced by t in [0, 1) along one axis, in index units: [n, 3] float64."""
    g = np.random.default_rng(8)
    idx = g.integers(0, RES - 1, (n, 3)).astype(np.float64)
    axis = g.integers(0, 3, n)
    idx[np.arange(n), axis] += g.random(n)
    return idx


def plane_voxels():
    """The three full planes x = 128, y = 300, z = 411 (stored implicitly: tests rebuild them with this function's rule)."""
    ax = np.arange(RES)
    return np.concatenate([np.stack(np.meshgrid([128], ax, ax, indexing="ij"), -1).reshape(-1, 3),
                           np.stack(np.meshgrid(ax, [300], ax, indexing="ij"), -1).reshape(-1, 3),
                           np.stack(np.meshgrid(ax, ax, [411], indexing="ij"), -1).reshape(-1, 3)]).astype(np.int32)


def sampled_voxels(vol):
    g = np.random.default_rng(9)
    rand = g.integers(0, RES, (20000, 3))
    near = np.argwhere(np.abs(vol) < 0.5)
    near = near[g.choice(len(near), min(20000, len(near)), replace=False)]
    return np.concatenate([plane_voxels(), rand.astype(np.int32), near.astype(np.int32)]).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference"))
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "unbounded"))
    args = ap.parse_args()
    install_stubs(args.reference)
    from utils import mesh_utils

    d, c, wv, fp, xyz = scene()
    V = d.shape[0]
    views = [types.SimpleNamespace(world_view_transform=wv[i], full_proj_transform=fp[i]) for i in range(V)]
    ex = mesh_utils.GaussianExtractor(types.SimpleNamespace(get_xyz=xyz), render=lambda *a, **k: None, pipe=None)
    ex.viewpoint_stack = views
    ex.depthmaps = d[:, None].clone()
    ex.rgbmaps = c.clone()
    ex.depth_normals = torch.zeros_like(c)
    _REC["planted"] = planted(3000)

    # what the reference computes on the way (same expressions, recorded for the normalisation check)
    from utils.render_utils import focus_point_fn
    c2ws = np.array([np.linalg.inv(np.asarray((cam.world_view_transform.T).cpu().numpy())) for cam in views])
    poses = c2ws[:, :3, :] @ np.diag([1, -1, -1, 1])
    center = focus_point_fn(poses)
    radius = np.linalg.norm(c2ws[:, :3, 3] - center, axis=-1).min()
    voxel_size = radius * 2 / RES

    # record the arguments the reference hands to marching_cubes_with_contraction: R and, from the closures, the centre
    # (fp32 tensor), radius and voxel size it uses
    from utils import mcube_utils
    orig = mcube_utils.marching_cubes_with_contraction

    def recording(**kw):
        _REC["call"] = kw
        return orig(**kw)
    mcube_utils.marching_cubes_with_contraction = recording
    print("running extract_mesh_unbounded(resolution=512) on the CPU ...", flush=True)
    mesh = ex.extract_mesh_unbounded(resolution=RES)
    kw = _REC["call"]
    cells = lambda f: {n: c.cell_contents for n, c in zip(f.__code__.co_freevars, f.__closure__)}  # noqa: E731
    un = cells(kw["inv_contraction"])["unnormalize"]
    center32 = cells(un)["center"].numpy()
    assert cells(un)["radius"] == radius and cells(kw["sdf"])["voxel_size"] == voxel_size and np.array_equal(center32, np.float32(center))
    R = kw["bounding_box_max"][0]
    vol = _REC["volume"]
    spacing = np.asarray(_REC["spacing"])
    world = np.asarray(mesh.vertices, np.float32)
    colors = np.asarray(mesh.vertex_colors, np.float32)

    vox = sampled_voxels(vol)
    sdf32 = vol[vox[:, 0], vox[:, 1], vox[:, 2]]
    xs = np.linspace(-R, R, RES)
    s = torch.from_numpy(np.stack([xs[vox[:, 0]], xs[vox[:, 1]], xs[vox[:, 2]]], -1).astype(np.float32))
    t64, _, m_sdf = S.torch_tsdf(s, center, radius, voxel_size, d.double(), fp.double(), torch.float64, margins=True)

    idx = _REC["planted"]
    pos = idx * spacing + np.float64(-R)           # what the stand-in returned plus x_min = -R, as the reference adds them
    y = torch.from_numpy(pos)
    mag = torch.linalg.norm(y, dim=-1)[..., None]
    w64 = torch.where(mag < 1, y, 1 / (2 - mag) * (y / mag)) * radius + torch.from_numpy(center)
    w64 = w64.clamp(-32, 32).numpy()
    m_w = (mag[:, 0] - 1).abs().numpy()
    _, _, col64, m_c = S.torch_tsdf(torch.from_numpy(world).double(), center, radius, voxel_size, d.double(), fp.double(), torch.float64,
                                    rgbs=c.double(), contracted=False, margins=True)

    os.makedirs(args.out, exist_ok=True)
    out = os.path.join(args.out, "unbounded.npz")
    np.savez_compressed(
        out, depth=d.numpy(), rgb=c.numpy(), world_view=wv.numpy(), full_proj=fp.numpy(), xyz=xyz.numpy(),
        center=center, radius=np.float64(radius), voxel_size=np.float64(voxel_size), R=np.float64(R), R_dtype=str(np.asarray(R).dtype),
        spacing=spacing, center32=center32, volume_sha256=hashlib.sha256(vol.tobytes()).hexdigest(),
        voxels=vox[3 * RES * RES:], sdf=sdf32, sdf64_minus_sdf=(t64.numpy() - sdf32).astype(np.float32),
        sdf_decided=np.packbits(m_sdf.numpy() > MARGIN),
        planted=idx, vertices=world, vertices64=w64, vertex_decided=m_w > MARGIN,
        colors=colors, colors64=col64.numpy(), color_decided=m_c.numpy() > MARGIN)
    keep = m_sdf.numpy() > MARGIN
    print(f"wrote {out} ({os.path.getsize(out) / 1024:.0f} KB): center {center}, radius {radius:.6g}, R {R!r} ({np.asarray(R).dtype}), "
          f"{len(vox)} voxels ({(~keep).sum()} within {MARGIN} of a decision), max |fp32 - fp64| {np.abs(sdf32 - t64.numpy())[keep].max():.3g}; "
          f"{len(world)} vertices, max |fp32 - fp64| {np.abs(world - w64).max():.3g}, colours {np.abs(colors - col64.numpy())[m_c.numpy() > MARGIN].max():.3g}")


if __name__ == "__main__":
    main()
