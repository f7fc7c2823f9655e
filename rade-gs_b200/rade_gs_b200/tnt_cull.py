"""Tanks and Temples mesh culling on the GPU: the reference's ``eval_tnt/cull_mesh.py``, the step the TNT protocol runs
before scoring, without pyrender, OpenGL, trimesh or Open3D.

    from rade_gs_b200 import ply_io, tnt_cull, tnt_eval
    vertices, faces = ply_io.load_triangle_mesh_ply("recon.ply")
    c2w = tnt_cull.load_poses("Barn_COLMAP_SfM.log")
    v, f, valid, counts = tnt_cull.cull_mesh(vertices, faces, c2w)
    ply_io.save_triangle_mesh_ply("recon_cull.ply", v, f)

or, for files, ``python -m rade_gs_b200.tnt_cull --traj-path <log> --ply-path <mesh.ply>``, which writes
``<mesh>_cull.ply`` for ``python -m rade_gs_b200.tnt_eval``.

For every camera the mesh's depth is rasterized (both facings, nearest surface, one exact sample at each pixel centre)
and every vertex is tested against it as ``Mesher.point_masks`` does; a vertex seen by at least ``min_views`` cameras
is valid, a face is kept when its three vertices are valid, and a vertex is kept when a kept face uses it.  Only one depth
map is held at a time, so memory is O(V + F + H W) whatever the number of views.  The contracts of the two kernels are at
``rgs_tnt_mesh_depth`` and ``rgs_tnt_visibility_count`` in include/rgs_b200.h; they are in csrc/rgs_tnt_cull.cu.

Deliberate differences from the reference:

* one camera convention for both steps.  The shipped script renders the depth with pyrender, whose cameras look down -z,
  from the OpenCV poses of the trajectory (its OpenCV-to-OpenGL flip is commented out), so each depth map shows what
  lies behind and mirrored, while the points are projected looking down +z.  Here both use the OpenCV pose.
  ``depth_c2w=c2w @ diag(1, -1, -1, 1)`` (CLI ``--shipped-depth-pose``) renders from the pose pyrender used, which
  reproduces the shipped script;
* the mesh is taken as read, with no ``merge_vertices``: merged vertices share a position and so a decision, so the kept
  faces are the same and only the vertex numbering differs;
* ``.json`` trajectories are rejected, as ``tnt_eval.load_trajectory`` does;
* pyrender's coverage rule, multisample resolve and 24-bit depth buffer are not reproduced: each pixel holds one exact
  fp32 sample at its centre;
* ``w2c`` is the fp64 inverse of the fp32 pose rounded to fp32 (torch inverts in fp32), and the projection's products
  are rounded one by one; both move a decision only when it lies within an ulp of its threshold;
* the PLY byte layout is this package's (``ply_io.save_triangle_mesh_ply``).

Inputs with a NaN or infinite coordinate raise ``ValueError``.  There is no CPU path: the work runs on a CUDA device.
"""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from diff_gaussian_rasterization import _C

from . import ply_io, tnt_eval
from .dtu_eval import _device

# cull_mesh.py:405-411: the Tanks and Temples camera
H, W = 1080, 1920
FX, FY = 1163.8678928442187, 1172.793101201448
CX, CY = 962.3120628412543, 542.0667209577691
FAR, ZNEAR, EPS, MIN_VIEWS = 20.0, 0.01, 0.005, 20
OPENGL_FLIP = np.diag([1.0, -1.0, -1.0, 1.0])


def load_poses(path: str) -> np.ndarray:
    """cull_mesh.py's ``get_traj``: float64 [n, 4, 4] camera-to-world poses from a ``.log`` or ``.npy`` trajectory; 3x4
    ``.npy`` poses get the row (0, 0, 0, 1)."""
    if path.endswith(".npy"):
        t = np.asarray(np.load(path), np.float64)
        if t.ndim == 3 and t.shape[1:] == (3, 4):
            t = np.concatenate([t, np.broadcast_to([[[0.0, 0.0, 0.0, 1.0]]], (len(t), 1, 4))], axis=1)
        if t.ndim != 3 or t.shape[1:] != (4, 4):
            raise ValueError(f"{path}: a trajectory must be [n, 4, 4] or [n, 3, 4], got {t.shape}")
        return t
    return tnt_eval.load_trajectory(path)


def _poses(c2w, name: str = "c2w") -> np.ndarray:
    c = (c2w.detach().cpu().numpy() if isinstance(c2w, torch.Tensor) else np.asarray(c2w)).astype(np.float64)
    if c.ndim == 2:
        c = c[None]
    if c.ndim != 3 or c.shape[1:] != (4, 4):
        raise ValueError(f"{name} must be [n, 4, 4], got {c.shape}")
    if not np.isfinite(c).all():
        raise ValueError(f"{name} has NaN or infinite entries")
    return c


def _w2c(c2w: np.ndarray) -> list:
    """Per view rows 0..2 of w2c as 12 floats: the fp64 inverse of the fp32-rounded pose, rounded to fp32."""
    inv = np.linalg.inv(c2w.astype(np.float32).astype(np.float64))
    return [list(map(float, r)) for r in inv[:, :3, :].astype(np.float32).reshape(-1, 12)]


def _mesh(vertices, faces, dev):
    v = vertices.detach() if isinstance(vertices, torch.Tensor) else torch.as_tensor(np.asarray(vertices))
    v = v.to(dev)
    if v.dim() != 2 or v.shape[1] != 3:
        raise ValueError(f"vertices must be [V, 3], got {tuple(v.shape)}")
    if v.numel() and not bool(torch.isfinite(v).all()):
        raise ValueError("vertices has NaN or infinite coordinates")
    f = (faces.detach() if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces))).to(dev, torch.int64).reshape(-1, 3)
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError("face index out of [0, V)")
    if v.shape[0] >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 vertices")
    return v, f


def _check_camera(H, W, znear, zfar):
    if int(H) < 2 or int(W) < 2:
        raise ValueError(f"the image must be at least 2 x 2, got {H} x {W}")
    if not (0 < znear < zfar):
        raise ValueError(f"need 0 < znear < zfar, got {znear}, {zfar}")


def render_depth(vertices, faces, c2w, H, W, fx, fy, cx, cy, znear=ZNEAR, zfar=FAR, device="cuda") -> torch.Tensor:
    """float32 [n, H, W]: the mesh's camera-space depth at every pixel centre from each OpenCV pose (0 where nothing lies
    in [znear, zfar]).  Replaces ``extract_depth_from_mesh``; meant for inspection and tests (it holds every map)."""
    dev = _device(device)
    _check_camera(H, W, znear, zfar)
    v, f = _mesh(vertices, faces, dev)
    v32, f32 = v.float().contiguous(), f.to(torch.int32).contiguous()
    out = torch.zeros(len(_poses(c2w)), int(H), int(W), device=dev)
    for k, m in enumerate(_w2c(_poses(c2w))):
        out[k] = _C._tnt_cull.mesh_depth(v32, f32, m, fx, fy, cx, cy, int(H), int(W), znear, zfar)
    return out


def point_masks(points, depths, c2w, fx, fy, cx, cy, eps=EPS, min_views=MIN_VIEWS, device="cuda"):
    """``Mesher.point_masks`` on given depth maps [n, H, W]: (valid bool [N], counts int32 [N]), counts the views that see
    each point and valid = counts >= min_views."""
    dev = _device(device)
    p, _ = _mesh(points, np.zeros((0, 3), np.int64), dev)
    p = p.float().contiguous()
    poses = _poses(c2w)
    d = depths.to(dev, torch.float32) if isinstance(depths, torch.Tensor) else torch.as_tensor(np.asarray(depths, np.float32), device=dev)
    if d.dim() != 3 or d.shape[0] != len(poses):
        raise ValueError(f"depths must be [n, H, W] with one map per pose, got {tuple(d.shape)}")
    _check_camera(d.shape[1], d.shape[2], ZNEAR, FAR)
    counts = torch.zeros(p.shape[0], dtype=torch.int32, device=dev)
    for k, m in enumerate(_w2c(poses)):
        _C._tnt_cull.visibility_count(p, d[k].contiguous(), m, fx, fy, cx, cy, eps, counts)
    return counts >= min_views, counts


def cull_mesh(vertices, faces, c2w, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY, far=FAR, znear=ZNEAR, eps=EPS, min_views=MIN_VIEWS, depth_c2w=None,
              device="cuda"):
    """``Mesher.cull_mesh``: (vertices [V'], faces int64 [F', 3], valid bool [V], counts int32 [V]).  The kept vertex rows
    are the input rows unchanged, in order; faces keep their order and are renumbered.  ``depth_c2w`` (default ``c2w``)
    sets the poses the depth is rendered from; ``c2w @ diag(1, -1, -1, 1)`` reproduces the shipped script."""
    dev = _device(device)
    _check_camera(H, W, znear, far)
    v, f = _mesh(vertices, faces, dev)
    poses = _poses(c2w)
    dposes = poses if depth_c2w is None else _poses(depth_c2w, "depth_c2w")
    if len(dposes) != len(poses):
        raise ValueError(f"depth_c2w has {len(dposes)} poses, c2w {len(poses)}")
    p, f32 = v.float().contiguous(), f.to(torch.int32).contiguous()
    counts = torch.zeros(v.shape[0], dtype=torch.int32, device=dev)
    for m, dm in zip(_w2c(poses), _w2c(dposes)):
        depth = _C._tnt_cull.mesh_depth(p, f32, dm, fx, fy, cx, cy, int(H), int(W), znear, far)
        _C._tnt_cull.visibility_count(p, depth, m, fx, fy, cx, cy, eps, counts)
    valid = counts >= min_views
    face_keep = valid[f].all(dim=1) if f.numel() else torch.zeros(0, dtype=torch.bool, device=dev)
    kept = f[face_keep]
    used = torch.zeros(v.shape[0], dtype=torch.bool, device=dev)
    used[kept.reshape(-1)] = True
    new_index = torch.cumsum(used.to(torch.int64), 0) - 1
    return v[used], new_index[kept], valid, counts


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Cull a Tanks and Temples mesh to the surface the trajectory's cameras see (eval_tnt/cull_mesh.py)")
    ap.add_argument("--traj-path", required=True, help="camera-to-world trajectory: .log or .npy ([n, 4, 4] or [n, 3, 4])")
    ap.add_argument("--ply-path", required=True, help="reconstruction PLY; the result goes to <ply without .ply>_cull.ply")
    ap.add_argument("--H", type=int, default=H)
    ap.add_argument("--W", type=int, default=W)
    ap.add_argument("--fx", type=float, default=FX)
    ap.add_argument("--fy", type=float, default=FY)
    ap.add_argument("--cx", type=float, default=CX)
    ap.add_argument("--cy", type=float, default=CY)
    ap.add_argument("--far", type=float, default=FAR)
    ap.add_argument("--eps", type=float, default=EPS)
    ap.add_argument("--min-views", type=int, default=MIN_VIEWS)
    ap.add_argument("--shipped-depth-pose", action="store_true",
                    help="render the depth from c2w @ diag(1, -1, -1, 1), the pose the shipped script's pyrender camera used")
    a = ap.parse_args(argv)
    c2w = load_poses(a.traj_path)
    vertices, faces = ply_io.load_triangle_mesh_ply(a.ply_path)
    v, f, valid, _ = cull_mesh(vertices, faces, c2w, a.H, a.W, a.fx, a.fy, a.cx, a.cy, a.far, eps=a.eps, min_views=a.min_views,
                               depth_c2w=c2w @ OPENGL_FLIP if a.shipped_depth_pose else None)
    out = a.ply_path.replace(".ply", "_cull.ply")
    ply_io.save_triangle_mesh_ply(out, v, f)
    print(f"kept {int(valid.sum())} of {len(valid)} vertices valid, {len(f)} of {len(faces)} faces; wrote {out}")
    return out


if __name__ == "__main__":
    main()
