"""Tetrahedra mesh extraction on the GPU: the unbounded-scene mesh path of RaDe-GS and Gaussian Opacity Fields
(mesh_extract_tetrahedra.py), without trimesh and without the reference's CPU detour for marching tetrahedra.

The pieces keep the reference's names and shapes::

    points, scales = tetra_points(gaussians.get_xyz, gaussians.get_scaling_with_3D_filter, gaussians._rotation)
    cells = delaunay(points)                                      # exact Delaunay on the GPU
    def evaluate_sdf(pts):                                        # evaluage_cull_alpha: the caller's loop over views
        cull = CullSDF(pts.shape[0], pts.device)
        for view in views:
            ret = integrate(pts, view, gaussians, pipeline, background, kernel_size)
            cull.add(ret["alpha_integrated"], ret["point_coordinate"], ret["render"][7], view.gt_mask)
        return cull.sdf()
    vertices, faces = extract_mesh(points, scales, cells, evaluate_sdf)

The arithmetic of the cull SDF, marching tetrahedra, the bisection and the filter is fixed bit for bit by the contract at
``rgs_tetra_*`` in include/rgs_b200.h; the kernels are in csrc/rgs_tetra.cu.  Every tensor argument must be on a CUDA device
(there is no CPU path), except the cells, which may come from the host.

Deliberate differences from the reference:

* ``delaunay`` replaces the reference's ``cpp.triangulate`` on the GPU: exact predicates with the symbolic perturbation
  CGAL uses, so the cells are unique and positively oriented (bit-equality with CGAL is not claimed).  It differs from
  Del(points) only by the rare near-flat hull cells whose circumsphere reaches its bounding ghost vertices, and it
  returns no cells for fewer than 4 distinct or coplanar points (scipy raises).
* ``triangulate`` (host points) falls back to ``scipy.spatial.Delaunay`` when the reference's CGAL binding (tetranerf) is
  not installed; where points are cospherical the two may return different cells, and scipy mixes orientations.
* ``marching_tetrahedra`` runs on the GPU in one pass at any size (the reference moves it to the CPU and, above 2^25 tets,
  loops over chunks); the vertices and the face order are the reference's, chunked order included.
* ``extract_mesh`` returns at once, without evaluating the SDF again, when the surface is empty.
"""
from __future__ import annotations

from typing import Callable

import numpy as np
import torch

from diff_gaussian_rasterization import _C


def _f32(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch tensor, got {type(t).__name__}")
    if t.device.type != "cuda":
        raise RuntimeError(f"{name} must be a CUDA tensor: there is no CPU path")
    return t.detach().float().contiguous()


def tetra_points(xyz: torch.Tensor, scaling_with_3D_filter: torch.Tensor, rotation: torch.Tensor):
    """``GaussianModel.get_tetra_points``: the 8 corners R(q/|q|) (+-3s) + xyz of every Gaussian (Gaussian-major, in
    ``trimesh.creation.box()`` order), then the P centres: ``points`` f32 [9P, 3]; ``scales`` f32 [9P, 1] = max(3s).
    ``rotation`` is the raw quaternion (``GaussianModel._rotation``); it is normalised here."""
    return _C.tetra_points(_f32(xyz, "xyz"), _f32(scaling_with_3D_filter, "scaling_with_3D_filter"), _f32(rotation, "rotation"))


def delaunay(points: torch.Tensor, return_stats: bool = False):
    """Exact Delaunay tetrahedralisation of ``points`` f32 [N, 3] on their CUDA device: int32 [T, 4] cells, every one
    positively oriented, rows canonical and sorted (contract at ``rgs_delaunay`` in include/rgs_b200.h).  Equal points
    count once (the smallest index represents them); fewer than 4 distinct or coplanar points give no cells.  With
    ``return_stats``, also a dict of the rounds, the largest cavity, the overflowed cavities and the mesh growths."""
    cells, stats = _C._delaunay.triangulate(_f32(points, "points"))
    return (cells, stats) if return_stats else cells


def triangulate(points) -> torch.Tensor:
    """Delaunay tetrahedralisation of ``points`` [N, 3] on the host: int32 [T, 4] cells (CPU).  Uses the reference's CGAL
    binding ``tetranerf.utils.extension.cpp.triangulate`` when it imports, ``scipy.spatial.Delaunay`` otherwise."""
    try:
        from tetranerf.utils.extension import cpp
    except ImportError:
        cpp = None
    if cpp is not None:
        return cpp.triangulate(points).cpu().int()
    from scipy.spatial import Delaunay

    pts = points.detach().cpu().double().numpy() if isinstance(points, torch.Tensor) else np.asarray(points, dtype=np.float64)
    if pts.shape[0] < 4:
        return torch.zeros((0, 4), dtype=torch.int32)
    return torch.from_numpy(np.ascontiguousarray(Delaunay(pts).simplices, dtype=np.int32))


class CullSDF:
    """``evaluage_cull_alpha`` of mesh_extract_tetrahedra.py: per point, the minimum ``alpha_integrated`` over the views whose
    (optionally ground-truth-masked) rendered alpha, sampled bilinearly at the point's pixel, exceeds 0.5; ``sdf()`` is
    0.5 minus that minimum, or -100 where no view saw the point.  One kernel per ``add``; the inputs are not modified."""

    def __init__(self, num_points: int, device="cuda"):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("CullSDF lives on a CUDA device: there is no CPU path")
        if int(num_points) < 0:
            raise ValueError(f"num_points must be non-negative, got {num_points}")
        self.final = torch.ones(int(num_points), dtype=torch.float32, device=device)
        self.weight = torch.zeros(int(num_points), dtype=torch.int32, device=device)

    def add(self, alpha_integrated: torch.Tensor, point_coordinate: torch.Tensor, render7: torch.Tensor, gt_mask: torch.Tensor | None = None):
        """One view: ``alpha_integrated`` [N], ``point_coordinate`` [N, 2] (pixels) and ``render7`` [H, W] as returned by
        ``integrate`` (``ret["render"][7]``); ``gt_mask`` [H, W] (or [1, H, W]) multiplies the rendered alpha."""
        empty = render7.new_empty((0,)) if isinstance(render7, torch.Tensor) else None
        gt = empty if gt_mask is None else _f32(gt_mask, "gt_mask")
        _C.tetra_cull_add(_f32(alpha_integrated, "alpha_integrated"), _f32(point_coordinate, "point_coordinate"), _f32(render7, "render7"), gt,
                          self.final, self.weight)
        return self

    def sdf(self) -> torch.Tensor:
        """f32 [N]: 0.5 - min alpha where at least one view passed the test, -100 elsewhere."""
        return _C.tetra_cull_finish(self.final, self.weight)


def _tets(tets, device) -> torch.Tensor:
    t = torch.as_tensor(tets)
    if t.dim() != 2 or t.shape[1] != 4:
        raise ValueError(f"tets must be [T, 4], got {tuple(t.shape)}")
    if t.dtype.is_floating_point or t.dtype == torch.bool:
        raise TypeError(f"tets must hold integers, got {t.dtype}")
    return t.to(device=device, dtype=torch.int64).contiguous()


def _unbatched_marching_tetrahedra(vertices, tets, sdf, scales):
    ends, end_sdf, end_scales, faces, interp_v = _C.tetra_marching(_f32(vertices, "vertices"), _f32(sdf, "sdf"), _f32(scales, "scales"),
                                                                   _tets(tets, vertices.device))
    return (ends, end_sdf), end_scales, faces, interp_v


def marching_tetrahedra(vertices: torch.Tensor, tets, sdf: torch.Tensor, scales: torch.Tensor):
    """utils/tetmesh.py's ``marching_tetrahedra``: ``vertices`` [B, N, 3], ``tets`` [T, 4] (shared), ``sdf`` [B, N],
    ``scales`` [B, N, 1].  Returns, as the reference, ``[verts_list, scale_list, faces_list, interp_list]`` where
    ``verts_list[b] = (endpoints [M, 2, 3], endpoint sdf [M, 2, 1])``, ``scale_list[b]`` [M, 2, 1], ``faces_list[b]`` int64
    [F, 3] and ``interp_list[b]`` int64 [M, 2] (the crossing edges, ascending)."""
    outs = [_unbatched_marching_tetrahedra(vertices[b], tets, sdf[b], scales[b]) for b in range(vertices.shape[0])]
    return list(zip(*outs))


def extract_mesh(points: torch.Tensor, scales: torch.Tensor, cells, evaluate_sdf: Callable[[torch.Tensor], torch.Tensor], n_binary_steps: int = 8):
    """``marching_tetrahedra_with_binary_search`` without the export: marching tetrahedra on ``evaluate_sdf(points)``,
    ``n_binary_steps`` bisection steps along every crossing edge (one ``evaluate_sdf`` call each), then the filter that keeps
    a vertex when its edge is no longer than the sum of its endpoints' scales and a face when its three vertices are kept.
    Returns ``(vertices f32 [V, 3], faces int64 [F, 3])`` on the points' device."""
    if int(n_binary_steps) < 0:
        raise ValueError(f"n_binary_steps must be non-negative, got {n_binary_steps}")
    pts = _f32(points, "points")
    sdf = evaluate_sdf(pts)
    (ends, end_sdf), end_scales, faces, _ = _unbatched_marching_tetrahedra(pts, cells, sdf, scales)
    M = ends.shape[0]
    if M == 0:
        return pts.new_zeros((0, 3)), torch.zeros((0, 3), dtype=torch.int64, device=pts.device)
    left, right = ends[:, 0].contiguous(), ends[:, 1].contiguous()
    left_sdf, right_sdf = end_sdf[:, 0, 0].contiguous(), end_sdf[:, 1, 0].contiguous()
    mid = torch.empty_like(left)
    none = left.new_empty((0,))
    _C.tetra_bisect(none, left, right, left_sdf, right_sdf, mid)
    for _ in range(int(n_binary_steps)):
        mid_sdf = evaluate_sdf(mid)
        _C.tetra_bisect(_f32(mid_sdf, "mid_sdf").reshape(-1), left, right, left_sdf, right_sdf, mid)
    return _C.tetra_filter(mid, ends, end_scales, faces)
