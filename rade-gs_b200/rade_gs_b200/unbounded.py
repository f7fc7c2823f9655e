"""Contracted-space TSDF meshing of unbounded scenes on the GPU: the reference's ``GaussianExtractor`` path
(utils/mesh_utils.py:163-271 and :23-44, utils/mcube_utils.py:17-95), which runs eager torch, scikit-image marching cubes
and trimesh / Open3D on the host.  It is the TSDF path for unbounded captures (Mip-NeRF 360, Tanks and Temples)::

    ex = GaussianExtractor(gaussians, render, pipe, kernel_size=0.0)
    ex.reconstruction(viewpoint_stack)                      # render() per view, the maps stay on the GPU
    mesh = ex.extract_mesh_unbounded(resolution=1024)       # tsdf.TriangleMesh on the GPU
    mesh = post_process_mesh(mesh, cluster_to_keep=1000)

``extract_mesh_unbounded_maps`` takes the maps and cameras directly, for callers without a ``GaussianModel``.

The same extractor has the reference's bounded half (utils/mesh_utils.py:118-160, :272-285)::

    ex.export_image(out_dir)                                # renders/, gt/, vis/depth_*.tiff, vis/normal_*.png
    mesh = ex.extract_mesh_bounded(voxel_size=0.004, sdf_trunc=0.02, depth_trunc=3)   # tsdf.ScalableTSDFVolume

where the reference's own class fails: it reads ``gt_alpha_mask`` (RaDe-GS's Camera holds ``gt_mask``; that is read
here) and calls ``save_img_u8`` / ``save_img_f32`` without importing them.

Stages (the arithmetic of each is fixed bit for bit by the contract at ``rgs_unbounded_*`` in include/rgs_b200.h; the
kernels are in csrc/rgs_unbounded.cu):

1. normalisation on the host in float64 (``normalization``): scene centre = the point nearest to all focal axes, radius =
   the nearest camera's distance to it; the bound R = min(quantile_0.95(|contract((xyz - c) / r)|) + 0.01, 1.9), the norms
   computed on the GPU and the quantile by numpy (no 2^24 limit);
2. the SDF of each ``crop``^3 block of the ``resolution``^3 grid over [-R, R]^3, in the reference's (i, j, k) order: every
   sample uncontracted to world space and fused over all views;
3. marching cubes per crop, vertices on their lattice edges in fp64 from the crop origin and spacing;
4. vertex merge at 10^-6 in contracted space (which also joins the crop seams);
5. back to world space, clipped to +-32;
6. vertex colours from the RGB maps.

R, the crop bounds and the samples follow the reference's numpy expressions, so they are float32 under numpy >= 2 and
float64 under numpy 1, as the reference's are; the marching-cubes vertex positions are then computed in fp64 from those
origin and spacing (which numpy computes as the reference does).

Deliberate differences from the reference:
  * marching cubes uses the repository's watertight triangle table (rgs_tsdf_extract's), not scikit-image's Lewiner
    table: the vertices on sign-change edges are the same, the triangles of ambiguous cells may differ; normals point to
    free space (positive SDF);
  * ``post_process_mesh`` with fewer than ``cluster_to_keep`` clusters keeps every cluster of at least 50 triangles (the
    reference raises IndexError);
  * ``reconstruction()`` keeps only the maps the meshes and the export read (RGB, median depth and normals) and keeps
    them on the GPU; the alpha and depth-normal maps are not kept, so ``export_image`` writes no depth-normal PNGs;
  * the bounded mesh (see ``tsdf.ScalableTSDFVolume``) uses the repository's watertight triangle table, its own
    deterministic vertex and triangle order and fp32 colour averages, and leaves the stored depth maps unmasked.
"""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from diff_gaussian_rasterization import _C

from .tsdf import ScalableTSDFVolume, TriangleMesh, rgbd_from_color_and_depth

CROP = 512                # the reference's crop edge (marching_cubes_with_contraction's cropN)
MAX_RANGE = 32.0          # world-space clip of the vertices (its max_range)


def _cuda_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor: there is no CPU path")
    return t.detach().to(torch.float32).contiguous()


def contract(x: torch.Tensor) -> torch.Tensor:
    """x if |x| < 1 else (2 - 1/|x|) x/|x|, per row of a CUDA float32 [N, 3] tensor."""
    return _C._unbounded.contract(_cuda_f32(x, "x").reshape(-1, 3), [0.0, 0.0, 0.0], 1.0, False, math.inf)[0].view(x.shape)


def uncontract(y: torch.Tensor) -> torch.Tensor:
    """y if |y| < 1 else y / (|y| (2 - |y|)), per row of a CUDA float32 [N, 3] tensor."""
    return _C._unbounded.contract(_cuda_f32(y, "y").reshape(-1, 3), [0.0, 0.0, 0.0], 1.0, True, math.inf)[0].view(y.shape)


def focus_point(poses: np.ndarray) -> np.ndarray:
    """The point nearest (least squares) to the optical axes of camera-to-world poses [V, 3, 4] (axis = column 2, origin =
    column 3): the solution of mean_v(A_v) x = mean_v(A_v o_v) with A_v = (I - d d^T)^T (I - d d^T)."""
    d, o = poses[:, :3, 2:3], poses[:, :3, 3:4]
    m = np.eye(3) - d * np.transpose(d, [0, 2, 1])
    a = np.transpose(m, [0, 2, 1]) @ m
    return np.linalg.inv(a.mean(0)) @ (a @ o).mean(0)[:, 0]


def normalization(world_view_transforms) -> tuple[np.ndarray, float]:
    """(center float64 [3], radius) of the views: camera-to-world = inv(world_view_transform^T) in fp32 as numpy gives it,
    OpenGL axes flipped to OpenCV's, centre = ``focus_point``, radius = the smallest camera distance to it."""
    w = [np.asarray(t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t, dtype=np.float32) for t in world_view_transforms]
    w = np.stack(w) if w else np.zeros((0, 4, 4), np.float32)
    if w.ndim != 3 or w.shape[1:] != (4, 4) or len(w) == 0:
        raise ValueError(f"world_view_transforms must be V >= 1 matrices 4x4, got shape {w.shape}")
    c2ws = np.array([np.linalg.inv(np.asarray(m.T)) for m in w])
    poses = c2ws[:, :3, :] @ np.diag([1, -1, -1, 1])
    center = focus_point(poses)
    radius = np.linalg.norm(c2ws[:, :3, 3] - center, axis=-1).min()
    return center, float(radius)


def scene_bound(xyz: torch.Tensor, center, radius: float):
    """R = min(quantile_0.95(|contract((xyz - center) / radius)|) + 0.01, 1.9) with the reference's numpy expressions over
    the fp32 norms: a numpy float32 under numpy >= 2 (NEP 50 keeps the quantile and the + 0.01 in float32), float64 under
    numpy 1.  The crop bounds and samples then come from numpy's linspace of that R, as in the reference."""
    _, norms = _C._unbounded.contract(_cuda_f32(xyz, "xyz").reshape(-1, 3), [float(c) for c in center], float(radius), False, math.inf)
    if norms.numel() == 0:
        raise ValueError("xyz must hold at least one point")
    R = np.quantile(norms.cpu().numpy(), q=0.95)
    return min(R + 0.01, 1.9)


def _views(depths: torch.Tensor, rgbs: torch.Tensor | None, full_proj_transforms) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor | None]:
    depths = _cuda_f32(depths, "depths")
    if depths.dim() == 4 and depths.shape[1] == 1:
        depths = depths[:, 0]
    if depths.dim() != 3 or depths.shape[0] == 0:
        raise ValueError(f"depths must be [V, H, W] (or [V, 1, H, W]) with V >= 1, got {tuple(depths.shape)}")
    if isinstance(full_proj_transforms, torch.Tensor):
        proj = full_proj_transforms
    else:
        proj = torch.stack([torch.as_tensor(t) for t in full_proj_transforms])
    proj = proj.detach().to(depths.device, torch.float32).contiguous()
    if tuple(proj.shape) != (depths.shape[0], 4, 4):
        raise ValueError(f"full_proj_transforms must be [V, 4, 4] with V = {depths.shape[0]}, got {tuple(proj.shape)}")
    if rgbs is not None:
        rgbs = _cuda_f32(rgbs, "rgbs")
        if tuple(rgbs.shape) != (depths.shape[0], 3, depths.shape[1], depths.shape[2]):
            raise ValueError(f"rgbs must be [V, 3, H, W] like depths {tuple(depths.shape)}, got {tuple(rgbs.shape)}")
    return depths, proj, rgbs


def crop_axes(R: float, resolution: int, crop: int):
    """[(lo, spacing, (xs, ys, zs) float32 numpy)] of every crop in the reference's (i, j, k) order, each value from the
    reference's numpy expressions (marching_cubes_with_contraction), in numpy's dtype."""
    N = resolution // crop
    edges = np.linspace(-R, R, N + 1)
    out = []
    for i in range(N):
        for j in range(N):
            for k in range(N):
                lo = (edges[i], edges[j], edges[k])
                hi = (edges[i + 1], edges[j + 1], edges[k + 1])
                sp = tuple((hi[a] - lo[a]) / (crop - 1) for a in range(3))
                out.append((lo, sp, tuple(np.linspace(lo[a], hi[a], crop).astype(np.float32) for a in range(3))))
    return out


def extract_mesh_unbounded_maps(depths: torch.Tensor, rgbs: torch.Tensor, world_view_transforms, full_proj_transforms, xyz: torch.Tensor,
                                resolution: int = 1024, crop: int = CROP) -> TriangleMesh:
    """The unbounded TSDF mesh from maps already rendered: depths [V, H, W] (median depth), rgbs [V, 3, H, W], the views'
    ``world_view_transform`` and ``full_proj_transform`` (4x4 each, as the reference's Camera holds them) and the Gaussian
    centres xyz [P, 3].  resolution must be a multiple of crop (512 in the reference; smaller crops serve tests)."""
    if crop < 2 or crop > 640:
        raise ValueError(f"crop must be in [2, 640], got {crop}")
    if resolution < crop or resolution % crop:
        raise ValueError(f"resolution must be a positive multiple of {crop}, got {resolution}")
    depths, proj, rgbs = _views(depths, rgbs, full_proj_transforms)
    if len(world_view_transforms) != depths.shape[0]:
        raise ValueError(f"{len(world_view_transforms)} world_view_transforms for {depths.shape[0]} views")
    U = _C._unbounded
    center, radius = normalization(world_view_transforms)
    c = [float(x) for x in center]
    voxel_size = radius * 2 / resolution
    trunc = float(np.float32(5 * voxel_size))
    R = scene_bound(xyz, center, radius)
    verts, tris, base = [], [], 0
    for lo, sp, axes in crop_axes(R, resolution, crop):
        xs, ys, zs = (torch.from_numpy(a).to(depths.device) for a in axes)
        sdf = U.sdf(xs, ys, zs, proj, depths, c, radius, trunc)
        v, t = U.mcubes(sdf, [float(x) for x in lo], [float(x) for x in sp])
        del sdf
        if t.shape[0]:
            verts.append(v)
            tris.append(t + base)
            base += v.shape[0]
    if not verts:
        z = depths.new_zeros((0, 3))
        return TriangleMesh(z, torch.zeros((0, 3), dtype=torch.int32, device=depths.device), z.clone())
    merged, triangles = U.merge(torch.cat(verts), torch.cat(tris))
    world, _ = U.contract(merged, c, radius, True, MAX_RANGE)
    colors = U.colors(world, proj, depths, rgbs, trunc)
    return TriangleMesh(world, triangles, colors)


def open3d_camera(cam):
    """(intrinsic 3x3 float64, world->camera extrinsic 4x4 float64) of a view as the reference's ``to_cam_open3d`` builds
    them: cx = W / 2, cy = H / 2, fx = W / (2 tan(FoVx / 2)), fy = H / (2 tan(FoVy / 2)), extrinsic =
    world_view_transform^T."""
    W, H = cam.image_width, cam.image_height
    K = np.array([[W / (2 * math.tan(cam.FoVx / 2.)), 0, W / 2], [0, H / (2 * math.tan(cam.FoVy / 2.)), H / 2], [0, 0, 1]], np.float64)
    return K, np.asarray(cam.world_view_transform.T.detach().cpu().numpy(), np.float64)


def post_process_mesh(mesh: TriangleMesh, cluster_to_keep: int = 1000) -> TriangleMesh:
    """Drop small connected clusters (triangles joined by shared edges): keep clusters of at least
    max(k-th largest size, 50) triangles, then drop unreferenced vertices and degenerate triangles.  With fewer than
    ``cluster_to_keep`` clusters every cluster of at least 50 triangles stays (the reference raises IndexError)."""
    if int(cluster_to_keep) < 0:
        raise ValueError(f"cluster_to_keep must be >= 0, got {cluster_to_keep}")
    if not mesh.triangles.is_cuda:
        raise ValueError("the mesh must be on a CUDA device: there is no CPU path")
    vidx, tris, _ = _C._unbounded.clusters(int(mesh.vertices.shape[0]), mesh.triangles.to(torch.int32), int(cluster_to_keep))
    keep = vidx.long()
    out = TriangleMesh(mesh.vertices[keep], tris, mesh.vertex_colors[keep] if mesh.vertex_colors.shape[0] else mesh.vertex_colors)
    if mesh.has_vertex_normals():
        out.vertex_normals = mesh.vertex_normals[keep]
    return out


class GaussianExtractor:
    """The reference's extractor (utils/mesh_utils.py:65) for the unbounded mesh.  ``render`` is the repository's or the
    reference's ``render(viewpoint_camera, pc, pipe, bg_color, kernel_size, ...)``; ``kernel_size`` is the 3D-filter size
    that render needs and the reference's extractor does not pass."""

    def __init__(self, gaussians, render, pipe, bg_color=None, kernel_size: float = 0.0):
        if bg_color is None:
            bg_color = [0, 0, 0]
        self.gaussians = gaussians
        self._render = render
        self._pipe = pipe
        self._background = torch.tensor(bg_color, dtype=torch.float32, device="cuda")
        self.kernel_size = kernel_size
        self.clean()

    @torch.no_grad()
    def clean(self):
        self.depthmaps = []
        self.rgbmaps = []
        self.normals = []
        self.viewpoint_stack = []

    @torch.no_grad()
    def reconstruction(self, viewpoint_stack):
        """Render every view; keep render()'s "render" [3, H, W], "median_depth" [1, H, W] and the normalised "normal"
        [3, H, W] on the GPU: 7 floats per pixel per view (the normals, which only ``export_image`` reads, are 3 of them; they
        are kept when render() returns "normal" for every view)."""
        self.clean()
        self.viewpoint_stack = list(viewpoint_stack)
        if not self.viewpoint_stack:
            raise ValueError("reconstruction needs at least one view")
        rgbs, depths, normals = [], [], []
        for cam in self.viewpoint_stack:
            pkg = self._render(cam, self.gaussians, self._pipe, self._background, self.kernel_size)
            rgbs.append(pkg["render"].detach().float())
            depths.append(pkg["median_depth"].detach().float())
            if "normal" in pkg:
                normals.append(torch.nn.functional.normalize(pkg["normal"].detach().float(), dim=0))
        shapes = {tuple(d.shape[-2:]) for d in depths}
        if len(shapes) != 1:
            raise ValueError(f"all views must have one size, got {sorted(shapes)}")
        self.rgbmaps = torch.stack(rgbs)
        self.depthmaps = torch.stack(depths)
        self.normals = torch.stack(normals) if len(normals) == len(depths) else []

    @torch.no_grad()
    def extract_mesh_bounded(self, voxel_size=0.004, sdf_trunc=0.02, depth_trunc=3, mask_backgrond=True) -> TriangleMesh:
        """The bounded TSDF mesh "used in the paper": every view fused into a ``tsdf.ScalableTSDFVolume`` with the
        reference's camera (cx = W / 2, cy = H / 2, fx = W / (2 tan(FoVx / 2)), extrinsic = world_view_transform^T).
        With ``mask_backgrond`` (the reference's spelling), depth is dropped where the camera's ``gt_mask`` < 0.5.  The
        stored depth maps are not changed (the reference zeroes them in place, so its later ``export_image`` writes the
        masked depth)."""
        if not len(self.viewpoint_stack):
            raise ValueError("call reconstruction() first")
        volume = ScalableTSDFVolume(voxel_length=voxel_size, sdf_trunc=sdf_trunc)
        for i, cam in enumerate(self.viewpoint_stack):
            mask = getattr(cam, "gt_mask", None) if mask_backgrond else None
            color, depth = rgbd_from_color_and_depth(self.rgbmaps[i], self.depthmaps[i], depth_trunc, mask)
            volume.integrate(color, depth, *open3d_camera(cam))
        return volume.extract_triangle_mesh()

    @torch.no_grad()
    def export_image(self, path):
        """Write ``renders/`` and ``gt/`` (8-bit PNGs of the render and of ``original_image[:3]``), ``vis/depth_*.tiff``
        (float32 median depth) and ``vis/normal_*.png`` (normal * 0.5 + 0.5) as the reference's save_img_u8 /
        save_img_f32 write them: (clip(nan_to_num(x), 0, 1) * 255).astype(uint8) on the GPU, then PIL encodes.  The
        reference's ``vis/depth_normal_*.png`` is not written: its depth normals are not kept."""
        from PIL import Image

        if not len(self.viewpoint_stack):
            raise ValueError("call reconstruction() first")
        if len(self.normals) != len(self.viewpoint_stack):
            raise ValueError("export_image needs the normal maps: render() must return \"normal\" for every view")
        S = _C._scalable_tsdf
        dirs = {k: os.path.join(path, k) for k in ("renders", "gt", "vis")}
        for d in dirs.values():
            os.makedirs(d, exist_ok=True)

        def png(img, name):
            with open(name, "wb") as f:
                Image.fromarray(img.cpu().numpy()).save(f, "PNG")

        for idx, cam in enumerate(self.viewpoint_stack):
            gt = cam.original_image[0:3].detach().to(self.rgbmaps.device, torch.float32).contiguous()
            png(S.image_u8(gt), os.path.join(dirs["gt"], f"{idx:05d}.png"))
            png(S.image_u8(self.rgbmaps[idx]), os.path.join(dirs["renders"], f"{idx:05d}.png"))
            with open(os.path.join(dirs["vis"], f"depth_{idx:05d}.tiff"), "wb") as f:
                Image.fromarray(torch.nan_to_num(self.depthmaps[idx][0]).cpu().numpy()).save(f, "TIFF")
            png(S.image_u8(self.normals[idx], 0.5, 0.5), os.path.join(dirs["vis"], f"normal_{idx:05d}.png"))

    @torch.no_grad()
    def extract_mesh_unbounded(self, resolution: int = 1024) -> TriangleMesh:
        if resolution % CROP:
            raise ValueError(f"resolution must be a multiple of {CROP}, got {resolution}")
        if not len(self.viewpoint_stack):
            raise ValueError("call reconstruction() first")
        return extract_mesh_unbounded_maps(self.depthmaps, self.rgbmaps, [c.world_view_transform for c in self.viewpoint_stack],
                                           [c.full_proj_transform for c in self.viewpoint_stack], self.gaussians.get_xyz, resolution, CROP)
