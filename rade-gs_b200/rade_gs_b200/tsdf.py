"""TSDF fusion and marching-cubes mesh extraction on the GPU: the mesh step of the reference's DTU path
(mesh_extract.py:66-105), which runs Open3D's ``o3d.t.geometry.VoxelBlockGrid`` on the CPU.

The calls mirror the Open3D ones that script makes, with Open3D's argument order and defaults::

    vbg = VoxelBlockGrid(voxel_size=0.002, block_resolution=16, block_count=50000)
    for depth, color, cam in views:                       # CUDA float32 [H, W] and [H, W, 3], straight from render()
        coords = vbg.compute_unique_block_coordinates(depth, intrinsic, extrinsic, 1.0, 8.0)
        vbg.integrate(coords, depth, color, intrinsic, extrinsic, 1.0, 8.0)
    mesh = vbg.extract_triangle_mesh()
    mesh.compute_vertex_normals()

The arithmetic is fixed bit for bit by the contract at ``rgs_tsdf_*`` in include/rgs_b200.h; the kernels are in
csrc/rgs_tsdf.cu.  The grid's arrays live here, on the GPU, and grow by doubling when a view needs more blocks than the
grid holds (Open3D's ``block_count`` is therefore an initial size, not a limit).  Depth and colour must be CUDA tensors:
there is no CPU path.  The camera (``intrinsic`` 3x3, world->camera ``extrinsic`` 4x4) may be a torch tensor on any
device, a numpy array or nested lists; it is converted to fp32 once.

``ScalableTSDFVolume`` is the bounded TSDF of the reference's ``GaussianExtractor.extract_mesh_bounded`` (Open3D's legacy
volume) on the same block storage; see its docstring and the contract at ``rgs_scalable_*``.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from diff_gaussian_rasterization import _C

BLOCK_RESOLUTION = 16
_BV = BLOCK_RESOLUTION ** 3


def _next_pow2(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


def _matrix(m, shape, name) -> torch.Tensor:
    if isinstance(m, torch.Tensor):
        t = m.detach().to("cpu", torch.float64)
    else:
        t = torch.as_tensor(np.asarray(m, dtype=np.float64))
    if tuple(t.shape) != shape:
        raise ValueError(f"{name} must be {shape[0]}x{shape[1]}, got {tuple(t.shape)}")
    return t.contiguous()


class TriangleMesh:
    """Vertices f32 [V, 3], triangles int32 [F, 3], vertex colours f32 [V, 3] and, after ``compute_vertex_normals()``,
    vertex normals f32 [V, 3] (an empty [0, 3] tensor before), all on the GPU."""

    def __init__(self, vertices: torch.Tensor, triangles: torch.Tensor, vertex_colors: torch.Tensor):
        self.vertices = vertices
        self.triangles = triangles
        self.vertex_colors = vertex_colors
        self.vertex_normals = vertices.new_zeros((0, 3))

    def compute_vertex_normals(self) -> "TriangleMesh":
        """Area-weighted vertex normals (rgs_tsdf_vertex_normals): the sum of the incident face normals, normalised;
        (0, 0, 0) for a vertex whose sum is zero."""
        self.vertex_normals = _C.tsdf_vertex_normals(self.vertices, self.triangles)
        return self

    def has_vertex_normals(self) -> bool:
        return self.vertex_normals.shape[0] == self.vertices.shape[0] and self.vertices.shape[0] > 0


class _BlockStore:
    """The arrays of an rgs_tsdf_grid on one CUDA device (16^3-voxel blocks with ``tsdf``, ``weight`` and ``color`` per
    voxel, their hash and the frame-local touch buffers), with growth by doubling and the accessors both volumes share."""

    def __init__(self, voxel_size: float, block_count: int, device, name: str, size_name: str = "voxel_size"):
        if not (math.isfinite(voxel_size) and voxel_size > 0 and np.float32(voxel_size) > 0):
            raise ValueError(f"{size_name} must be positive and finite, got {voxel_size}")
        if int(block_count) < 1:
            raise ValueError(f"block_count must be at least 1, got {block_count}")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError(f"{name} lives on a CUDA device: there is no CPU path")
        self.voxel_size = float(np.float32(voxel_size))
        self.counters = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._allocate(int(block_count))
        self._set_frame(self.hash_keys.numel())
        self._calls = 0
        self._allocated_bound = 0        # >= the allocated block count (exact after every touch)

    # ---- storage ----------------------------------------------------------------------------------------------------------
    def _allocate(self, capacity: int):
        dev = self.device
        self.hash_keys = torch.full((_next_pow2(2 * capacity),), -1, dtype=torch.int64, device=dev)   # -1 = free (RGS_TSDF_EMPTY_KEY)
        self.hash_values = torch.full((self.hash_keys.numel(),), -1, dtype=torch.int32, device=dev)
        self.tsdf = torch.zeros(capacity * _BV, dtype=torch.float32, device=dev)
        self.weight = torch.zeros(capacity * _BV, dtype=torch.float32, device=dev)
        self.color = torch.zeros(capacity * _BV * 3, dtype=torch.float32, device=dev)
        self.stamps = torch.zeros(capacity, dtype=torch.int32, device=dev)

    def _set_frame(self, slots: int):
        self.frame_keys = torch.empty(slots, dtype=torch.int64, device=self.device)
        self.frame_list = torch.empty(slots // 2, dtype=torch.int64, device=self.device)

    @property
    def capacity(self) -> int:
        return self.stamps.numel()

    def _grow(self, need: int):
        """Double the capacity until `need` blocks fit: pools copied to the front of larger zeroed pools, keys rehashed."""
        cap = self.capacity
        while cap < need:
            cap *= 2
        old = (self.hash_keys, self.hash_values, self.tsdf, self.weight, self.color, self.stamps)
        self._allocate(cap)
        for new, o in zip((self.tsdf, self.weight, self.color, self.stamps), old[2:]):
            new[:o.numel()] = o
        _C.tsdf_rehash(self, old[0], old[1])

    def _allocated(self) -> int:
        return int(self.counters[0].item())

    def _touch(self, touch, *args) -> torch.Tensor:
        """Run a touch entry of _C, doubling the frame-local hash until the view's blocks fit."""
        while True:
            n, coords, allocated = touch(self, *args)
            self._allocated_bound = allocated
            if n >= 0:
                return coords
            self._set_frame(2 * self.frame_keys.numel())

    def _reserve(self, n: int):
        """Grow so that n more blocks fit whatever the next integrate call inserts."""
        if self._allocated_bound + n > self.capacity:
            self._allocated_bound = self._allocated()
            if self._allocated_bound + n > self.capacity:
                self._grow(self._allocated_bound + n)

    # ---- accessors --------------------------------------------------------------------------------------------------------
    def attribute(self, name: str) -> torch.Tensor:
        """View [capacity, 16, 16, 16, C] of a voxel attribute, indexed [pool index, z, y, x, channel]."""
        R = BLOCK_RESOLUTION
        if name in ("tsdf", "weight"):
            return getattr(self, name).view(self.capacity, R, R, R, 1)
        if name == "color":
            return self.color.view(self.capacity, R, R, R, 3)
        raise KeyError(f"no attribute {name!r}: the grid holds tsdf, weight and color")

    def active_blocks(self):
        """(keys int64 [N] ascending, pool indices int32 [N]) of the allocated blocks.  key = (bx + 2^20) << 42 |
        (by + 2^20) << 21 | (bz + 2^20); ``block_coordinates(keys)`` decodes it."""
        return _C.tsdf_active_blocks(self)

    def block_coordinates(self, keys: torch.Tensor) -> torch.Tensor:
        m = (1 << 21) - 1
        return (torch.stack([keys >> 42 & m, keys >> 21 & m, keys & m], 1) - (1 << 20)).to(torch.int32)


class VoxelBlockGrid(_BlockStore):
    """Sparse grid of 16^3-voxel blocks with ``tsdf``, ``weight`` and ``color`` (3 channels) per voxel, on one CUDA device."""

    def __init__(self, voxel_size: float, block_resolution: int = BLOCK_RESOLUTION, block_count: int = 50000, device="cuda"):
        if block_resolution != BLOCK_RESOLUTION:
            raise ValueError(f"block_resolution must be {BLOCK_RESOLUTION} (the kernels are written for 16^3 blocks), got {block_resolution}")
        super().__init__(voxel_size, block_count, device, "VoxelBlockGrid")

    # ---- Open3D's calls ---------------------------------------------------------------------------------------------------
    def compute_unique_block_coordinates(self, depth: torch.Tensor, intrinsic, extrinsic, depth_scale: float = 1.0, depth_max: float = 3.0,
                                         trunc_voxel_multiplier: float = 8.0) -> torch.Tensor:
        """int32 [N, 3] coordinates of the blocks within the truncation band of the depth map, ascending (x, y, z)."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        return self._touch(_C.tsdf_touch, depth, K, E, depth_scale, depth_max, trunc_voxel_multiplier)

    def integrate(self, block_coords: torch.Tensor, depth: torch.Tensor, color: torch.Tensor, intrinsic, extrinsic, depth_scale: float = 1.0,
                  depth_max: float = 3.0, trunc_voxel_multiplier: float = 8.0) -> None:
        """Fuse one view into the given blocks (allocated when new).  color: float32 [H, W, 3], stored as given."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        n = int(block_coords.shape[0]) if block_coords.dim() == 2 else 0
        self._reserve(n)
        self._calls += 1
        _C.tsdf_integrate(self, block_coords, depth, color, K, E, depth_scale, depth_max, trunc_voxel_multiplier, self._calls)
        self._allocated_bound += n

    def extract_triangle_mesh(self, weight_threshold: float = 3.0) -> TriangleMesh:
        v, c, t = _C.tsdf_extract(self, weight_threshold)
        return TriangleMesh(v, t, c)


def rgbd_from_color_and_depth(rgb: torch.Tensor, depth: torch.Tensor, depth_trunc: float, mask: torch.Tensor | None = None):
    """Open3D's ``RGBDImage.create_from_color_and_depth(depth_scale=1, depth_trunc, convert_rgb_to_intensity=False)`` of what
    the reference's extract_mesh_bounded hands it: (color uint8 [H, W, 3], depth float32 [H, W]) on the GPU.

    rgb float32 [3, H, W] becomes ``np.asarray(rgb * 255, dtype=np.uint8)`` bit for bit: not clamped, numpy's x86-64 cast
    truncates and wraps (1.01 -> 1, -0.01 -> 254; NaN and |x| >= 2^31 -> 0).  depth float32 [1, H, W] or [H, W]: 0 where
    ``mask < 0.5`` (mask: H * W floats, e.g. the camera's gt_mask [1, H, W]), then 0 where depth >= depth_trunc."""
    for t, name in ((rgb, "rgb"), (depth, "depth"), (mask, "mask")):
        if t is not None and (not isinstance(t, torch.Tensor) or not t.is_cuda):
            raise ValueError(f"{name} must be a CUDA tensor: there is no CPU path")
    if not isinstance(depth_trunc, (int, float)) or math.isnan(depth_trunc):
        raise ValueError(f"depth_trunc must be a number, got {depth_trunc!r}")
    m = None if mask is None else mask.detach().to(torch.float32)
    return _C._scalable_tsdf.rgbd(rgb.detach().to(torch.float32), depth.detach().to(torch.float32), float(depth_trunc), m)


class ScalableTSDFVolume(_BlockStore):
    """Open3D's legacy ``ScalableTSDFVolume(voxel_length, sdf_trunc, color_type=RGB8)`` on the GPU, the volume of the
    reference's ``GaussianExtractor.extract_mesh_bounded``::

        vol = ScalableTSDFVolume(voxel_length=0.004, sdf_trunc=0.02)
        for rgb, depth, K, E in views:          # render()'s [3, H, W] colour and [1, H, W] depth, CUDA float32
            color, d = rgbd_from_color_and_depth(rgb, depth, depth_trunc=3.0)
            vol.integrate(color, d, K, E)
        mesh = vol.extract_triangle_mesh()     # TriangleMesh, colours in [0, 1]

    Volume units are 16^3 voxels and stored as the blocks of ``VoxelBlockGrid`` (same arrays, growth and accessors).  The
    rules (every 4th pixel allocates the units within sdf_trunc of its point; voxel centres at (g + 0.5) voxel_length; the
    SDF is the distance along the ray; colour averaged over 8-bit values) are fixed bit for bit by the contract at
    ``rgs_scalable_*`` in include/rgs_b200.h.  ``block_count`` is an initial size: the volume grows by doubling."""

    def __init__(self, voxel_length: float, sdf_trunc: float, block_count: int = 1024, device="cuda"):
        if not (isinstance(sdf_trunc, (int, float)) and math.isfinite(sdf_trunc) and sdf_trunc > 0 and np.float32(sdf_trunc) > 0):
            raise ValueError(f"sdf_trunc must be positive and finite, got {sdf_trunc}")
        super().__init__(voxel_length, block_count, device, "ScalableTSDFVolume", "voxel_length")
        self.sdf_trunc = float(np.float32(sdf_trunc))

    @property
    def voxel_length(self) -> float:
        return self.voxel_size

    def touch(self, depth: torch.Tensor, intrinsic, extrinsic) -> torch.Tensor:
        """int32 [N, 3] coordinates, ascending, of the units one view allocates (the first half of ``integrate``)."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        return self._touch(_C._scalable_tsdf.touch, depth, K, E, self.sdf_trunc)

    def integrate(self, color: torch.Tensor, depth: torch.Tensor, intrinsic, extrinsic) -> None:
        """Fuse one view: color uint8 [H, W, 3] and depth float32 [H, W] as ``rgbd_from_color_and_depth`` returns them,
        intrinsic 3x3, world->camera extrinsic 4x4."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        units = self._touch(_C._scalable_tsdf.touch, depth, K, E, self.sdf_trunc)
        n = int(units.shape[0])
        self._reserve(n)
        self._calls += 1
        _C._scalable_tsdf.integrate(self, units, depth, color, K, E, self.sdf_trunc, self._calls)
        self._allocated_bound += n

    def extract_triangle_mesh(self) -> TriangleMesh:
        """Marching cubes over voxels of weight >= 1; vertices moved onto the voxel centres (+ voxel_length / 2) and colours
        scaled to [0, 1]."""
        v, c, t = _C.tsdf_extract(self, 1.0)
        half = np.float32(0.5) * np.float32(self.voxel_size)
        return TriangleMesh(v + float(half), t, c / c.new_full((1,), 255.0))
