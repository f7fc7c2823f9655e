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


class VoxelBlockGrid:
    """Sparse grid of 16^3-voxel blocks with ``tsdf``, ``weight`` and ``color`` (3 channels) per voxel, on one CUDA device."""

    def __init__(self, voxel_size: float, block_resolution: int = BLOCK_RESOLUTION, block_count: int = 50000, device="cuda"):
        if block_resolution != BLOCK_RESOLUTION:
            raise ValueError(f"block_resolution must be {BLOCK_RESOLUTION} (the kernels are written for 16^3 blocks), got {block_resolution}")
        if not (math.isfinite(voxel_size) and voxel_size > 0 and np.float32(voxel_size) > 0):
            raise ValueError(f"voxel_size must be positive and finite, got {voxel_size}")
        if int(block_count) < 1:
            raise ValueError(f"block_count must be at least 1, got {block_count}")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("VoxelBlockGrid lives on a CUDA device: there is no CPU path")
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

    # ---- Open3D's calls ---------------------------------------------------------------------------------------------------
    def compute_unique_block_coordinates(self, depth: torch.Tensor, intrinsic, extrinsic, depth_scale: float = 1.0, depth_max: float = 3.0,
                                         trunc_voxel_multiplier: float = 8.0) -> torch.Tensor:
        """int32 [N, 3] coordinates of the blocks within the truncation band of the depth map, ascending (x, y, z)."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        while True:
            n, coords, allocated = _C.tsdf_touch(self, depth, K, E, depth_scale, depth_max, trunc_voxel_multiplier)
            self._allocated_bound = allocated
            if n >= 0:
                return coords
            self._set_frame(2 * self.frame_keys.numel())

    def integrate(self, block_coords: torch.Tensor, depth: torch.Tensor, color: torch.Tensor, intrinsic, extrinsic, depth_scale: float = 1.0,
                  depth_max: float = 3.0, trunc_voxel_multiplier: float = 8.0) -> None:
        """Fuse one view into the given blocks (allocated when new).  color: float32 [H, W, 3], stored as given."""
        K, E = _matrix(intrinsic, (3, 3), "intrinsic"), _matrix(extrinsic, (4, 4), "extrinsic")
        n = int(block_coords.shape[0]) if block_coords.dim() == 2 else 0
        if self._allocated_bound + n > self.capacity:
            self._allocated_bound = self._allocated()
            if self._allocated_bound + n > self.capacity:
                self._grow(self._allocated_bound + n)
        self._calls += 1
        _C.tsdf_integrate(self, block_coords, depth, color, K, E, depth_scale, depth_max, trunc_voxel_multiplier, self._calls)
        self._allocated_bound += n

    def extract_triangle_mesh(self, weight_threshold: float = 3.0) -> TriangleMesh:
        v, c, t = _C.tsdf_extract(self, weight_threshold)
        return TriangleMesh(v, t, c)

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
