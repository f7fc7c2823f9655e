"""Scenes for the tetrahedra mesh tests: seeded Gaussians and an analytic stand-in for ``integrate``.

The stand-in returns what mesh_extract_tetrahedra.py reads from ``integrate`` (``alpha_integrated``, ``point_coordinate`` and
``render[7]``) from elementwise +, -, x, /, comparisons and ``where`` only, one torch operation per call and no division by
a Python scalar (CUDA turns that into a multiplication by the reciprocal).  So it gives the same bits on the CPU, where the
fixtures are made by the reference's code, and on the GPU, where the kernels are checked against them.

A view is an axis-aligned pinhole camera: ``axes`` / ``signs`` pick the camera's right, down and forward world axes, the
pixel is (f * right / forward + W / 2 - 0.5, f * down / forward + H / 2 - 0.5), and the alpha a view integrates at a point
is 1 - k * |p - o|^2, so the cull SDF is max_k |p - o|^2 - 0.5 over the views that see the point: a sphere.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch


@dataclass
class View:
    axes: tuple            # world axis of camera right, down, forward
    signs: tuple           # +-1 per camera axis
    center: np.ndarray     # f32 [3]
    focal: float
    k: float               # alpha = 1 - k |p - origin|^2
    mask: np.ndarray       # f32 [H, W]: render[7]
    gt_mask: np.ndarray | None   # f32 [1, H, W] or None

    @property
    def image_height(self):
        return self.mask.shape[0]

    @property
    def image_width(self):
        return self.mask.shape[1]


ORIGIN = np.zeros(3, np.float32)


def integrate(points: torch.Tensor, view: View) -> dict:
    """The stand-in: ``{"alpha_integrated" [N], "point_coordinate" [N, 2], "render" [9, H, W]}`` on the points' device."""
    dev = points.device
    c = torch.from_numpy(np.asarray(view.center, np.float32)).to(dev)
    d = points - c
    cam = [d[:, a] * float(s) for a, s in zip(view.axes, view.signs)]
    H, W = view.image_height, view.image_width
    fwd = cam[2]
    u = (cam[0] / fwd) * float(view.focal) + float(W * 0.5 - 0.5)
    v = (cam[1] / fwd) * float(view.focal) + float(H * 0.5 - 0.5)
    behind = fwd <= 0
    far = torch.full_like(u, -1.0e4)
    u = torch.where(behind, far, u)
    v = torch.where(behind, far, v)
    o = points - torch.from_numpy(ORIGIN).to(dev)
    r2 = (o[:, 0] * o[:, 0] + o[:, 1] * o[:, 1]) + o[:, 2] * o[:, 2]
    alpha = 1.0 - r2 * float(view.k)
    render = torch.zeros((9, H, W), dtype=torch.float32, device=dev)
    render[7] = torch.from_numpy(view.mask).to(dev)
    return {"alpha_integrated": alpha, "point_coordinate": torch.stack([u, v], dim=-1), "render": render}


def _blocks(rng, H, W, values, p, block=12):
    """An [H, W] f32 image of constant 12x12 blocks, each one of ``values``.  Sampled values come near 0.5 only within a
    pixel of a block border, which keeps the fixtures' margin (no sample within 1e-5 of 0.5) easy to meet."""
    grid = rng.choice(np.asarray(values, np.float32), size=(-(-H // block), -(-W // block)), p=p)
    return np.ascontiguousarray(np.repeat(np.repeat(grid, block, 0), block, 1)[:H, :W], dtype=np.float32)


def make_views(seed: int, n_views: int, H: int, W: int, gt_every: int | None, blank: bool = False):
    """``n_views`` views around the origin, looking along +-x, +-y, +-z in turn; masks are seeded blocks with a zero
    rectangle (points there are not seen); every ``gt_every``-th view gets a 0/1 ground-truth mask.  ``blank``: all masks
    zero, so no point is seen and the surface is empty."""
    rng = np.random.default_rng(seed)
    dirs = [((1, 2, 0), (1, 1, 1)), ((0, 2, 1), (-1, 1, -1)), ((2, 1, 0), (1, 1, -1)), ((0, 1, 2), (1, 1, 1)), ((2, 0, 1), (1, 1, 1)),
            ((1, 0, 2), (1, 1, -1))]
    views = []
    for i in range(n_views):
        axes, signs = dirs[i % len(dirs)]
        center = np.zeros(3, np.float32)
        center[axes[2]] = -3.0 * signs[2]
        center += rng.normal(0, 0.05, 3).astype(np.float32)
        mask = _blocks(rng, H, W, (0.0, 0.3, 0.8, 1.0), (0.15, 0.1, 0.15, 0.6))
        y0, x0 = rng.integers(0, H // 2), rng.integers(0, W // 2)
        mask[y0:y0 + H // 4, x0:x0 + W // 4] = 0.0
        if blank:
            mask[:] = 0.0
        gt = None
        if gt_every and i % gt_every == 0:
            gt = _blocks(rng, H, W, (0.0, 1.0), (0.2, 0.8))[None]
        views.append(View(axes, signs, center.astype(np.float32), float(np.float32(W * 0.9)), float(np.float32(rng.uniform(0.8, 1.2))), mask, gt))
    return views


def views_of(d) -> list:
    """The views stored in a fixture (tests/golden/tetra/*.npz)."""
    views = []
    for i in range(int(d["n_views"].item())):
        fk = d[f"view{i}_focal_k"]
        views.append(View(tuple(int(a) for a in d[f"view{i}_axes"]), tuple(float(s) for s in d[f"view{i}_signs"]), d[f"view{i}_center"],
                          float(fk[0]), float(fk[1]), d[f"view{i}_mask"], d.get(f"view{i}_gt")))
    return views


def make_gaussians(seed: int, P: int):
    """P Gaussians near the unit sphere, with the raw parameters GaussianModel keeps: xyz, log-scales, raw rotation and
    filter_3D (f32 numpy)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(P, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    xyz = (d * rng.uniform(0.55, 0.9, (P, 1))).astype(np.float32)
    log_scale = np.log(rng.uniform(0.01, 0.06, (P, 3))).astype(np.float32)
    rot = rng.normal(size=(P, 4)).astype(np.float32)
    filt = rng.uniform(0.0, 0.01, (P, 1)).astype(np.float32)
    return xyz, log_scale, rot, filt


def sample_mask_f64(view: View, coord: np.ndarray) -> np.ndarray:
    """The bilinear, zero-padded sample of render[7] (* gt_mask) at the pixel coordinates, in fp64: the margin check's arbiter."""
    H, W = view.image_height, view.image_width
    m = view.mask.astype(np.float64)
    if view.gt_mask is not None:
        m = (view.mask * view.gt_mask[0]).astype(np.float64)   # the product is formed in fp32, as the reference does
    x = coord[:, 0].astype(np.float64)
    y = coord[:, 1].astype(np.float64)
    gx = (x * 2 + 1) / (W - 1) - 1
    gy = (y * 2 + 1) / (H - 1) - 1
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    x0, y0 = np.floor(ix), np.floor(iy)
    out = np.zeros(len(x))
    for dx in (0, 1):
        for dy in (0, 1):
            xc, yc = x0 + dx, y0 + dy
            w = (1 - np.abs(ix - xc)) * (1 - np.abs(iy - yc))
            ok = (xc >= 0) & (xc <= W - 1) & (yc >= 0) & (yc <= H - 1)
            val = np.zeros(len(x))
            val[ok] = m[yc[ok].astype(np.int64), xc[ok].astype(np.int64)]
            out += w * val
    return out
