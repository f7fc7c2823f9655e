"""Deterministic synthetic scenes and cameras for parity tests and the benchmark (SURVEY.md appendix C).

Nothing here is on the product path; it only produces inputs of the shape the reference's ``render()`` hands to
the rasterizer (``gaussian_renderer/__init__.py:35-71``): positions, activated scales / opacities, unit
quaternions, SH coefficients ``[P,16,3]``, and the camera matrices in the reference's transposed (row-vector)
convention (``scene/cameras.py:54-57``, ``utils/graphics_utils.py:67-87``).
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass

import torch

# name -> (P, W, H, focal_px, log-scale mean, require_coord, require_depth)   (BASELINE.md section 2)
CONFIGS = {
    "C1": (300_000, 800, 800, 1100.0, -4.4, False, True),
    "C2": (1_000_000, 1600, 1200, 1400.0, -4.6, False, True),
    "C3": (3_000_000, 1920, 1080, 1600.0, -5.0, True, False),
    "C4": (10_000_000, 4096, 4096, 3600.0, -5.6, False, True),
}


@contextlib.contextmanager
def _one_thread():
    """Synthesis on one CPU thread: torch's threaded, vectorised exp / normal sampling can change last bits with the thread
    count, and the stored fixtures pin these inputs by their bits (tools/golden_inputs.py)."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        yield
    finally:
        torch.set_num_threads(n)


@dataclass
class Scene:
    means3D: torch.Tensor      # [P,3]
    scales: torch.Tensor       # [P,3] activated
    rotations: torch.Tensor    # [P,4] unit (r,x,y,z)
    opacities: torch.Tensor    # [P,1] activated
    shs: torch.Tensor          # [P,16,3]
    viewmatrix: torch.Tensor   # [4,4] world_view_transform (transposed convention)
    projmatrix: torch.Tensor   # [4,4] full_proj_transform
    campos: torch.Tensor       # [3]
    bg: torch.Tensor           # [3]
    width: int
    height: int
    tanfovx: float
    tanfovy: float

    def to(self, device):
        kw = {}
        for k, v in self.__dict__.items():
            kw[k] = v.to(device) if isinstance(v, torch.Tensor) else v
        return Scene(**kw)


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    """OpenGL-style perspective with z in [0,1], as the reference builds it (utils/graphics_utils.py:67-87)."""
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def look_at_view(eye, target, up=(0.0, -1.0, 0.0)) -> torch.Tensor:
    """world->view 4x4 (maths convention, column vectors) for a camera at `eye` looking at `target`, +z forward."""
    eye = torch.tensor(eye, dtype=torch.float64)
    f = torch.tensor(target, dtype=torch.float64) - eye
    f = f / f.norm()
    upv = torch.tensor(up, dtype=torch.float64)
    r = torch.linalg.cross(upv, f)
    r = r / r.norm()
    u = torch.linalg.cross(f, r)
    R = torch.stack([r, u, f])  # rows
    V = torch.eye(4, dtype=torch.float64)
    V[:3, :3] = R
    V[:3, 3] = -R @ eye
    return V.float()


def make_scene(P: int, W: int, H: int, focal: float, mu: float, seed: int = 1234, sh_rest_std: float = 0.1,
               view: torch.Tensor | None = None, bg=(0.0, 0.0, 0.0), zmin: float = 2.0, zmax: float = 10.0) -> Scene:
    """SURVEY.md appendix C recipe.  Draw order: z, x, y, scales, rotations, opacity, SH-dc, SH-rest."""
    with _one_thread():
        return _make_scene(P, W, H, focal, mu, seed, sh_rest_std, view, bg, zmin, zmax)


def _make_scene(P, W, H, focal, mu, seed, sh_rest_std, view, bg, zmin, zmax) -> Scene:
    g = torch.Generator().manual_seed(seed)
    tanx, tany = W / (2 * focal), H / (2 * focal)

    def U(*shape):
        return torch.rand(*shape, generator=g)

    def N(*shape):
        return torch.randn(*shape, generator=g)

    z = U(P) * (zmax - zmin) + zmin
    x = (U(P) * 2 - 1) * 1.1 * tanx * z
    y = (U(P) * 2 - 1) * 1.1 * tany * z
    pts_cam = torch.stack([x, y, z], dim=1)
    scales = torch.exp(N(P, 3) * 0.6 + mu)
    rot = N(P, 4)
    rot = rot / rot.norm(dim=1, keepdim=True)
    opacity = torch.sigmoid(N(P, 1) * 2)
    sh = torch.cat([N(P, 1, 3), sh_rest_std * N(P, 15, 3)], dim=1)

    Vm = torch.eye(4) if view is None else view          # maths convention (column vectors)
    # place the points in the world so that they land where the recipe put them in camera space
    Rinv = Vm[:3, :3].t()
    means = (pts_cam - Vm[:3, 3]) @ Rinv.t()
    viewmatrix = Vm.t().contiguous()                      # reference stores the transpose
    proj = projection_matrix(0.01, 100.0, 2 * math.atan(tanx), 2 * math.atan(tany)).t()
    projmatrix = (viewmatrix @ proj).contiguous()
    campos = viewmatrix.inverse()[3, :3].contiguous()
    return Scene(means.contiguous(), scales, rot, opacity, sh.contiguous(), viewmatrix, projmatrix, campos,
                 torch.tensor(bg, dtype=torch.float32), W, H, tanx, tany)


def make_config(name: str, seed: int = 1234) -> tuple[Scene, bool, bool]:
    P, W, H, f, mu, coord, depth = CONFIGS[name]
    return make_scene(P, W, H, f, mu, seed=seed), coord, depth


def make_upstream_grads(H: int, W: int, seed: int = 4321, device="cpu") -> dict:
    """Upstream gradients ~N(0,1) per pixel-channel; depth / normal / alpha / coord grads scaled 0.1 (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)

    def N(c, s=1.0):
        return (torch.randn(c, H, W, generator=g) * s).to(device)

    with _one_thread():
        return {
            "color": N(3), "coord": N(3, 0.1), "mcoord": N(3, 0.1), "depth": N(1, 0.1), "mdepth": N(1, 0.1),
            "alpha": N(1, 0.1), "normal": N(3, 0.1),
        }
