"""Analytic depth / colour views for the TSDF tests: pinhole cameras (pixel centres at i + 0.5) looking at planes and
spheres, ray-cast in float64 and rounded to float32 once."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class View:
    K: np.ndarray        # 3x3 float64
    E: np.ndarray        # 4x4 float64 world -> camera
    depth: np.ndarray    # float32 [H, W]
    color: np.ndarray    # float32 [H, W, 3]


@dataclass
class Scene:
    vs: float
    depth_max: float
    views: list = field(default_factory=list)
    trunc_mult: float = 8.0
    depth_scale: float = 1.0


def look_at(eye, target, up=(0.0, 1.0, 0.0)):
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    z = target - eye
    z /= np.linalg.norm(z)
    if abs(np.dot(z, up / np.linalg.norm(up))) > 0.99:
        up = np.array([1.0, 0.0, 0.0])
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    E = np.eye(4)
    E[:3, :3] = np.stack([x, y, z])
    E[:3, 3] = -E[:3, :3] @ eye
    return E


def intrinsic(W, H, fov_deg=60.0, cx=None, cy=None):
    f = W / (2 * np.tan(np.radians(fov_deg) / 2))
    return np.array([[f, 0, W / 2 if cx is None else cx], [0, f, H / 2 if cy is None else cy], [0, 0, 1.0]])


def render(K, E, H, W, planes=(), spheres=(), max_depth=np.inf):
    """planes: (normal n, offset c) with n.x = c; spheres: (centre, radius).  Depth is camera z (0 where nothing is hit)."""
    j, i = np.mgrid[0:H, 0:W].astype(np.float64)
    dc = np.stack([(i + 0.5 - K[0, 2]) / K[0, 0], (j + 0.5 - K[1, 2]) / K[1, 1], np.ones_like(i)], -1)   # camera ray with z = 1
    R, t = E[:3, :3], E[:3, 3]
    C = -R.T @ t
    dw = dc @ R                      # R^T d per pixel
    best = np.full((H, W), np.inf)
    for n, c in planes:
        n = np.asarray(n, np.float64)
        den = dw @ n
        with np.errstate(divide="ignore", invalid="ignore"):
            s = (c - C @ n) / den
        best = np.where((s > 0) & (s < best), s, best)
    for ctr, r in spheres:
        oc = C - np.asarray(ctr, np.float64)
        a = np.sum(dw * dw, -1)
        b = 2 * dw @ oc
        cc = oc @ oc - r * r
        disc = b * b - 4 * a * cc
        with np.errstate(invalid="ignore"):
            s = (-b - np.sqrt(disc)) / (2 * a)
        best = np.where((disc >= 0) & (s > 0) & (s < best), s, best)
    depth = np.where(np.isfinite(best) & (best < max_depth), best, 0.0)
    p = C + dw * np.where(np.isfinite(best), best, 0.0)[..., None]
    color = 0.5 + 0.5 * np.sin(np.stack([3.1 * p[..., 0] + 0.3, 2.3 * p[..., 1] - 0.7, 1.7 * p[..., 2] + 1.1], -1))
    return depth.astype(np.float32), color.astype(np.float32)


def orbit(n, radius, target=(0.0, 0.0, 0.0), seed=0):
    """n camera centres spread over a sphere (Fibonacci lattice) around target."""
    k = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * k / n)
    th = np.pi * (1 + 5 ** 0.5) * k + seed
    d = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    return np.asarray(target) + radius * d


def sphere_scene(n_views=30, W=96, H=80, vs=0.02, r=0.3, centre=(0.0, 0.0, 0.0), dist=1.2, depth_max=3.0):
    sc = Scene(vs=vs, depth_max=depth_max)
    for eye in orbit(n_views, dist, centre):
        K = intrinsic(W, H, 50.0)
        E = look_at(eye, centre)
        d, c = render(K, E, H, W, spheres=[(centre, r)])
        sc.views.append(View(K, E, d, c))
    return sc


def make(name):
    """The scene families of the bit-exact tests."""
    if name == "fronto":
        sc = Scene(vs=0.01, depth_max=3.0)
        K, E = intrinsic(64, 48), np.eye(4)
        for k in range(4):
            d, c = render(K, E, 48, 64, planes=[((0, 0, 1.0), 1.2345 + 0.001 * k)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "tilted":
        sc = Scene(vs=0.01, depth_max=3.0)
        K = intrinsic(80, 60)
        for k in range(5):
            E = look_at((0.1 * k, -0.05 * k, -1.0), (0.0, 0.0, 0.5))
            d, c = render(K, E, 60, 80, planes=[((0.3, -0.2, 1.0), 0.6)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "sphere":
        return sphere_scene(12, 64, 48)
    if name == "occluders":
        sc = Scene(vs=0.015, depth_max=3.0)
        K = intrinsic(72, 56)
        for k in range(6):
            E = look_at((0.3 * np.cos(k), 0.2 * np.sin(k), -1.5), (0, 0, 0))
            d, c = render(K, E, 56, 72, planes=[((0, 0, 1.0), 0.4)], spheres=[((0.05, 0, -0.2), 0.15), ((-0.2, 0.1, 0.0), 0.1)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "masked":        # zero pixels (a mask) and pixels beyond depth_max
        sc = Scene(vs=0.01, depth_max=1.3)
        K = intrinsic(64, 48)
        rng = np.random.default_rng(3)
        for k in range(4):
            E = look_at((0.02 * k, 0, -1.0), (0, 0, 0.3))
            d, c = render(K, E, 48, 64, planes=[((0.1, 0.4, 1.0), 0.2)])
            d[rng.random(d.shape) < 0.2] = 0.0
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "on_grid":       # the plane z = 0.75 passes through grid points: tsdf exactly 0 there (0 is outside)
        sc = Scene(vs=1 / 64, depth_max=3.0)
        K = intrinsic(64, 48)
        for k in range(4):
            d, c = render(K, np.eye(4), 48, 64, planes=[((0, 0, 1.0), 0.75)])
            sc.views.append(View(K, np.eye(4), d, c))
        return sc
    if name == "far_negative":  # blocks far from the origin at negative coordinates
        sc = Scene(vs=0.01, depth_max=3.0)
        ctr = np.array([-3000.0, -1200.5, -2500.25])
        for eye in orbit(6, 1.0, ctr, seed=1):
            K, E = intrinsic(48, 40, 45.0), look_at(eye, ctr)
            d, c = render(K, E, 40, 48, spheres=[(ctr, 0.25)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "straddle":      # a plane on a block boundary (x = 16 vs)
        sc = Scene(vs=0.01, depth_max=3.0)
        K = intrinsic(64, 48)
        for k in range(4):
            E = look_at((-0.8, 0.01 * k, 0.05), (0.5, 0.0, 0.0))
            d, c = render(K, E, 48, 64, planes=[((1.0, 0, 0), 0.16)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name in ("1x1", "7x5", "800x600"):
        W, H = map(int, name.split("x"))
        sc = Scene(vs=0.01 if W > 100 else 0.004, depth_max=3.0)
        K = intrinsic(W, H, 40.0)
        for k in range(3):
            E = look_at((0.05 * k, 0, -1.0), (0, 0, 0))
            d, c = render(K, E, H, W, planes=[((0.2, 0.1, 1.0), 0.1)], spheres=[((0, 0, -0.1), 0.2)])
            sc.views.append(View(K, E, d, c))
        return sc
    if name == "few_views":     # two views: every weight stays below the threshold 3
        return sphere_scene(2, 64, 48)
    if name == "many_views":
        return sphere_scene(40, 48, 40)
    raise ValueError(name)


FAMILIES = ["fronto", "tilted", "sphere", "occluders", "masked", "on_grid", "far_negative", "straddle", "1x1", "7x5", "800x600", "few_views", "many_views"]
