"""Scene families aimed at the integrate kernels' edges (test_gpu_integrate_exact.py, test_integrate_f64_host.py).  Each family
is a Case: splats, query points, the SH degree or precomputed colours.  Built in camera space (identity view, blend_scenes.build)
where a point has to land on a given pixel or depth."""
from __future__ import annotations

import math
import os
import sys
from dataclasses import dataclass

import numpy as np
import torch

import blend_scenes as bs
from rade_gs_b200 import scenes

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gen_golden_integrate import make_points  # noqa: E402


@dataclass
class Case:
    sc: scenes.Scene
    points: torch.Tensor          # [PN,3] world space
    deg: int = 3
    colors_precomp: torch.Tensor | None = None


def _U(g):
    return lambda *s: torch.rand(*s, generator=g)


def _cam_points(sc, u, v, z):
    """World points (identity view) whose fp32 projection is exactly (u, v) at view depth z where that is representable: x is
    nudged ulp by ulp until the kernel's expression float(focal * x / (z + 1e-7f) + W / 2.) gives u."""
    fx = np.float32(sc.width / (2.0 * np.float32(sc.tanfovx)))
    fy = np.float32(sc.height / (2.0 * np.float32(sc.tanfovy)))
    z = np.asarray(z, np.float32)
    den = z + np.float32(1e-7)

    def solve(target, f, size):
        x = ((np.asarray(target, np.float64) - size / 2.0) * den / f).astype(np.float32)
        for _ in range(64):
            im = (f * x / den).astype(np.float64) + size / 2.0
            im = im.astype(np.float32).astype(np.float64)
            off = im - target
            if not (off != 0).any():
                break
            x = np.where(off > 0, np.nextafter(x, np.float32(-np.inf)), np.where(off < 0, np.nextafter(x, np.float32(np.inf)), x))
        return x

    x = solve(u, fx, sc.width)
    y = solve(v, fy, sc.height)
    return torch.from_numpy(np.stack([x, y, z], 1).astype(np.float32))


def generic():
    """A C1-sized scene (300k splats, 800x800) with 10^6 points made the way mesh extraction makes them."""
    sc = scenes.make_config("C1")[0]
    return Case(sc, make_points(sc, 1_000_000, 41))


def ragged(W, H, P, seed):
    """Ragged image sizes, with points in the last (partial) tile row and column."""
    sc = bs.tiny(W, H, P, seed)
    g = torch.Generator().manual_seed(seed + 1)
    U = _U(g)
    n = 400
    z = (2.0 + 4.0 * U(n)).float()
    u = torch.where(U(n) < 0.5, (W - 1) // 16 * 16 + U(n) * (W - (W - 1) // 16 * 16), U(n) * W)
    v = torch.where(U(n) < 0.5, (H - 1) // 16 * 16 + U(n) * (H - (H - 1) // 16 * 16), U(n) * H)
    pts = _cam_points(sc, u.double().numpy(), v.double().numpy(), z.numpy())
    return Case(sc, torch.cat([make_points(sc, 3000, seed + 2), pts]).contiguous())


def edge_points():
    """Points whose fp32 projection is exactly an integer pixel coordinate, a multiple of 16, or one ulp below W / H; points
    at view z = 0.2f and one ulp either side; points behind the camera and outside the image."""
    W, H = 96, 80
    sc = bs.tiny(W, H, 600, 51)
    g = torch.Generator().manual_seed(52)
    U = _U(g)
    ints = np.arange(0, W, 1.0)
    n = ints.size
    z = (2.0 + 4.0 * U(n)).numpy()
    a = _cam_points(sc, ints, (U(n) * H).double().numpy(), z)                       # integer x
    b = _cam_points(sc, (U(H) * W).double().numpy(), np.arange(0, H, 1.0), (2.0 + 4.0 * U(H)).numpy())  # integer y
    mx, my = np.arange(0, W, 16.0), np.arange(0, H, 16.0)
    c = _cam_points(sc, np.repeat(mx, my.size), np.tile(my, mx.size), np.full(mx.size * my.size, 3.0, np.float32))
    below = np.array([np.nextafter(np.float32(W), np.float32(0))] * 8, np.float64)
    d = _cam_points(sc, below, (U(8) * H).double().numpy(), np.full(8, 3.0, np.float32))
    belowy = np.array([np.nextafter(np.float32(H), np.float32(0))] * 8, np.float64)
    e = _cam_points(sc, (U(8) * W).double().numpy(), belowy, np.full(8, 3.0, np.float32))
    z02 = np.float32(0.2)
    zs = np.array([np.nextafter(z02, np.float32(0)), z02, np.nextafter(z02, np.float32(1))] * 10, np.float32)
    f = torch.stack([(U(30) - 0.5).float() * 0.1, (U(30) - 0.5).float() * 0.1, torch.from_numpy(zs)], 1)
    behind = torch.stack([U(50) - 0.5, U(50) - 0.5, -U(50) * 3], 1).float()
    outside = torch.stack([(U(50) + 1.2) * 3 * torch.sign(U(50) - 0.5), U(50) - 0.5, 3 + U(50)], 1).float()
    return Case(sc, torch.cat([a, b, c, d, e, f, behind, outside, make_points(sc, 2000, 53)]).contiguous(), deg=1)


def degenerate():
    """Needles and flat discs: discs thinner than the well-conditioned limit take `condition == 0` (zero invray, skip in
    front of the plane, dz = tcen behind it); points on both sides of every splat's plane."""
    nd = bs.needles(128, 96, 300, seed=61)
    g = torch.Generator().manual_seed(62)
    U = _U(g)
    P = 300
    z = 2.0 + 4.0 * U(P)
    thin = torch.where(torch.arange(P) % 2 == 0, torch.full((P,), 1e-6), torch.full((P,), 1e-3))
    s = (2.0 + 4.0 * U(P)) * z / 100.0
    scales = torch.stack([s, s * (0.5 + U(P)), thin], 1)
    q = torch.randn(P, 4, generator=g)
    disc = bs.build(128, 96, 100.0, U(P) * 128, U(P) * 96, z, scales, q / q.norm(dim=1, keepdim=True), 0.3 + 0.7 * U(P), 63)
    sc = scenes.Scene(torch.cat([nd.means3D, disc.means3D]), torch.cat([nd.scales, disc.scales]), torch.cat([nd.rotations, disc.rotations]),
                      torch.cat([nd.opacities, disc.opacities]), torch.cat([nd.shs, disc.shs]), disc.viewmatrix, disc.projmatrix, disc.campos,
                      disc.bg, 128, 96, disc.tanfovx, disc.tanfovy)
    # points just in front of and just behind each splat along the view ray, and the box corners
    c = sc.means3D
    ray = c / c.norm(dim=1, keepdim=True)
    d = torch.cat([c - 0.02 * ray, c + 0.02 * ray, c - 0.3 * ray, c + 0.3 * ray])
    return Case(sc, torch.cat([d, make_points(sc, 6000, 64)]).contiguous())


def deep_lists():
    """Tiles whose lists hold 255/256/257, 8191/8192/8193 and 70 000 entries.  In the 70 000-entry tile the nearer entries are
    small splats on the left half of the tile and the last 600 (deepest) cover the right half, so right-half pixels have
    contributors past list position 65 536.  Every tile after the first starts at a range.x that is not a multiple of 32."""
    lengths = [255, 256, 257, 8191, 8192, 8193]
    g = torch.Generator().manual_seed(71)
    U = _U(g)
    focal = 120.0
    us, vs, zs, ss, os_ = [], [], [], [], []
    for i, n in enumerate(lengths):
        us.append(16 * i + 7.5 + (U(n) * 2 - 1))
        vs.append(7.5 + (U(n) * 2 - 1))
        zs.append(2.0 + 6.0 * U(n))
        ss.append((0.8 + 0.8 * U(n, 3)))
        os_.append(torch.full((n,), min(0.02, 160.0 / n)) * (1 + U(n)))
    n_far, n_near = 600, 70_000 - 600
    x0 = 16 * len(lengths)
    us += [x0 + 1.0 + 5.0 * U(n_near), x0 + 10.0 + 4.0 * U(n_far)]
    vs += [1.0 + 14.0 * U(n_near), 1.0 + 14.0 * U(n_far)]
    zs += [2.0 + 2.0 * U(n_near), 6.0 + 1.0 * U(n_far)]
    ss += [0.25 + 0.1 * U(n_near, 3), 0.8 + 0.4 * U(n_far, 3)]
    os_ += [0.1 + 0.2 * U(n_near), 0.02 + 0.02 * U(n_far)]
    u, v, z, o = torch.cat(us), torch.cat(vs), torch.cat(zs), torch.cat(os_)
    P = u.shape[0]
    sig = torch.cat(ss) * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    sc = bs.build(16 * (len(lengths) + 1), 16, focal, u, v, z, sig, q / q.norm(dim=1, keepdim=True), o, 72)
    uu = torch.arange(sc.width).repeat(16).double() + 0.25
    vv = torch.arange(16).repeat_interleave(sc.width).double() + 0.75
    pts = _cam_points(sc, uu.numpy(), vv.numpy(), (1.5 + 6.0 * U(uu.numel())).numpy())
    return Case(sc, torch.cat([pts, make_points(sc, 8000, 73)]).contiguous(), deg=0)


def overflow():
    """3000 wide splats with alpha just above 1/255 everywhere in a 16x16 image: every pixel reaches 2048 used entries."""
    g = torch.Generator().manual_seed(81)
    U = _U(g)
    P, focal = 3000, 40.0
    z = 2.0 + 6.0 * U(P)
    sig = (50.0 * z / focal)[:, None].expand(P, 3).clone()
    sc = bs.build(16, 16, focal, 7.5 + U(P) - 0.5, 7.5 + U(P) - 0.5, z, sig, torch.tensor([[1.0, 0, 0, 0]]).expand(P, 4), torch.full((P,), 0.0042), 82)
    uu = torch.arange(16).repeat(16).double() + 0.5
    vv = torch.arange(16).repeat_interleave(16).double() + 0.5
    pts = torch.cat([_cam_points(sc, uu.numpy(), vv.numpy(), np.full(256, z_, np.float32)) for z_ in (1.0, 5.0, 9.0)])
    return Case(sc, pts.contiguous(), deg=0)


def corners_crowding():
    """Opaque small splats centred near pixel corners: the centre sample stops early while corner samples go on, so entries are
    used through corners only.  Plus 1500 points on one camera ray (one pixel) and duplicated points."""
    g = torch.Generator().manual_seed(91)
    U = _U(g)
    W, H, P, focal = 64, 48, 4000, 60.0
    z = 2.0 + 6.0 * U(P)
    u = torch.randint(0, W + 1, (P,), generator=g).double() + 0.08 * (U(P) - 0.5)
    v = torch.randint(0, H + 1, (P,), generator=g).double() + 0.08 * (U(P) - 0.5)
    sig = (0.25 + 0.3 * U(P, 3)) * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    sc = bs.build(W, H, focal, u, v, z, sig, q / q.norm(dim=1, keepdim=True), 0.95 + 0.05 * U(P), 92)
    zr = torch.linspace(1.0, 9.0, 1500)
    ray = torch.stack([0.013 * zr, -0.021 * zr, zr], 1)
    base = make_points(sc, 6000, 93)
    return Case(sc, torch.cat([base, ray, base[:500], base[:500]]).contiguous())


def colours(kind):
    """SH degree 0 / 3, precomputed colours; every case with a nonzero background."""
    sc = bs.tiny(80, 64, 1500, 101)
    pts = make_points(sc, 8000, 102)
    if kind == "precomp":
        g = torch.Generator().manual_seed(103)
        return Case(sc, pts, deg=0, colors_precomp=torch.rand(sc.means3D.shape[0], 3, generator=g) * 1.5 - 0.2)
    return Case(sc, pts, deg=0 if kind == "sh0" else 3)


FAMILIES = {
    "generic_C1": generic,
    "ragged_97x61": lambda: ragged(97, 61, 400, 21),
    "ragged_1x1": lambda: ragged(1, 1, 31, 22),
    "ragged_1000x3": lambda: ragged(1000, 3, 300, 23),
    "edge_points": edge_points,
    "degenerate": degenerate,
    "deep_lists": deep_lists,
    "overflow": overflow,
    "corners_crowding": corners_crowding,
    "colour_sh0": lambda: colours("sh0"),
    "colour_sh3": lambda: colours("sh3"),
    "colour_precomp": lambda: colours("precomp"),
}
