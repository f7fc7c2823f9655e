"""Scene families aimed at the blend kernels' culling and list handling (used by test_blend_f64_host.py and
test_gpu_blend_exact.py).  Every scene is built in camera space (identity view) from a seed, so a splat can be put on a given
pixel: u = focal x / z + (W - 1) / 2.  scenes.make_scene is not used: its draw order is pinned by fixture digests."""
from __future__ import annotations

import math

import torch

from rade_gs_b200 import scenes


def _quat_z(theta):
    """Unit quaternion (r, x, y, z) of a rotation by theta about the optical axis."""
    return torch.stack([torch.cos(theta / 2), torch.zeros_like(theta), torch.zeros_like(theta), torch.sin(theta / 2)], 1)


def build(W, H, focal, u, v, z, scales, rots, opac, seed=0, bg=(0.2, 0.3, 0.1)) -> scenes.Scene:
    """Scene with centres at pixel (u, v), depth z; scales [P,3], unit quaternions [P,4], opacities [P]."""
    g = torch.Generator().manual_seed(seed)
    P = u.shape[0]
    x = (u - (W - 1) / 2) * z / focal
    y = (v - (H - 1) / 2) * z / focal
    tanx, tany = W / (2 * focal), H / (2 * focal)
    proj = scenes.projection_matrix(0.01, 100.0, 2 * math.atan(tanx), 2 * math.atan(tany)).t().contiguous()
    sh = torch.cat([torch.randn(P, 1, 3, generator=g), 0.1 * torch.randn(P, 15, 3, generator=g)], 1)
    return scenes.Scene(torch.stack([x, y, z], 1).float().contiguous(), scales.float().contiguous(), rots.float().contiguous(),
                        opac.float().reshape(P, 1).contiguous(), sh.contiguous(), torch.eye(4), proj, torch.zeros(3),
                        torch.tensor(bg, dtype=torch.float32), W, H, tanx, tany)


def needles(W=96, H=64, P=120, seed=1):
    """Scale ratios 1e3-1e4, in-plane long axis crossing many 8x4 blocks; a third each random, axis-aligned and 45 degrees."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal, z = 0.9 * W, 3.0 + 4.0 * U(P)
    long = (0.3 + 0.7 * U(P)) * W * z / focal           # screen length ~0.3-1 image width (one sigma)
    ratio = 10.0 ** (3 + U(P))
    scales = torch.stack([long, long / ratio, long / ratio], 1)
    k = torch.arange(P) % 3
    theta = torch.where(k == 0, U(P) * 2 * math.pi, torch.where(k == 1, (U(P) < 0.5).float() * (math.pi / 2), torch.full((P,), math.pi / 4)))
    rots = _quat_z(theta)
    tilt = torch.randn(P, 4, generator=g)
    rots = torch.where((torch.arange(P) % 6 == 0)[:, None], tilt / tilt.norm(dim=1, keepdim=True), rots)  # a few fully random
    return build(W, H, focal, U(P) * W, U(P) * H, z, scales, rots, 0.2 + 0.8 * U(P), seed)


def huge_near(W=96, H=64, P=60, seed=2):
    """Splats wider than the image, and centres at z in (0.2, 0.25)."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal = 0.9 * W
    near = torch.arange(P) % 2 == 0
    z = torch.where(near, 0.2 + 0.05 * U(P), 3.0 + 3.0 * U(P))
    s = torch.where(near, 0.002 + 0.01 * U(P), (1.0 + 2.0 * U(P)) * W * z / focal)
    scales = s[:, None] * (0.5 + U(P, 3))
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, U(P) * W, U(P) * H, z, scales, q / q.norm(dim=1, keepdim=True), 0.05 + 0.5 * U(P), seed)


def deep(lengths, opaque=False, seed=3, focal=120.0):
    """One pile per 16x16 tile, pile i with exactly lengths[i] splats: every splat's footprint stays inside its tile (centre
    within 1 px of the tile centre, radius 3 sigma <= 6 px).  Low opacity (the whole list matters) or, with `opaque`, opacities
    up to 1 so that the pixels of one warp stop at different list positions."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    W, H = 16 * len(lengths), 16
    us, vs, ops = [], [], []
    for i, n in enumerate(lengths):
        us.append(16 * i + 7.5 + (U(n) * 2 - 1))
        vs.append(7.5 + (U(n) * 2 - 1))
        ops.append(0.3 + 0.7 * U(n) if opaque else torch.full((n,), min(0.02, 160.0 / n)) * (1 + U(n)))
    u, v, o = torch.cat(us), torch.cat(vs), torch.cat(ops)
    P = u.shape[0]
    z = 2.0 + 6.0 * U(P)
    sig = (0.8 + 0.8 * U(P, 3)) * z[:, None] / focal      # <= 1.6 px
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, u, v, z, sig, q / q.norm(dim=1, keepdim=True), o, seed)


def opaque(W=64, H=48, P=300, seed=4):
    """Stacks of opacity-1.0 splats: alpha is clamped at 0.99 and T_final falls next to 1e-4."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal = 0.9 * W
    z = 2.0 + 6.0 * U(P)
    scales = (2.0 + 6.0 * U(P, 3)) * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, U(P) * W, U(P) * H, z, scales, q / q.norm(dim=1, keepdim=True), torch.ones(P), seed)


def faint(W=64, H=48, P=400, seed=5):
    """Opacity just above 1/255: alpha >= 1/255 only right at the centres, where the decision is close."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal = 0.9 * W
    z = 2.0 + 6.0 * U(P)
    scales = (1.0 + 6.0 * U(P, 3)) * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, U(P) * W, U(P) * H, z, scales, q / q.norm(dim=1, keepdim=True), (1 / 255) * (1 + 0.01 * U(P)), seed)


def frustum_edge(W=96, H=64, P=80, seed=6):
    """Centres beyond 1.3 tan(fov) (preprocess clamps them for the Jacobian) whose footprints reach into the image."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal = 0.9 * W
    z = 2.0 + 4.0 * U(P)
    side = torch.randint(0, 4, (P,), generator=g)
    out = 1.3 * 0.5 + 0.05 + 0.3 * U(P)                   # offset from the centre over the image size; the clamp is at 0.65
    u = torch.where(side == 0, (W - 1) / 2 + out * W, torch.where(side == 1, (W - 1) / 2 - out * W, U(P) * W))
    v = torch.where(side == 2, (H - 1) / 2 + out * H, torch.where(side == 3, (H - 1) / 2 - out * H, U(P) * H))
    scales = (0.3 + 0.5 * U(P, 3)) * W * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, u, v, z, scales, q / q.norm(dim=1, keepdim=True), 0.3 + 0.7 * U(P), seed)


def tiny(W, H, P, seed=7):
    """Ragged and tiny images with few splats."""
    g = torch.Generator().manual_seed(seed)
    U = lambda *s: torch.rand(*s, generator=g)
    focal = 0.9 * max(W, H) + 2.0
    z = 2.0 + 4.0 * U(P)
    scales = (0.5 + 3.0 * U(P, 3)) * z[:, None] / focal
    q = torch.randn(P, 4, generator=g)
    return build(W, H, focal, U(P) * W, U(P) * H, z, scales, q / q.norm(dim=1, keepdim=True), 0.1 + 0.9 * U(P), seed)
