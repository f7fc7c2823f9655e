"""Analytic views for the unbounded-mesh tests and benchmark: cameras in the reference's conventions
(``world_view_transform`` = the transposed world->view matrix, ``full_proj_transform`` = world_view_transform @
projection^T, z in [0, 1]) and per-pixel depth / RGB maps ray-cast from a unit sphere, a ground plane and a far
background sphere, so that samples land in the contracted region too.  Also a torch restatement of the reference's eager
TSDF expressions (utils/mesh_utils.py:171-232), used as the eager comparison and for the fp32-vs-fp64 error bound."""
from __future__ import annotations

import math

import numpy as np
import torch

SPHERE_R = 1.0
GROUND_Z = -1.2
SKY_R = 12.0


def camera(eye, target=(0.0, 0.0, 0.0), W=64, H=48, fovx=math.radians(60)):
    """(world_view_transform, full_proj_transform) fp32 [4, 4] of a pinhole at `eye` looking at `target` (y down)."""
    from rade_gs_b200 import scenes as sc
    fovy = 2 * math.atan(math.tan(fovx / 2) * H / W)
    up = (0.0, 0.0, -1.0) if abs(eye[2]) < 0.95 * math.dist(eye, target) else (0.0, -1.0, 0.0)
    V = sc.look_at_view(eye, target, up=up)
    Pm = sc.projection_matrix(0.01, 100.0, fovx, fovy)
    return V.t().contiguous(), (V.t() @ Pm.t()).contiguous()


def ring(n, dist=3.0, height=0.6, seed=0):
    g = np.random.default_rng(seed)
    a = 2 * np.pi * (np.arange(n) / n) + g.uniform(0, 0.1)
    h = height + g.uniform(-0.3, 0.3, n)
    return [(float(dist * np.cos(t)), float(dist * np.sin(t)), float(z)) for t, z in zip(a, h)]


def _hits(o, d):
    """Nearest positive ray parameter against the sphere, the ground and the sky (d need not be unit)."""
    def sphere(r):
        b = (o * d).sum(-1)
        a = (d * d).sum(-1)
        c = (o * o).sum(-1) - r * r
        disc = b * b - a * c
        s = np.sqrt(np.maximum(disc, 0))
        t0, t1 = (-b - s) / a, (-b + s) / a
        t = np.where(t0 > 1e-6, t0, t1)
        return np.where((disc >= 0) & (t > 1e-6), t, np.inf)
    with np.errstate(all="ignore"):
        tg = (GROUND_Z - o[..., 2]) / d[..., 2]
    tg = np.where(tg > 1e-6, tg, np.inf)
    return np.minimum(np.minimum(sphere(SPHERE_R), tg), sphere(SKY_R))


def maps(eye, wvt, W, H, fovx=math.radians(60)):
    """(depth [H, W], rgb [3, H, W]) fp32: view-space z of the first hit through each pixel's grid_sample position."""
    fovy = 2 * math.atan(math.tan(fovx / 2) * H / W)
    Vm = wvt.double().numpy().T                         # world -> view (column vectors)
    R = Vm[:3, :3]
    u = 2 * np.arange(W) / (W - 1) - 1
    v = 2 * np.arange(H) / (H - 1) - 1
    uu, vv = np.meshgrid(u, v)
    dc = np.stack([uu * math.tan(fovx / 2), vv * math.tan(fovy / 2), np.ones_like(uu)], -1)   # camera ray with z = 1
    dw = dc @ R                                          # R^T dc per row
    o = np.broadcast_to(np.asarray(eye, np.float64), dw.shape)
    t = _hits(o, dw)
    p = o + t[..., None] * dw
    rgb = 0.5 + 0.45 * np.stack([np.sin(1.3 * p[..., 0]), np.cos(1.7 * p[..., 1]), np.sin(0.9 * p[..., 2] + 0.5)])
    return t.astype(np.float32), rgb.astype(np.float32)


def views(n, W=64, H=48, seed=0, dist=3.0):
    """(depths [V, H, W], rgbs [V, 3, H, W], world_view [V, 4, 4], full_proj [V, 4, 4]) on the CPU."""
    eyes = ring(n, dist=dist, seed=seed)
    D, C, WV, FP = [], [], [], []
    for e in eyes:
        wvt, fp = camera(e, W=W, H=H)
        d, c = maps(e, wvt, W, H)
        D.append(d)
        C.append(c)
        WV.append(wvt)
        FP.append(fp)
    return torch.from_numpy(np.stack(D)), torch.from_numpy(np.stack(C)), torch.stack(WV), torch.stack(FP)


def sphere_xyz(P=4000, seed=1):
    g = np.random.default_rng(seed)
    n = g.normal(size=(P, 3))
    return torch.from_numpy((SPHERE_R * n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32))


# ---- the reference's eager expressions, restated in torch (any device, fp32 or fp64) --------------------------------

def torch_tsdf(samples, center, radius, voxel_size, depths, proj, dtype=torch.float32, rgbs=None, contracted=True, margins=False):
    """compute_unbounded_tsdf as the reference writes it (utils/mesh_utils.py:193-232), in `dtype`.  contracted=True:
    `samples` [N, 3] are contracted coordinates (inv_contraction, adaptive truncation); False: world points and the constant
    truncation of the colouring pass.  Returns (tsdf [N], weight [N]), then rgb [N, 3] when `rgbs` is given, then, with
    margins=True, each sample's smallest distance over the views to a discrete decision (|pix| = 1, w = 0, sdf = -trunc,
    and |s| = 1 / |p| = 1 of the contraction and the truncation)."""
    x = samples.to(dtype)
    big = torch.full_like(x[:, 0], float("inf"))
    margin = big.clone()
    if contracted:
        center = torch.as_tensor(np.asarray(center), dtype=dtype, device=x.device)
        mag = torch.linalg.norm(x, ord=2, dim=-1)[..., None]
        margin = torch.minimum(margin, (mag[:, 0] - 1).abs())
        x = torch.where(mag < 1, x, (1 / (2 - mag) * (x / mag)))
        x = x * radius + center
        mask = torch.linalg.norm(x, dim=-1) > 1
        margin = torch.minimum(margin, (torch.linalg.norm(x, dim=-1) - 1).abs())
        trunc = 5 * voxel_size * torch.ones_like(x[:, 0])
        trunc[mask] *= 1 / (2 - torch.linalg.norm(x, dim=-1)[mask].clamp(max=1.9))
    else:
        trunc = 5 * voxel_size
    t = torch.ones_like(x[:, 0])
    w = torch.ones_like(x[:, 0])
    col = torch.zeros((x.shape[0], 3), dtype=dtype, device=x.device)
    for i in range(depths.shape[0]):
        M = proj[i].to(dtype=dtype, device=x.device)
        h = torch.cat([x, torch.ones_like(x[..., :1])], dim=-1) @ M
        z = h[..., -1:]
        pix = h[..., :2] / h[..., -1:]
        mp = ((pix > -1.) & (pix < 1.) & (z > 0)).all(dim=-1)
        g = pix[None, None]
        d = torch.nn.functional.grid_sample(depths[i][None, None].to(dtype=dtype, device=x.device), g, mode="bilinear",
                                            padding_mode="border", align_corners=True).reshape(-1, 1)
        sdf = (d - z).flatten()
        if margins:
            m = torch.minimum((pix.abs() - 1).abs().amin(-1), z[:, 0].abs())
            m = torch.where(mp, torch.minimum(m, (sdf + trunc).abs()), m)
            margin = torch.minimum(margin, torch.nan_to_num(m, nan=0.0))
        mp = mp & (sdf > -trunc)
        if rgbs is not None:
            c = torch.nn.functional.grid_sample(rgbs[i][None].to(dtype=dtype, device=x.device), g, mode="bilinear", padding_mode="border",
                                                align_corners=True).reshape(3, -1).T
        sdf = torch.clamp(sdf / trunc, min=-1.0, max=1.0)[mp]
        wm = w[mp]
        t[mp] = (t[mp] * wm + sdf) / (wm + 1)
        if rgbs is not None:
            col[mp] = (col[mp] * wm[:, None] + c[mp]) / (wm + 1)[:, None]
        w[mp] = wm + 1
    out = (t, w) + ((col,) if rgbs is not None else ()) + ((margin,) if margins else ())
    return out
