"""numpy float32 restatement of the bounded-TSDF contract at ``rgs_scalable_*`` in include/rgs_b200.h (RGBD conversion,
strided touch, ray-distance integration, the shifted extraction), operation by operation, so that every stored bit of the
kernels can be compared.  Test infrastructure only.  The grid is tsdf_f32's dict  key -> (tsdf, weight, color)."""
from __future__ import annotations

import numpy as np

import tsdf_f32 as T

F = np.float32


def numpy_u8(x):
    """numpy's float32 -> uint8 cast on x86-64, stated: the low byte of the int32 truncation, 0 for NaN and |x| >= 2^31."""
    x = np.asarray(x, F)
    ok = (x > F(-2.0 ** 31)) & (x < F(2.0 ** 31))
    return np.where(ok, np.trunc(np.where(ok, x, 0)).astype(np.int64) & 0xFF, 0).astype(np.uint8)


def rgbd(rgb, depth, depth_trunc, mask=None):
    """rgb float32 [3, H, W], depth [1, H, W] or [H, W] -> (uint8 [H, W, 3], float32 [H, W])."""
    rgb = np.asarray(rgb, F)
    color = numpy_u8(np.transpose(rgb, (1, 2, 0)) * F(255))
    d = np.asarray(depth, F).reshape(rgb.shape[1:]).copy()
    if mask is not None:
        d[np.asarray(mask, F).reshape(d.shape) < F(0.5)] = 0
    with np.errstate(invalid="ignore"):
        d[d.astype(np.float64) >= float(depth_trunc)] = 0
    return color, d


def image_u8(img, scale=1.0, offset=0.0):
    """save_img_u8's conversion of img [3, H, W] * scale + offset -> uint8 [H, W, 3]."""
    x = np.transpose(np.asarray(img, F), (1, 2, 0)) * F(scale) + F(offset)
    return (np.clip(np.nan_to_num(x), F(0), F(1)) * F(255)).astype(np.uint8)


class Camera:
    def __init__(self, intrinsic, extrinsic, H, W, voxel_length, sdf_trunc):
        K = np.asarray(intrinsic, np.float64)
        E = np.asarray(extrinsic, np.float64)
        self.H, self.W = H, W
        self.fx, self.fy, self.cx, self.cy = F(K[0, 0]), F(K[1, 1]), F(K[0, 2]), F(K[1, 2])
        self.R = E[:3, :3].astype(F)
        self.t = E[:3, 3].astype(F)
        self.vs = F(voxel_length)
        self.trunc = F(sdf_trunc)


def touch(cam: Camera, depth):
    depth = np.asarray(depth, F).reshape(cam.H, cam.W)
    v, u = np.mgrid[0:cam.H:4, 0:cam.W:4]
    d = depth[v, u]
    with np.errstate(invalid="ignore"):
        ok = d > 0
    u, v, d = u[ok].astype(F), v[ok].astype(F), d[ok]
    q = [((u - cam.cx) * d) / cam.fx - cam.t[0], ((v - cam.cy) * d) / cam.fy - cam.t[1], d - cam.t[2]]
    p = [(cam.R[0, k] * q[0] + cam.R[1, k] * q[1]) + cam.R[2, k] * q[2] for k in range(3)]
    bs = F(cam.vs * F(T.RES))
    with np.errstate(invalid="ignore", over="ignore"):
        lo = np.stack([np.floor((pk - cam.trunc) / bs) for pk in p], 1)
        hi = np.stack([np.floor((pk + cam.trunc) / bs) for pk in p], 1)
        inr = np.all((lo >= T.KEY_LO) & (hi <= T.KEY_HI), axis=1)
    lo, hi = lo[inr].astype(np.int64), hi[inr].astype(np.int64)
    if len(lo) == 0:
        return np.zeros((0, 3), np.int32)
    ext = (hi - lo).max(0) + 1
    keys = []
    for dz in range(ext[2]):
        for dy in range(ext[1]):
            for dx in range(ext[0]):
                o = np.array([dx, dy, dz])
                m = np.all(lo + o <= hi, axis=1)
                keys.append(T.pack(lo[m] + o))
    return T.unpack(np.unique(np.concatenate(keys))).astype(np.int32)


def integrate(grid: dict, cam: Camera, units, depth, color_u8):
    depth = np.asarray(depth, F).reshape(cam.H, cam.W)
    color = np.asarray(color_u8, np.uint8).reshape(cam.H, cam.W, 3).astype(F)
    keys = np.unique(T.pack(units))
    for k in keys:
        if int(k) not in grid:
            grid[int(k)] = (np.zeros(T.BV, F), np.zeros(T.BV, F), np.zeros((T.BV, 3), F))
    if len(keys) == 0:
        return
    p = (T.grid_points(T.unpack(keys)).astype(F) + F(0.5)) * cam.vs
    R, t = cam.R, cam.t
    xc = ((R[0, 0] * p[..., 0] + R[0, 1] * p[..., 1]) + R[0, 2] * p[..., 2]) + t[0]
    yc = ((R[1, 0] * p[..., 0] + R[1, 1] * p[..., 1]) + R[1, 2] * p[..., 2]) + t[1]
    zc = ((R[2, 0] * p[..., 0] + R[2, 1] * p[..., 1]) + R[2, 2] * p[..., 2]) + t[2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = np.floor(((xc / zc) * cam.fx + cam.cx) + F(0.5))
        v = np.floor(((yc / zc) * cam.fy + cam.cy) + F(0.5))
        ok = (zc > 0) & (u >= 0) & (u < cam.W) & (v >= 0) & (v < cam.H)
    u, v = np.where(ok, u, 0), np.where(ok, v, 0)
    ui, vi = u.astype(np.int64), v.astype(np.int64)
    d = depth[vi, ui]
    xn, yn = (u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy
    with np.errstate(invalid="ignore", over="ignore"):
        sdf = (d - zc) * np.sqrt((F(1) + xn * xn) + yn * yn)
        ok &= (d > 0) & (sdf > -cam.trunc)
        obs = np.minimum(F(1), sdf / cam.trunc)
    col = color[vi, ui]
    for n, k in enumerate(keys):
        ts, w, c = grid[int(k)]
        m = ok[n]
        w1 = w[m] + F(1)
        ts[m] = (w[m] * ts[m] + obs[n][m]) / w1
        c[m] = (w[m][:, None] * c[m] + col[n][m]) / w1[:, None]
        w[m] = w1


def extract(grid: dict, voxel_length):
    """-> vertices, colours in [0, 1], triangles of ScalableTSDFVolume.extract_triangle_mesh."""
    v, c, t = T.extract(grid, voxel_length, 1.0)
    return v + F(0.5) * F(voxel_length), c / F(255), t
