"""fp64 model of the 3D smoothing filter (csrc/rgs_activation.cu, filter3d_distance/finish_kernel), with every (point, camera)
decision classified against its fp32 bound (tests/f32_error.py).

The operation is GaussianModel.compute_3D_filter (scene/gaussian_model.py:179-232), written from the math: for every camera,
p_cam = xyz R + T; the camera is valid for the point when z > 0.2 and the projection (x / z f_x + W / 2, y / z f_y + H / 2)
lies within the image widened by 15 % on each side; distance = the smallest valid z (z clamped to 0.001 first), the
largest distance over the seen points for a point no camera sees; filter = distance / max f_x * sqrt(0.2).

A decision (`z > 0.2` or one of the four screen comparisons) whose fp32 value lies within its bound of the threshold is
*ambiguous*: the camera is then possibly but not surely valid.  Every point gets an interval for its distance:
  * surely seen (some camera surely valid): [min over the possibly valid cameras of z - e, min over the surely valid of z + e];
  * surely unseen (no camera possibly valid): the interval of the largest distance over the seen points;
  * otherwise the hull of both.
With no ambiguous decision the interval is the fp64 minimum (or maximum) within its bound.  The filter multiplies by the
fp32 1 / focal and sqrt(0.2): two more roundings on both ends.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from f32_error import ETA, R, U, f32

CAM_BLOCK = 64   # cameras evaluated at once


def camera_table(cameras):
    """The [n, 16] fp32 table fused.compute_3D_filter builds (R row-major, T, focal_x, focal_y, W, H) and max focal_x."""
    rows, focal = [], 0.0
    for cam in cameras:
        W, H = cam.image_width, cam.image_height
        fx, fy = W / (2 * math.tan(cam.FoVx / 2.)), H / (2 * math.tan(cam.FoVy / 2.))
        rows.append(np.concatenate([np.asarray(cam.R, np.float32).reshape(9), np.asarray(cam.T, np.float32).reshape(3),
                                    np.asarray([fx, fy, W, H], np.float32)]))
        focal = max(focal, fx)
    return np.stack(rows), focal


def _decide(val: R, thr, above: bool):
    """(surely, possibly) for `val > thr` / `val >= thr` (above) or `val <= thr`."""
    d = val.v - thr if above else thr - val.v
    return d > val.e, d >= -val.e


def distance_intervals(xyz, table, device="cpu") -> dict:
    """Per point: lo, hi of its distance, and `ambiguous` (some decision of the point is ambiguous)."""
    pts = torch.as_tensor(xyz, dtype=torch.float32).to(device)
    cams = torch.as_tensor(table, dtype=torch.float32).to(device)
    P = pts.shape[0]
    x, y, z = (R.input(pts[:, k:k + 1]) for k in range(3))
    inf = torch.full((P,), float("inf"), dtype=torch.float64, device=device)
    p_lo, s_hi, p_max = inf.clone(), inf.clone(), torch.full_like(inf, -float("inf"))
    any_sure = torch.zeros(P, dtype=torch.bool, device=device)
    any_poss = torch.zeros_like(any_sure)
    amb = torch.zeros_like(any_sure)
    for b in range(0, cams.shape[0], CAM_BLOCK):
        C = cams[b:b + CAM_BLOCK].double()[None]          # [1, n, 16]
        c = lambda k: R(C[..., k].expand(P, -1))
        xc, yc, zc = (z.fma(c(6 + j), y.fma(c(3 + j), x * c(j))) + c(9 + j) for j in range(3))   # xyz @ R + T
        ds, dp = _decide(zc, f32(0.2), True)
        zz = zc.maximum(f32(0.001))
        Wc, Hc = C[..., 14], C[..., 15]
        px = (xc / zz) * c(12) + R((Wc * 0.5).expand(P, -1))
        py = (yc / zz) * c(13) + R((Hc * 0.5).expand(P, -1))
        sure, poss = ds, dp
        for val, thr, above in ((px, -0.15 * Wc, True), (px, Wc * 1.15, False), (py, -0.15 * Hc, True), (py, 1.15 * Hc, False)):
            s, p = _decide(val, thr.float().double(), above)
            sure, poss = sure & s, poss & p
        amb |= (poss & ~sure).any(1)
        lo, hi = zz.v - zz.e, zz.v + zz.e
        p_lo = torch.minimum(p_lo, torch.where(poss, lo, inf[:, None]).amin(1))
        s_hi = torch.minimum(s_hi, torch.where(sure, hi, inf[:, None]).amin(1))
        p_max = torch.maximum(p_max, torch.where(poss, hi, -inf[:, None]).amax(1))
        any_sure |= sure.any(1)
        any_poss |= poss.any(1)
    seen_hi = torch.minimum(s_hi, p_max)
    m_lo = torch.where(any_sure, p_lo, -inf).max()
    m_hi = torch.where(any_poss, seen_hi, -inf).max()
    lo = torch.where(any_sure, p_lo, torch.where(any_poss, torch.minimum(p_lo, m_lo), m_lo))
    hi = torch.where(any_sure, s_hi, torch.where(any_poss, torch.maximum(seen_hi, m_hi), m_hi))
    return {"lo": lo, "hi": hi, "ambiguous": amb, "surely_seen": any_sure, "possibly_seen": any_poss}


def filter_intervals(xyz, cameras, device="cpu"):
    """(lo, hi) of filter_3D per point and the distance intervals."""
    table, focal = camera_table(cameras)
    d = distance_intervals(xyz, table, device)
    inv = float(np.float32(1.0) / np.float32(focal))
    k = inv * f32(0.4472135954999579)
    lo = d["lo"] * k * (1 - 2.01 * U) - 2 * ETA
    hi = d["hi"] * k * (1 + 2.01 * U) + 2 * ETA
    return lo, hi, d
