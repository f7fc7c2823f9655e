"""numpy fp64 restatement of the DTU evaluation contract (include/rgs_b200.h, rgs_dtu_*): surface sampling, the sequential
greedy radius downsample, masking and statistics, brute-force nearest neighbours and the mask cull."""
from __future__ import annotations

import numpy as np
from scipy import ndimage
from scipy.spatial import cKDTree


def sample(vertices, faces, density):
    v = np.asarray(vertices, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    out = [v]
    with np.errstate(all="ignore"):
        for a, b, c in f:
            e1, e2 = v[b] - v[a], v[c] - v[a]
            l1 = np.sqrt((e1[0] * e1[0] + e1[1] * e1[1]) + e1[2] * e1[2])
            l2 = np.sqrt((e2[0] * e2[0] + e2[1] * e2[1]) + e2[2] * e2[2])
            cr = np.array([e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]])
            area2 = np.sqrt((cr[0] * cr[0] + cr[1] * cr[1]) + cr[2] * cr[2])
            if not area2 > 0:
                continue
            thr = density * np.sqrt((l1 * l2) / area2)
            n1, n2 = np.floor(l1 / thr), np.floor(l2 / thr)
            c0 = (np.arange(int(n1) + 1, dtype=np.float64) + 0.5) / max(n1, 1e-7)
            c1 = (np.arange(int(n2) + 1, dtype=np.float64) + 0.5) / max(n2, 1e-7)
            C0, C1 = np.meshgrid(c0, c1, indexing="ij")
            ok = (C0 + C1) < 1
            k0, k1 = C0[ok][:, None], C1[ok][:, None]
            out.append((e1[None] * k0 + e2[None] * k1) + v[a][None])
    return np.concatenate(out, 0)


def dist2(a, b):
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def greedy_downsample(points, r):
    """kept mask of the greedy maximal independent set in index order (eval.py:86-94), neighbours with d2 <= r * r."""
    p = np.asarray(points, np.float64)
    r2 = r * r
    tree = cKDTree(p)
    kept = np.ones(len(p), bool)
    for i, cand in enumerate(tree.query_ball_point(p, r * (1 + 1e-9))):
        if kept[i]:
            cand = np.asarray(cand, np.int64)
            nb = cand[dist2(p[cand], p[i]) <= r2]
            kept[nb] = False
            kept[i] = True
    return kept


def nearest(reference, query, chunk=2048):
    ref = np.asarray(reference, np.float64)
    q = np.asarray(query, np.float64)
    out = np.empty(len(q))
    for s in range(0, len(q), chunk):
        out[s:s + chunk] = np.sqrt(dist2(q[s:s + chunk, None, :], ref[None, :, :]).min(axis=1))
    return out


def mask_and_score(down, stl, obs_mask, bb, res, plane, patch, max_dist):
    """eval.py:96-134 on the downsampled data: (in-ObsMask indices into down, dist_d2s, dist_s2d, mean_d2s, mean_s2d)."""
    BB = np.asarray(bb).astype(np.float32)
    inbound = ((down >= BB[:1] - patch) & (down < BB[1:] + patch * 2)).sum(axis=-1) == 3
    data_in = down[inbound]
    grid = np.around((data_in - BB[:1]) / res).astype(np.int32)
    gin = ((grid >= 0) & (grid < np.expand_dims(obs_mask.shape, 0))).sum(axis=-1) == 3
    g = grid[gin]
    in_obs = obs_mask[g[:, 0], g[:, 1], g[:, 2]].astype(bool)
    idx = np.where(inbound)[0][gin][in_obs]
    d2s = nearest(stl, down[idx])
    P = np.asarray(plane, np.float64).reshape(4)
    above = (((P[0] * stl[:, 0] + P[1] * stl[:, 1]) + P[2] * stl[:, 2]) + P[3]) > 0
    s2d = nearest(data_in, stl[above])
    with np.errstate(all="ignore"):
        return idx, d2s, s2d, d2s[d2s < max_dist].mean(), s2d[s2d < max_dist].mean()


DISK6 = (np.add.outer(np.arange(-6, 7) ** 2, np.arange(-6, 7) ** 2) <= 36).astype(np.uint8)


def dilate(mask):
    return ndimage.binary_dilation(np.asarray(mask) > 0, structure=DISK6, border_value=0)


def cull_pixels(vertices, proj, W, H):
    """Per view the fp64 quantities of the contract: (gx, gy, column, row) arrays [n_views, V]."""
    v = np.asarray(vertices, np.float64)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    out = []
    for P in proj:
        c = [((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] for r in range(3)]
        zz = c[2] + 1e-6
        with np.errstate(all="ignore"):
            gx = (c[0] / zz / (W - 1) - 0.5) * 2
            gy = (c[1] / zz / (H - 1) - 0.5) * 2
            out.append((gx, gy, ((gx + 1) / 2) * (W - 1), ((gy + 1) / 2) * (H - 1)))
    return out


def cull_keep(vertices, proj, dilated):
    n, H, W = dilated.shape
    keep = np.ones(len(vertices), bool)
    for k, (gx, gy, u, v) in enumerate(cull_pixels(vertices, proj, W, H)):
        valid = (gx > -1) & (gx < 1) & (gy > -1) & (gy < 1)
        ui = np.where(valid, np.rint(np.where(valid, u, 0)), 0).astype(np.int64)
        vi = np.where(valid, np.rint(np.where(valid, v, 0)), 0).astype(np.int64)
        keep &= ~valid | dilated[k][vi, ui].astype(bool)
    return keep


def cull_near_boundary(vertices, proj, W, H, tol=1e-3):
    """Vertices whose fp64 projection lies within `tol` pixels of a rounding (x.5) or validity (0, W-1) boundary in some view."""
    near = np.zeros(len(vertices), bool)
    for gx, gy, u, v in cull_pixels(vertices, proj, W, H):
        for t, S in ((u, W), (v, H)):
            with np.errstate(invalid="ignore"):
                near |= (np.abs(t - np.floor(t) - 0.5) < tol) | (np.abs(t) < tol) | (np.abs(t - (S - 1)) < tol) | ~np.isfinite(t)
    return near
