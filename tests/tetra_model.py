"""numpy model of the tetrahedra extraction contract (include/rgs_b200.h, rgs_tetra_cull_* / marching / bisect / filter):
fp32, every operation rounded on its own in the header's order.  It is the second checker beside the fixtures that the
reference's own code made (tools/gen_golden_tetra.py)."""
from __future__ import annotations

import numpy as np

F = np.float32
CHUNK = 32 * 1024 * 1024

TRIANGLE_TABLE = np.array([
    [-1, -1, -1, -1, -1, -1], [1, 0, 2, -1, -1, -1], [4, 0, 3, -1, -1, -1], [1, 4, 2, 1, 3, 4], [3, 1, 5, -1, -1, -1], [2, 3, 0, 2, 5, 3],
    [1, 4, 0, 1, 5, 4], [4, 2, 5, -1, -1, -1], [4, 5, 2, -1, -1, -1], [4, 1, 0, 4, 5, 1], [3, 2, 0, 3, 5, 2], [1, 3, 5, -1, -1, -1],
    [4, 1, 2, 4, 3, 1], [3, 0, 4, -1, -1, -1], [2, 0, 1, -1, -1, -1], [-1, -1, -1, -1, -1, -1]], dtype=np.int64)
NUM_TRIANGLES = np.array([0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0], dtype=np.int64)
TET_EDGES = np.array([[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]], dtype=np.int64)


def cull_add(final, weight, alpha, coord, render7, gt_mask=None):
    """One view, in place on final f32 [N] and weight int32 [N]."""
    H, W = render7.shape
    x, y = coord[:, 0].astype(F), coord[:, 1].astype(F)
    gx = ((x * F(2)) + F(1)) / F(W - 1) - F(1)
    gy = ((y * F(2)) + F(1)) / F(H - 1) - F(1)
    ix = ((gx + F(1)) * F(W) - F(1)) * F(0.5)
    iy = ((gy + F(1)) * F(H) - F(1)) * F(0.5)
    x0, y0 = np.floor(ix), np.floor(iy)
    wx = ix - x0
    ex = F(1) - wx
    wy = iy - y0
    ey = F(1) - wy
    x1, y1 = x0 + F(1), y0 + F(1)
    img = render7.astype(F) if gt_mask is None else (render7.astype(F) * np.asarray(gt_mask, F).reshape(H, W))

    def m(xc, yc):
        with np.errstate(invalid="ignore"):
            ok = (xc >= 0) & (xc <= F(W - 1)) & (yc >= 0) & (yc <= F(H - 1))
        out = np.zeros(len(xc), F)
        out[ok] = img[yc[ok].astype(np.int64), xc[ok].astype(np.int64)]
        return out

    with np.errstate(invalid="ignore", over="ignore"):
        v = (ey * ex) * m(x0, y0)
        v = v + (ey * wx) * m(x1, y0)
        v = v + (wy * ex) * m(x0, y1)
        v = v + (wy * wx) * m(x1, y1)
        ok = v > F(0.5)
    a, f = alpha.astype(F), final
    mn = np.where(np.isnan(a), a, np.where(np.isnan(f), f, np.where(f < a, f, a)))
    final[ok] = mn[ok]
    weight[ok] += 1


def cull_finish(final, weight):
    return np.where(weight > 0, F(0.5) - final, F(-100)).astype(F)


def marching(points, sdf, scales, tets):
    """-> (ends f32 [M,2,3], end_sdf f32 [M,2,1], end_scales f32 [M,2,1], faces int64 [F,3], interp int64 [M,2])."""
    N, T = points.shape[0], tets.shape[0]
    tets = np.asarray(tets, np.int64)
    if T and (tets.min() < 0 or tets.max() >= N):
        raise ValueError("a tet index lies outside [0, N)")
    occ = sdf.reshape(-1) > 0
    occ4 = occ[tets] if T else np.zeros((0, 4), bool)
    s = occ4.sum(-1)
    valid = np.nonzero((s > 0) & (s < 4))[0]
    code = (occ4[valid] * (1 << np.arange(4))).sum(-1)
    edges = tets[valid][:, TET_EDGES.reshape(-1)].reshape(-1, 2)
    edges = np.sort(edges, axis=1)
    uniq, inv = np.unique(edges, axis=0, return_inverse=True) if len(edges) else (np.zeros((0, 2), np.int64), np.zeros(0, np.int64))
    inv = inv.reshape(-1)
    cross = occ[uniq[:, 0]] != occ[uniq[:, 1]] if len(uniq) else np.zeros(0, bool)
    mapping = np.full(len(uniq), -1, np.int64)
    mapping[cross] = np.arange(cross.sum())
    idx_map = mapping[inv].reshape(-1, 6)
    interp = uniq[cross]
    n_chunks = T // CHUNK + 1 if T > CHUNK else 1
    chunk_len = max(1, -(-T // n_chunks))
    ntri = NUM_TRIANGLES[code]
    group = 2 * (valid // chunk_len) + (ntri == 2)
    order = np.argsort(group, kind="stable")
    tri = TRIANGLE_TABLE[code[order]]
    ent = np.take_along_axis(idx_map[order], np.maximum(tri, 0), axis=1)
    faces = ent[np.arange(6)[None, :] < 3 * ntri[order][:, None]].reshape(-1, 3)
    sdf1 = sdf.reshape(-1).astype(F)
    sc = scales.reshape(-1).astype(F)
    return (points[interp.reshape(-1)].reshape(-1, 2, 3).astype(F), sdf1[interp.reshape(-1)].reshape(-1, 2, 1), sc[interp.reshape(-1)].reshape(-1, 2, 1),
            faces.astype(np.int64), interp.astype(np.int64))


def midpoints(left, right):
    return (left + right) * F(0.5)


def bisect(mid_sdf, left, right, left_sdf, right_sdf):
    """One step in place (left, right f32 [M,3], left_sdf, right_sdf f32 [M]); returns the next midpoints."""
    mid = midpoints(left, right)
    m = mid_sdf.reshape(-1).astype(F)
    low = ((m < 0) & (left_sdf < 0)) | ((m > 0) & (left_sdf > 0))
    left_sdf[low] = m[low]
    right_sdf[~low] = m[~low]
    left[low] = mid[low]
    right[~low] = mid[~low]
    return midpoints(left, right)


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c): the product is exact in fp64, the fp64 sum's error is recovered by TwoSum and
    decides the one case where rounding the fp64 sum to fp32 would round twice (an exact fp32 midpoint)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.astype(F)
    other = np.nextafter(r, np.where(s > r.astype(np.float64), F(np.inf), F(-np.inf)).astype(F))
    mid = (r.astype(np.float64) + other.astype(np.float64)) * 0.5
    fix = (s == mid) & (err != 0) & ((err > 0) == (other.astype(np.float64) > r.astype(np.float64)))
    return np.where(fix, other, r).astype(F)


def filter_mesh(points, ends, end_scales, faces):
    d = ends[:, 0].astype(F) - ends[:, 1].astype(F)
    dist = np.sqrt(fma32(d[:, 2], d[:, 2], fma32(d[:, 1], d[:, 1], d[:, 0] * d[:, 0])))
    es = end_scales.reshape(-1, 2).astype(F)
    keep = dist <= es[:, 0] + es[:, 1]
    new = np.cumsum(keep) - 1
    fk = keep[faces].all(axis=1) if len(faces) else np.zeros(0, bool)
    return points[keep].astype(F), new[faces[fk]].astype(np.int64).reshape(-1, 3)


def extract_mesh(points, scales, cells, evaluate_sdf, n_binary_steps=8, record=None):
    """The whole chain; ``record`` (a list) receives (mid points, mid sdf) per step."""
    sdf = evaluate_sdf(points)
    ends, end_sdf, end_scales, faces, _ = marching(points, sdf, scales, cells)
    if len(ends) == 0:
        return np.zeros((0, 3), F), np.zeros((0, 3), np.int64)
    left, right = ends[:, 0].copy(), ends[:, 1].copy()
    lsdf, rsdf = end_sdf[:, 0, 0].copy(), end_sdf[:, 1, 0].copy()
    mid = midpoints(left, right)
    for _ in range(n_binary_steps):
        msdf = evaluate_sdf(mid)
        if record is not None:
            record.append((mid.copy(), msdf.copy()))
        mid = bisect(msdf, left, right, lsdf, rsdf)
    return filter_mesh(mid, ends, end_scales, faces)
