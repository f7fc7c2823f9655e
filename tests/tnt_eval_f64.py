"""numpy fp64 restatement of the Tanks and Temples evaluation contract (include/rgs_b200.h, rgs_tnt_*, and the host steps
of rade_gs_b200.tnt_eval): transform, polygon crop, voxel downsample, nearest distances, ICP moments, Umeyama, the ICP
loop, the seeded RANSAC, the histogram and the F-score.  Needs no GPU and no package."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

MAX_POINT_NUMBER = 4e6


def transform(T, p):
    p = np.asarray(p, np.float64)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def crop_mask(p, axis, axis_min, axis_max, polygon):
    """Inclusive axis range, then the crossing-number test with half-open edges and crossings strictly below u."""
    p = np.asarray(p, np.float64)
    uv = [a for a in range(3) if a != axis]
    w, pu, pv = p[:, axis], p[:, uv[0]], p[:, uv[1]]
    poly = np.asarray(polygon, np.float64).reshape(-1, 2)
    count = np.zeros(len(p), np.int64)
    with np.errstate(all="ignore"):
        for k in range(len(poly)):
            (au, av), (bu, bv) = poly[k], poly[(k + 1) % len(poly)]
            cond = ((av < pv) & (pv <= bv)) | ((bv < pv) & (pv <= av))
            xu = au + ((pv - av) * (bu - au)) / (bv - av)
            count += cond & (xu < pu)
    return (w >= axis_min) & (w <= axis_max) & (count % 2 == 1)


def crop(p, volume, T=None):
    """(cropped in input order, kept mask); volume = (axis, axis_min, axis_max, polygon [K, 2]) or None."""
    q = transform(T, p) if T is not None else np.asarray(p, np.float64).copy()
    if volume is None:
        return q, np.ones(len(q), bool)
    keep = crop_mask(q, *volume)
    return q[keep], keep


def voxel_down_sample(p, voxel):
    """(means [V, 3] in ascending key order, counts [V]): origin = min - voxel * 0.5, index floor((p - origin) / voxel),
    means = the sequential sum from 0.0 in input order divided by the count."""
    p = np.asarray(p, np.float64)
    if len(p) == 0:
        return np.zeros((0, 3)), np.zeros(0, np.int64)
    origin = p.min(axis=0) - voxel * 0.5
    idx = np.floor((p - origin) / voxel).astype(np.int64)
    if idx.max() >= 1 << 21:
        raise ValueError("more than 2^21 voxels along an axis")
    key = idx[:, 0] << 42 | idx[:, 1] << 21 | idx[:, 2]
    order = np.argsort(key, kind="stable")
    sk = key[order]
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    counts = np.diff(np.r_[starts, len(p)])
    sums = np.zeros((len(starts), 3))
    for k in range(int(counts.max())):
        live = counts > k
        sums[live] = sums[live] + p[order[starts[live] + k]]
    return sums / counts[:, None].astype(np.float64), counts


def uniform_for_registration(p):
    n = len(p)
    return p[::int(round(n / float(MAX_POINT_NUMBER)))] if n > MAX_POINT_NUMBER else p


def dist2(a, b):
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest(reference, query, k=8):
    """(distance, index): the exact minimum of sqrt(d2) over the reference, searched among a kd-tree's k nearest."""
    ref, q = np.asarray(reference, np.float64), np.asarray(query, np.float64)
    if len(q) == 0:
        return np.zeros(0), np.zeros(0, np.int64)
    k = min(k, len(ref))
    _, cand = cKDTree(ref).query(q, k=k)
    cand = cand.reshape(len(q), k)
    d2 = dist2(q[:, None, :], ref[cand])
    j = d2.argmin(axis=1)
    return np.sqrt(d2[np.arange(len(q)), j]), cand[np.arange(len(q)), j]


def moments(src, tgt, dist, index, threshold):
    """The header's 18 moments (summation order free: compared to 1e-12)."""
    c = dist < threshold
    n = int(c.sum())
    m = np.zeros(18)
    if n == 0:
        return m
    s, t = src[c], tgt[index[c]]
    inv = 1.0 / n
    m[0], m[1] = n, dist2(s, t).sum()
    ms, mt = s.sum(axis=0) * inv, t.sum(axis=0) * inv
    sc, tc = s - ms, t - mt
    m[2:5], m[5:8] = ms, mt
    m[8:17] = (inv * (tc.T @ sc)).reshape(-1)
    m[17] = inv * ((sc[:, 0] ** 2 + sc[:, 1] ** 2) + sc[:, 2] ** 2).sum()
    return m


def umeyama(m):
    T = np.eye(4)
    if m[0] == 0:
        return T
    U, D, Vt = np.linalg.svd(m[8:17].reshape(3, 3))
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    c = (1.0 / m[17]) * D.dot(S)
    T[:3, 3] = m[5:8] - (c * R) @ m[2:5]
    T[:3, :3] = c * R
    return T


def icp(source, target, threshold, max_iteration=20, rel_fitness=1e-6, rel_rmse=1e-6):
    """Open3D's loop: (T, fitness, rmse, iterations, per-iteration transforms, per-evaluation correspondence counts)."""
    src = np.asarray(source, np.float64).copy()
    tgt = np.asarray(target, np.float64)

    def evaluate(s):
        d, idx = nearest(tgt, s)
        m = moments(s, tgt, d, idx, threshold)
        return m, (m[0] / len(s) if len(s) else 0.0), (float(np.sqrt(m[1] / m[0])) if m[0] else 0.0)

    T = np.eye(4)
    m, fit, rmse = evaluate(src)
    hist, counts, it = [], [int(m[0])], 0
    for it in range(1, max_iteration + 1):
        up = umeyama(m)
        T = up @ T
        hist.append(T.copy())
        src = transform(up, src)
        prev = (fit, rmse)
        m, fit, rmse = evaluate(src)
        counts.append(int(m[0]))
        if abs(prev[0] - fit) < rel_fitness and abs(prev[1] - rmse) < rel_rmse:
            break
    return T, fit, rmse, it, hist, counts


def ransac_hypotheses(n, count, ransac_n, seed):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, n, (count, ransac_n))
    while True:
        s = np.sort(idx, axis=1)
        dup = (s[:, 1:] == s[:, :-1]).any(axis=1)
        if not dup.any():
            return idx
        idx[dup] = rng.integers(0, n, (int(dup.sum()), ransac_n))


def ransac(src, dst, seed, iterations=100000, max_distance=0.2, ransac_n=6):
    """Seeded RANSAC over correspondences i <-> i: (T, inlier count, inlier rmse, winning hypothesis)."""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    hyp = ransac_hypotheses(len(src), iterations, ransac_n, seed)
    S, D = src[hyp], dst[hyp]
    inv = 1.0 / ransac_n
    ms, md = S.sum(axis=1) * inv, D.sum(axis=1) * inv
    sc, dc = S - ms[:, None], D - md[:, None]
    var = (sc * sc).sum(axis=(1, 2)) * inv
    U, Dv, Vt = np.linalg.svd(inv * np.einsum("bki,bkj->bij", dc, sc))
    sgn = np.ones((len(hyp), 3))
    sgn[np.linalg.det(U) * np.linalg.det(Vt) < 0, 2] = -1.0
    R = U @ (sgn[:, :, None] * Vt)
    best = (-1, np.inf, -1, np.eye(4))
    with np.errstate(all="ignore"):
        c = (1.0 / var) * (Dv * sgn).sum(axis=1)
        cR = c[:, None, None] * R
        t = md - np.einsum("bij,bj->bi", cR, ms)
        for b in range(0, len(hyp), 4096):
            moved = np.einsum("bij,nj->bni", cR[b:b + 4096], src) + t[b:b + 4096, None]
            d2 = ((moved - dst[None]) ** 2).sum(axis=2)
            inl = np.sqrt(d2) < max_distance
            cnt = inl.sum(axis=1)
            rmse = np.sqrt(np.where(inl, d2, 0.0).sum(axis=1) / np.maximum(cnt, 1))
            for k in range(len(cnt)):
                if cnt[k] > best[0] or (cnt[k] == best[0] and rmse[k] < best[1]):
                    T = np.eye(4)
                    T[:3, :3], T[:3, 3] = cR[b + k], t[b + k]
                    best = (int(cnt[k]), float(rmse[k]), b + k, T)
    if best[0] <= 0:
        return np.eye(4), 0, 0.0, -1
    return best[3], best[0], best[1], best[2]


def f_score_histo(d1, d2, tau, plot_stretch=5):
    """get_f1_score_histo2 (F = 0 when precision and recall are both 0)."""
    if not (len(d1) and len(d2)):
        z = np.array([0])
        return 0, 0, 0, z, z, z, z
    recall = float(sum(d < tau for d in d2)) / float(len(d2))
    precision = float(sum(d < tau for d in d1)) / float(len(d1))
    fscore = 2 * recall * precision / (recall + precision) if recall + precision > 0 else 0.0
    bins = np.arange(0, tau * plot_stretch, tau / 100)
    h1, e1 = np.histogram(d1, bins)
    h2, e2 = np.histogram(d2, bins)
    return precision, recall, fscore, e1, np.cumsum(h1).astype(float) / len(d1), e2, np.cumsum(h2).astype(float) / len(d2)


def evaluate(source, gt, volume, gt_trans, traj, gt_traj, tau, seed, ransac_iterations=100000, max_iteration=20):
    """run.py's pipeline: a dict with the alignment, each stage's (T, fitness, rmse, iterations) and the scores."""
    n = len(gt_traj)
    T0 = ransac(np.asarray(traj)[:n, :3, 3], transform(gt_trans, np.asarray(gt_traj)[:, :3, 3]), seed, ransac_iterations)[0]
    gt_crop = crop(gt, volume)[0]
    stages, T = [], T0
    for voxel, thr in ((tau, 80 * tau), (tau / 2.0, 20 * tau), (None, 2 * tau)):
        s = crop(source, volume, T)[0]
        if voxel is None:
            s, t = uniform_for_registration(s), uniform_for_registration(gt_crop)
        else:
            s, t = voxel_down_sample(s, voxel)[0], voxel_down_sample(gt_crop, voxel)[0]
        Ti, fit, rmse, it, hist, counts = icp(s, t, thr, max_iteration)
        T = Ti @ T
        stages.append(dict(T=T, fitness=fit, rmse=rmse, iterations=it, history=hist, counts=counts))
    s = voxel_down_sample(crop(source, volume, T)[0], tau / 2.0)[0]
    t = voxel_down_sample(gt_crop, tau / 2.0)[0]
    d1, d2 = nearest(t, s)[0], nearest(s, t)[0]
    p, r, f, e1, c1, e2, c2 = f_score_histo(d1, d2, tau)
    return dict(alignment=T0, stages=stages, T=T, precision=p, recall=r, fscore=f, d1=d1, d2=d2, edges=e1, cum_source=c1, cum_target=c2, source=s,
                target=t)
