"""An independent exact model of the Delaunay predicates and a validity checker for (points, cells).

Coordinates are fp32; every predicate first evaluates an fp64 determinant with a generous error bound and falls back to
exact arithmetic in Python integers (the fp32 values scaled by a common power of two) when the bound cannot decide.
Sign conventions are those of include/rgs_b200.h: orient3d = sign det[b - a, c - a, d - a]; insphere = -sign D5 with
D5 = det of the rows (x, y, z, x^2 + y^2 + z^2, 1), > 0 when e lies strictly inside the sphere of a positive a, b, c, d;
the perturbed insphere adds eps_i to the lifted coordinate of point i, eps of a lexicographically larger point infinitely
larger, and reads the sign off the 5 x 5 determinant's cofactors of the lifted column.
"""
from __future__ import annotations

from collections import defaultdict

import numpy as np

FILTER = 1e-12   # relative bound on the fp64 determinants (far above their actual rounding error)


def _ints(pts):
    """fp32 rows -> Python-integer rows, all scaled by one power of two."""
    fr = [[float(v).as_integer_ratio() for v in row] for row in np.asarray(pts, dtype=np.float32)]
    shift = max(d.bit_length() - 1 for row in fr for _, d in row)
    return [[n << (shift - (d.bit_length() - 1)) for n, d in row] for row in fr]


def _det(m):
    """Exact determinant of a square integer matrix (Bareiss)."""
    a = [list(r) for r in m]
    n, sign, prev = len(a), 1, 1
    for k in range(n - 1):
        if a[k][k] == 0:
            for r in range(k + 1, n):
                if a[r][k]:
                    a[k], a[r] = a[r], a[k]
                    sign = -sign
                    break
            else:
                return 0
        for i in range(k + 1, n):
            for j in range(k + 1, n):
                a[i][j] = (a[i][j] * a[k][k] - a[i][k] * a[k][j]) // prev
        prev = a[k][k]
    return sign * a[n - 1][n - 1]


def _sgn(v):
    return int(v > 0) - int(v < 0)


def orient3d(a, b, c, d):
    p = np.asarray([a, b, c, d], dtype=np.float32).astype(np.float64)
    m = p[1:] - p[0]
    det = np.linalg.det(m)
    perm = np.abs(m).prod(axis=1).sum() * 6 + np.prod(np.abs(m).max(axis=0)) * 6
    if abs(det) > FILTER * perm:
        return _sgn(det)
    q = _ints([a, b, c, d])
    return _sgn(_det([[q[i][k] - q[0][k] for k in range(3)] for i in (1, 2, 3)]))


def _lifted(q):
    return [[r[0], r[1], r[2], r[0] * r[0] + r[1] * r[1] + r[2] * r[2], 1] for r in q]


def insphere(a, b, c, d, e):
    p = np.asarray([a, b, c, d, e], dtype=np.float32).astype(np.float64)
    m = p[:4] - p[4]
    lm = np.concatenate([m, (m * m).sum(axis=1, keepdims=True)], axis=1)
    det = np.linalg.det(lm)
    scale = np.abs(m).max() ** 5 * 120 + 1e-300
    if abs(det) > FILTER * scale:
        return -_sgn(det)
    return -_sgn(_det(_lifted(_ints([a, b, c, d, e]))))


def _lex_key(p):
    return tuple(float(v) for v in np.asarray(p, dtype=np.float32))


def insphere_perturbed(a, b, c, d, e):
    s = insphere(a, b, c, d, e)
    if s:
        return s
    pts = [a, b, c, d, e]
    M = _lifted(_ints(pts))
    order = sorted(range(5), key=lambda i: _lex_key(pts[i]), reverse=True)
    for i in order:   # cofactor of (i, lifted column 3)
        minor = [[M[r][c] for c in range(5) if c != 3] for r in range(5) if r != i]
        cof = (-1) ** (i + 3) * _det(minor)
        if cof:
            return -_sgn(cof)
    return 0


# ---------------------------------------------------------------------------------------------------------------------

def _faces(cell):
    """The four faces of a cell as (sorted vertex triple, parity of the oriented face's permutation to sorted order)."""
    a, b, c, d = (int(v) for v in cell)
    out = []
    for f in ((b, c, d), (a, d, c), (a, b, d), (a, c, b)):   # outward-consistent orientation of each face
        s = sorted(f)
        perm = [f.index(v) for v in s]
        inv = sum(1 for i in range(3) for j in range(i + 1, 3) if perm[i] > perm[j])
        out.append((tuple(s), inv & 1))
    return out


def check(points, cells, lattice=False, hull_tolerance=1e-9):
    """Raise AssertionError unless `cells` is a valid Delaunay tetrahedralization of the distinct `points` (see the
    module docstring for the predicates).  Returns the number of interior faces checked."""
    P = np.asarray(points, dtype=np.float32)
    C = np.asarray(cells, dtype=np.int64).reshape(-1, 4)
    assert ((C >= 0) & (C < len(P))).all(), "index out of range"
    for t in C:
        assert orient3d(*P[t]) > 0, f"cell {t.tolist()} is not positive"
    owners = defaultdict(list)
    for ci, t in enumerate(C):
        for tri, par in _faces(t):
            owners[tri].append((ci, par))
    boundary_edges = defaultdict(int)
    interior = 0
    for tri, own in owners.items():
        assert len(own) <= 2, f"face {tri} lies in {len(own)} cells"
        if len(own) == 2:
            assert own[0][1] != own[1][1], f"face {tri} has the same orientation in both cells"
            (c0, _), (c1, _) = own
            e = [v for v in C[c1] if v not in tri][0]
            assert insphere_perturbed(*P[C[c0]], P[e]) < 0, f"face {tri} is not locally Delaunay"
            interior += 1
        else:
            for i in range(3):
                boundary_edges[tuple(sorted((tri[i], tri[(i + 1) % 3])))] += 1
    assert all(n % 2 == 0 for n in boundary_edges.values()), "the boundary is not a closed surface"
    if len(C):
        # full-dimensional: every distinct point is a vertex
        assert _distinct_reps(P) <= set(np.unique(C).tolist()), "a distinct point is not a vertex"
        vol = _volume(P, C)
        from scipy.spatial import ConvexHull
        hull = ConvexHull(P.astype(np.float64)).volume
        if lattice:
            assert vol == hull, (vol, hull)
        else:
            assert vol <= hull * (1 + hull_tolerance) and vol >= hull * (1 - 1e-6), (vol, hull)
    return interior


def _distinct_reps(P):
    seen = {}
    for i, p in enumerate(P.tolist()):
        seen.setdefault(tuple(v + 0.0 for v in p), i)
    return set(seen.values())


def _volume(P, C):
    p = P.astype(np.float64)[C]
    return float(np.abs(np.linalg.det(p[:, 1:] - p[:, :1])).sum() / 6.0)


def reorient(points, cells):
    """scipy's cells with every negative one flipped (its orientation is mixed)."""
    P = np.asarray(points, dtype=np.float64)
    C = np.asarray(cells, dtype=np.int64).copy()
    neg = np.linalg.det(P[C[:, 1:]] - P[C[:, :1]]) < 0
    C[neg, 2], C[neg, 3] = C[neg, 3].copy(), C[neg, 2].copy()
    return C


def ghosts(points):
    """The four ghost vertices of include/rgs_b200.h: fl32(c + 2^30 R s), c the box centre, R the smallest power of two
    >= the box's largest side (at least 2^-100)."""
    import math
    P = np.asarray(points, dtype=np.float32).astype(np.float64)
    lo, hi = P.min(axis=0), P.max(axis=0)
    ext = float((hi - lo).max())
    m, e = math.frexp(ext)
    R = max(ext if m == 0.5 else math.ldexp(1.0, e), 2.0 ** -100)
    c = 0.5 * (lo + hi)
    S = 2.0 ** 30 * R
    signs = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], dtype=np.float64)
    return (c + S * signs).astype(np.float32)


def check_gpu(points, cells, rel=1e-11):
    """The checker at scale, on the cells' CUDA device: every cell positive and every interior face locally Delaunay,
    decided in torch fp64 where |det| exceeds `rel` times a bound on its terms and by the exact model above elsewhere;
    no face in three cells.  Returns the counts (all violations must be 0)."""
    import torch
    p = points.double()
    c = cells.long()
    v = p[c]
    d = v[:, 1:] - v[:, :1]
    o = torch.linalg.det(d)
    so = d.abs().amax(dim=(1, 2)) ** 3 * 6
    amb = (o.abs() <= rel * so).nonzero().flatten().tolist()
    bad = int((o < -rel * so).sum())
    P = points.cpu().numpy()
    C = cells.cpu().numpy()
    bad += sum(orient3d(*P[C[i]]) <= 0 for i in amb)
    f = torch.stack([c[:, [1, 2, 3]], c[:, [0, 2, 3]], c[:, [0, 1, 3]], c[:, [0, 1, 2]]], 1).reshape(-1, 3).sort(dim=1).values
    opp = c.reshape(-1)
    order = torch.argsort(f[:, 2], stable=True)
    order = order[torch.argsort(f[order, 1], stable=True)]
    order = order[torch.argsort(f[order, 0], stable=True)]
    fs = f[order]
    same = (fs[1:] == fs[:-1]).all(dim=1)
    triple = bool((same[1:] & same[:-1]).any())
    i = same.nonzero().flatten()
    bad_faces, n_amb5 = 0, 0
    for lo in range(0, len(i), 1 << 22):        # in chunks: the lifted 4 x 4 systems of 9 M points do not fit at once
        j = i[lo:lo + (1 << 22)]
        a, b = order[j], order[j + 1]
        ca, e = c[a // 4], opp[b]
        q = torch.cat([p[ca], p[e][:, None]], 1)
        m = q[:, :4] - q[:, 4:]
        d5 = torch.linalg.det(torch.cat([m, (m * m).sum(-1, keepdim=True)], -1))
        s5 = m.abs().amax(dim=(1, 2)) ** 5 * 120
        amb5 = (d5.abs() <= rel * s5).nonzero().flatten()
        bad_faces += int((d5 < -rel * s5).sum())     # -D5 > 0: the opposite vertex lies inside
        Ca, E = ca[amb5].cpu().numpy(), e[amb5].cpu().numpy()
        bad_faces += sum(insphere_perturbed(*P[Ca[k]], P[E[k]]) >= 0 for k in range(len(E)))
        n_amb5 += len(E)
    return {"negative_cells": bad, "faces_in_three_cells": triple, "non_delaunay_faces": bad_faces, "interior_faces": int(len(i)),
            "exact_cells": len(amb), "exact_faces": n_amb5}
