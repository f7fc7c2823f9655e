"""numpy restatement of the unbounded-scene mesh stages (contract at rgs_unbounded_* in include/rgs_b200.h): fp32 arrays,
so every operation is one IEEE fp32 operation rounded on its own, in the order the contract writes it; vertex positions
in fp64.  The GPU kernels must reproduce every output bit for bit.  The triangle table is re-derived here from the face
rule of rgs_tsdf_extract, independently of the compile-time derivation in csrc/rgs_mcubes.cuh."""
from __future__ import annotations

import numpy as np

f32 = np.float32
ONE, TWO = f32(1.0), f32(2.0)


def norm3(p: np.ndarray) -> np.ndarray:
    p = p.astype(np.float32)
    return np.sqrt((p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1]) + p[..., 2] * p[..., 2])


def _scale_rows(s: np.ndarray, p: np.ndarray, m: np.ndarray) -> np.ndarray:
    return s[..., None] * (p / m[..., None])


def contract(p: np.ndarray, center=(0.0, 0.0, 0.0), radius=1.0) -> np.ndarray:
    c, r = np.asarray(center, np.float32), f32(radius)
    with np.errstate(all="ignore"):
        q = (p.astype(np.float32) - c) / r
        m = norm3(q)
        out = _scale_rows(TWO - ONE / m, q, m)
    return np.where((m < 1)[..., None], q, out).astype(np.float32)


def uncontract(y: np.ndarray) -> np.ndarray:
    y = y.astype(np.float32)
    with np.errstate(all="ignore"):
        m = norm3(y)
        out = _scale_rows(ONE / (TWO - m), y, m)
    return np.where((m < 1)[..., None], y, out).astype(np.float32)


def inv_contraction(y: np.ndarray, center, radius, max_range=32.0) -> np.ndarray:
    c, r, mr = np.asarray(center, np.float32), f32(radius), f32(max_range)
    with np.errstate(all="ignore"):
        w = uncontract(y) * r + c
    return np.where(w > mr, mr, np.where(w < -mr, -mr, w)).astype(np.float32)


def project(p: np.ndarray, M: np.ndarray):
    """(u, v, w, in view) of points p [N, 3] under the row-major 4x4 M."""
    M = M.astype(np.float32)
    with np.errstate(all="ignore"):
        h = [((p[:, 0] * M[0, j] + p[:, 1] * M[1, j]) + p[:, 2] * M[2, j]) + M[3, j] for j in range(4)]
        w = h[3]
        u, v = h[0] / w, h[1] / w
    ok = (u > -1) & (u < 1) & (v > -1) & (v < 1) & (w > 0)
    return u, v, w, ok


def bilinear(u: np.ndarray, v: np.ndarray, W: int, H: int):
    """(flat offsets [4, N], weights [4, N], in-image [4, N]) of grid_sample(bilinear, border, align_corners=True)."""
    with np.errstate(all="ignore"):
        ix = ((u + ONE) / TWO) * f32(W - 1)
        iy = ((v + ONE) / TWO) * f32(H - 1)
    ix = np.minimum(f32(W - 1), np.maximum(ix, f32(0)))
    iy = np.minimum(f32(H - 1), np.maximum(iy, f32(0)))
    ix = np.nan_to_num(ix)   # only masked samples can be NaN; keep the gather in range
    iy = np.nan_to_num(iy)
    x0, y0 = np.floor(ix), np.floor(iy)
    x1, y1 = x0 + ONE, y0 + ONE
    wt = [(x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)]
    xi, yi = x0.astype(np.int64), y0.astype(np.int64)
    offs, ins = [], []
    for q in range(4):
        x, y = xi + (q & 1), yi + (q >> 1)
        ins.append((x < W) & (y < H))
        offs.append(np.where(ins[-1], y * W + x, 0))
    return np.array(offs), np.array(wt, dtype=np.float32), np.array(ins)


def sample(img: np.ndarray, b) -> np.ndarray:
    offs, wt, ins = b
    flat = img.reshape(-1).astype(np.float32)
    acc = np.zeros(offs.shape[1], np.float32)
    for q in range(4):
        acc = np.where(ins[q], acc + flat[offs[q]] * wt[q], acc)
    return acc


def sdf(xs, ys, zs, proj, depth, center, radius, trunc0) -> np.ndarray:
    """The n^3 crop (rgs_unbounded_sdf), [n, n, n]."""
    xs, ys, zs = (np.asarray(a, np.float32) for a in (xs, ys, zs))
    s = np.stack(np.meshgrid(xs, ys, zs, indexing="ij"), -1).reshape(-1, 3)
    return sdf_points(s, proj, depth, center, radius, trunc0).reshape(len(xs), len(ys), len(zs))


def sdf_points(s, proj, depth, center, radius, trunc0) -> np.ndarray:
    """The same at arbitrary contracted samples s [N, 3] (fp32)."""
    s = np.asarray(s, np.float32)
    c, r, t0 = np.asarray(center, np.float32), f32(radius), f32(trunc0)
    with np.errstate(all="ignore"):
        p = uncontract(s) * r + c
        pm = norm3(p)
        trunc = np.where(pm > 1, t0 * (ONE / (TWO - np.where(pm > f32(1.9), f32(1.9), pm))), t0).astype(np.float32)
    t = np.ones(len(p), np.float32)
    w = np.ones(len(p), np.float32)
    V, H, W = depth.shape
    for v in range(V):
        u, vv, h, ok = project(p, proj[v])
        d = sample(depth[v], bilinear(u, vv, W, H))
        with np.errstate(all="ignore"):
            sd = d - h
            ok &= sd > -trunc
            cl = np.minimum(np.maximum(sd / trunc, f32(-1)), ONE)
            tn = (t * w + cl) / (w + ONE)
        t = np.where(ok, tn, t)
        w = np.where(ok, w + ONE, w)
    return t


def colors(points, proj, depth, rgb, trunc) -> np.ndarray:
    p = np.asarray(points, np.float32)
    col = np.zeros((len(p), 3), np.float32)
    w = np.ones(len(p), np.float32)
    tr = f32(trunc)
    V, H, W = depth.shape
    for v in range(V):
        u, vv, h, ok = project(p, proj[v])
        b = bilinear(u, vv, W, H)
        with np.errstate(all="ignore"):
            ok &= (sample(depth[v], b) - h) > -tr
        wp = w + ONE
        for k in range(3):
            col[:, k] = np.where(ok, (col[:, k] * w + sample(rgb[v, k], b)) / wp, col[:, k])
        w = np.where(ok, wp, w)
    return col


# ---- marching cubes ---------------------------------------------------------------------------------------------------

def _other_axis(a, k):
    return (1 if a == 0 else 0) if k == 0 else (1 if a == 2 else 2)


def _edge_corner(e, hi):
    a, o = e // 4, e % 4
    p = [0, 0, 0]
    p[_other_axis(a, 0)] = o & 1
    p[_other_axis(a, 1)] = o >> 1 & 1
    p[a] = hi
    return p[0] + 2 * p[1] + 4 * p[2]


def _bit(c, k):
    return c >> k & 1


def tri_table() -> list[list[int]]:
    """Per case the edge triples: face segments directed so that (segment x outward face normal) points to the inside
    corner of the first edge, loops walked from their lowest edge and fanned."""
    table = []
    for cs in range(256):
        inside = [(cs >> c) & 1 for c in range(8)]
        change = [inside[_edge_corner(e, 0)] != inside[_edge_corner(e, 1)] for e in range(12)]
        succ = {}
        for a in range(3):
            for s in range(2):
                fe = [e for e in range(12) if e // 4 != a and _bit(_edge_corner(e, 0), a) == s]
                ch = [e for e in fe if change[e]]
                if len(ch) == 2:
                    segs = [ch]
                elif len(ch) == 4:
                    segs = [[e for e in fe if c in (_edge_corner(e, 0), _edge_corner(e, 1))] for c in range(8) if _bit(c, a) == s and inside[c]]
                else:
                    assert not ch
                    segs = []
                for A, B in segs:
                    ia = _edge_corner(A, 0) if inside[_edge_corner(A, 0)] else _edge_corner(A, 1)
                    ma = [_bit(_edge_corner(A, 0), k) + _bit(_edge_corner(A, 1), k) for k in range(3)]
                    mb = [_bit(_edge_corner(B, 0), k) + _bit(_edge_corner(B, 1), k) for k in range(3)]
                    inn = [2 * _bit(ia, k) - ma[k] for k in range(3)]
                    nrm = [0, 0, 0]
                    nrm[a] = 1 if s else -1
                    d = np.subtract(mb, ma)
                    if np.dot(np.cross(d, nrm), inn) < 0:
                        A, B = B, A
                    assert A not in succ
                    succ[A] = B
        tris, seen = [], set()
        for e in range(12):
            if not change[e] or e in seen:
                continue
            loop, cur = [], e
            while True:
                loop.append(cur)
                seen.add(cur)
                cur = succ[cur]
                if cur == e:
                    break
            for k in range(1, len(loop) - 1):
                tris.append([loop[0], loop[k], loop[k + 1]])
        table.append(tris)
    return table


_TABLE = None


def table():
    global _TABLE
    if _TABLE is None:
        _TABLE = tri_table()
    return _TABLE


def mcubes(f: np.ndarray, lo, spacing):
    """(vertices fp64 [V, 3], triangles int32 [F, 3]) of one crop (rgs_unbounded_mcubes)."""
    n = f.shape[0]
    lo = np.asarray(lo, np.float64)
    sp = np.asarray(spacing, np.float64)
    inside = f < 0
    vm = np.zeros(f.shape, np.int64)
    for a in range(3):
        sl = [slice(None)] * 3
        sl[a] = slice(0, n - 1)
        sh = [slice(None)] * 3
        sh[a] = slice(1, n)
        vm[tuple(sl)] |= (inside[tuple(sl)] != inside[tuple(sh)]).astype(np.int64) << a
    cnt = ((vm & 1) + (vm >> 1 & 1) + (vm >> 2 & 1)).reshape(-1)
    voff = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    flat_f = f.reshape(-1)
    strides = (n * n, n, 1)
    verts = []
    for g in np.flatnonzero(cnt):
        p = np.unravel_index(g, f.shape)
        for a in range(3):
            if vm.reshape(-1)[g] >> a & 1:
                f0, f1 = np.float64(flat_f[g]), np.float64(flat_f[g + strides[a]])
                t = f0 / (f0 - f1)
                x = [np.float64(p[k]) + (t if k == a else 0.0) for k in range(3)]
                verts.append([x[k] * sp[k] + lo[k] for k in range(3)])
    cs = np.zeros((n - 1,) * 3, np.int64)
    for c in range(8):
        cs |= inside[c & 1:n - 1 + (c & 1), c >> 1 & 1:n - 1 + (c >> 1 & 1), c >> 2 & 1:n - 1 + (c >> 2 & 1)].astype(np.int64) << c
    tris = []
    T = table()
    vflat = vm.reshape(-1)
    for cell in np.flatnonzero(cs.reshape(-1)):
        i, j, k = np.unravel_index(cell, cs.shape)
        g = (i * n + j) * n + k
        for tri in T[cs.reshape(-1)[cell]]:
            row = []
            for e in tri:
                a, o = e // 4, e % 4
                h = g + (o & 1) * strides[_other_axis(a, 0)] + (o >> 1) * strides[_other_axis(a, 1)]
                row.append(voff[h] + bin(vflat[h] & ((1 << a) - 1)).count("1"))
            tris.append(row)
    return np.array(verts, np.float64).reshape(-1, 3), np.array(tris, np.int32).reshape(-1, 3)


# ---- merge and clusters -----------------------------------------------------------------------------------------------

def merge(verts: np.ndarray, tris: np.ndarray):
    """(vertices fp32 [U, 3], triangles int32 [F, 3]) of rgs_unbounded_merge."""
    keys = np.rint(verts * 1e6).astype(np.int64)
    assert np.all(np.abs(keys) < (1 << 21) + 1)
    _, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
    rep = first[inv.reshape(-1)]
    surv = rep == np.arange(len(verts))
    newid = np.cumsum(surv) - surv
    return verts[surv].astype(np.float32), newid[rep[tris]].astype(np.int32).reshape(-1, 3)


def clusters(V: int, tris: np.ndarray, k: int):
    """(kept vertex indices, kept triangles renumbered, cluster sizes) of post_process_mesh, with scipy's components."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    F = len(tris)
    if F == 0:
        return np.zeros(0, np.int64), np.zeros((0, 3), np.int32), np.zeros(0, np.int64)
    e = np.concatenate([np.sort(tris[:, [0, 1]], 1), np.sort(tris[:, [1, 2]], 1), np.sort(tris[:, [2, 0]], 1)])
    t = np.tile(np.arange(F), 3)
    _, eid = np.unique(e, axis=0, return_inverse=True)
    eid = eid.reshape(-1)
    g = sp.coo_matrix((np.ones(3 * F), (t, eid)), shape=(F, eid.max() + 1)).tocsr()
    adj = g @ g.T
    nc, lab = connected_components(adj, directed=False)
    sizes = np.bincount(lab, minlength=nc)
    srt = np.sort(sizes)
    if k == 0:
        thr = srt[0]
    elif k <= nc:
        thr = srt[-k]
    else:
        thr = 0
    thr = max(int(thr), 50)
    keep = sizes[lab] >= thr
    kept = tris[keep]
    ref = np.zeros(V, bool)
    ref[kept.reshape(-1)] = True
    newid = np.cumsum(ref) - ref
    kept = kept[(kept[:, 0] != kept[:, 1]) & (kept[:, 1] != kept[:, 2]) & (kept[:, 0] != kept[:, 2])]
    return np.flatnonzero(ref), newid[kept].astype(np.int32).reshape(-1, 3), sizes
