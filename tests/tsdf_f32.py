"""numpy float32 restatement of the TSDF contract in include/rgs_b200.h (touch, integrate, triangle table, marching cubes,
vertex normals), operation by operation, so that every stored bit of rgs_tsdf.cu can be compared.  Test infrastructure
only: the product never imports it.  numpy float32 arithmetic rounds every operation on its own and never contracts to
FMA, which is the contract's arithmetic.

The grid is a dict  key -> (tsdf [4096], weight [4096], color [4096, 3])  with voxels x fastest inside a block."""
from __future__ import annotations

import numpy as np

F = np.float32
RES = 16
BV = RES ** 3
BIAS = 1 << 20
KEY_LO, KEY_HI = -BIAS + 1, BIAS - 2      # block range a camera may reach


def pack(b):
    b = np.asarray(b, np.int64).reshape(-1, 3) + BIAS
    return (b[:, 0] << 42) | (b[:, 1] << 21) | b[:, 2]


def unpack(k):
    k = np.asarray(k, np.int64)
    m = (1 << 21) - 1
    return np.stack([(k >> 42) & m, (k >> 21) & m, k & m], 1) - BIAS


class Camera:
    """fp32 parameters as the contract takes them: intrinsic 3x3 and world->camera extrinsic 4x4 (any float type)."""

    def __init__(self, intrinsic, extrinsic, H, W, voxel_size, depth_scale=1.0, depth_max=3.0, trunc_voxel_multiplier=8.0):
        K = np.asarray(intrinsic, np.float64)
        E = np.asarray(extrinsic, np.float64)
        self.H, self.W = H, W
        self.fx, self.fy, self.cx, self.cy = F(K[0, 0]), F(K[1, 1]), F(K[0, 2]), F(K[1, 2])
        self.R = E[:3, :3].astype(F)
        self.t = E[:3, 3].astype(F)
        self.vs = F(voxel_size)
        self.depth_scale, self.depth_max = F(depth_scale), F(depth_max)
        self.trunc = F(F(trunc_voxel_multiplier) * self.vs)


# ---- touch --------------------------------------------------------------------------------------------------------------

def touch(cam: Camera, depth):
    depth = np.asarray(depth, F).reshape(cam.H, cam.W)
    d = depth / cam.depth_scale
    j, i = np.nonzero((d > 0) & (d <= cam.depth_max))
    d = d[j, i]
    xn = ((i.astype(F) + F(0.5)) - cam.cx) / cam.fx
    yn = ((j.astype(F) + F(0.5)) - cam.cy) / cam.fy
    bs = F(cam.vs * F(RES))
    ends = []
    for z in (d - cam.trunc, d + cam.trunc):
        q = [xn * z - cam.t[0], yn * z - cam.t[1], z - cam.t[2]]
        pw = [(cam.R[0, k] * q[0] + cam.R[1, k] * q[1]) + cam.R[2, k] * q[2] for k in range(3)]
        ends.append(np.stack([np.floor(p / bs) for p in pw], 1))
    lo, hi = np.minimum(ends[0], ends[1]), np.maximum(ends[0], ends[1])
    ok = np.all((lo >= KEY_LO) & (hi <= KEY_HI), axis=1)
    lo, hi = lo[ok].astype(np.int64), hi[ok].astype(np.int64)
    if len(lo) == 0:
        return np.zeros((0, 3), np.int32)
    ext = (hi - lo).max(0) + 1
    keys = []
    for dz in range(ext[2]):
        for dy in range(ext[1]):
            for dx in range(ext[0]):
                o = np.array([dx, dy, dz])
                m = np.all(lo + o <= hi, axis=1)
                keys.append(pack(lo[m] + o))
    return unpack(np.unique(np.concatenate(keys))).astype(np.int32)


# ---- integrate ----------------------------------------------------------------------------------------------------------

_V = np.arange(BV)
_LOCAL = np.stack([_V % RES, _V // RES % RES, _V // (RES * RES)], 1)    # (x, y, z) of voxel v = x + 16 y + 256 z


def grid_points(blocks):
    """int64 [n, 4096, 3] grid points of blocks [n, 3]."""
    return np.asarray(blocks, np.int64)[:, None, :] * RES + _LOCAL[None]


def integrate(grid: dict, cam: Camera, block_coords, depth, color):
    depth = np.asarray(depth, F).reshape(cam.H, cam.W)
    color = np.asarray(color, F).reshape(cam.H, cam.W, 3)
    keys = np.unique(pack(block_coords))
    for k in keys:
        if int(k) not in grid:
            grid[int(k)] = (np.zeros(BV, F), np.zeros(BV, F), np.zeros((BV, 3), F))
    if len(keys) == 0:
        return
    p = grid_points(unpack(keys)).astype(F) * cam.vs                    # [n, 4096, 3]
    R, t = cam.R, cam.t
    xc = ((R[0, 0] * p[..., 0] + R[0, 1] * p[..., 1]) + R[0, 2] * p[..., 2]) + t[0]
    yc = ((R[1, 0] * p[..., 0] + R[1, 1] * p[..., 1]) + R[1, 2] * p[..., 2]) + t[1]
    zc = ((R[2, 0] * p[..., 0] + R[2, 1] * p[..., 1]) + R[2, 2] * p[..., 2]) + t[2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = np.floor((cam.fx * xc) / zc + cam.cx)
        v = np.floor((cam.fy * yc) / zc + cam.cy)
        ok = (zc > 0) & (u >= 0) & (u < cam.W) & (v >= 0) & (v < cam.H)
    ui, vi = np.where(ok, u, 0).astype(np.int64), np.where(ok, v, 0).astype(np.int64)
    d = depth[vi, ui] / cam.depth_scale
    sdf = d - zc
    ok &= (d > 0) & (d <= cam.depth_max) & (sdf >= -cam.trunc)
    obs = np.minimum(sdf, cam.trunc) / cam.trunc
    col = color[vi, ui]
    for n, k in enumerate(keys):
        ts, w, c = grid[int(k)]
        m = ok[n]
        w1 = w[m] + F(1)
        ts[m] = (w[m] * ts[m] + obs[n][m]) / w1
        c[m] = (w[m][:, None] * c[m] + col[n][m]) / w1[:, None]
        w[m] = w1


def active(grid: dict):
    keys = np.array(sorted(grid), np.int64)
    if len(keys) == 0:
        return keys, np.zeros((0, BV), F), np.zeros((0, BV), F), np.zeros((0, BV, 3), F)
    return keys, np.stack([grid[int(k)][0] for k in keys]), np.stack([grid[int(k)][1] for k in keys]), np.stack([grid[int(k)][2] for k in keys])


# ---- triangle table -----------------------------------------------------------------------------------------------------

CORNERS = np.array([[c & 1, c >> 1 & 1, c >> 2 & 1] for c in range(8)])


def _other(a):
    return [b for b in range(3) if b != a]


def edge_ends(e):
    """corner positions (2 x 3 ints) of edge e: axis e // 4, offsets (e & 1, e >> 1 & 1) on the other axes."""
    a, o = e // 4, e % 4
    p = np.zeros(3, int)
    b, c = _other(a)
    p[b], p[c] = o & 1, o >> 1 & 1
    q = p.copy()
    q[a] = 1
    return p, q


def corner_id(p):
    return int(p[0] + 2 * p[1] + 4 * p[2])


def face_segments(case):
    """{first edge: second edge} of the directed iso-segments of all six faces, and the ambiguous faces (axis, side)."""
    inside = [(case >> c) & 1 for c in range(8)]
    succ, ambiguous = {}, []
    for a in range(3):
        for s in range(2):
            n_out = np.zeros(3, int)
            n_out[a] = 1 if s else -1
            fe = [e for e in range(12) if e // 4 != a and edge_ends(e)[0][a] == s]
            ch = [e for e in fe if inside[corner_id(edge_ends(e)[0])] != inside[corner_id(edge_ends(e)[1])]]
            if len(ch) == 2:
                pairs = [tuple(ch)]
            elif len(ch) == 4:   # ambiguous face: cut off each inside corner with its own segment
                ambiguous.append((a, s))
                pairs = [tuple(e for e in fe if c in (corner_id(edge_ends(e)[0]), corner_id(edge_ends(e)[1])))
                         for c in range(8) if CORNERS[c][a] == s and inside[c]]
            else:
                assert not ch
                pairs = []
            for A, B in pairs:
                pa, qa = edge_ends(A)
                pb, qb = edge_ends(B)
                ma, mb = pa + qa, pb + qb                       # doubled midpoints
                ins = 2 * (pa if inside[corner_id(pa)] else qa)
                if np.dot(np.cross(mb - ma, n_out), ins - ma) < 0:
                    A, B = B, A
                assert A not in succ
                succ[A] = B
    return succ, ambiguous


def loops(case):
    succ, _ = face_segments(case)
    assert sorted(succ) == sorted(succ.values())           # every sign-change edge: one segment out, one in
    seen, out = set(), []
    for e in sorted(succ):
        if e in seen:
            continue
        loop = [e]
        while succ[loop[-1]] != e:
            loop.append(succ[loop[-1]])
        seen.update(loop)
        out.append(loop)
    return out


def triangle_table():
    """list of 256 lists of (e0, e1, e2), derived from the rule in the header."""
    return [[(lp[0], lp[k], lp[k + 1]) for lp in loops(case) for k in range(1, len(lp) - 1)] for case in range(256)]


TABLE = triangle_table()
MAX_TRI = max(len(t) for t in TABLE)


# ---- marching cubes -----------------------------------------------------------------------------------------------------

def extract(grid: dict, vs, weight_threshold=3.0):
    """-> vertices f32 [V,3], colors f32 [V,3], triangles int32 [F,3] in the contract's order."""
    vs, thr = F(vs), F(weight_threshold)
    keys, ts, w, col = active(grid)
    N = len(keys)
    if N == 0:
        return np.zeros((0, 3), F), np.zeros((0, 3), F), np.zeros((0, 3), np.int32)
    blocks = unpack(keys)
    nbr = np.full((N, 27), -1, np.int64)
    for k in range(27):
        o = np.array([k % 3 - 1, k // 3 % 3 - 1, k // 9 - 1])
        nk = pack(blocks + o)
        pos = np.searchsorted(keys, nk)
        hit = (pos < N) & (keys[np.minimum(pos, N - 1)] == nk)
        nbr[:, k] = np.where(hit, pos, -1)
    ts, w, col = ts.reshape(-1), w.reshape(-1), col.reshape(-1, 3)
    valid = w >= thr
    inside = ts < 0
    bi = np.repeat(np.arange(N), BV)
    loc = np.tile(_LOCAL, (N, 1))

    def fetch(off):
        """flat voxel index of g + off for every voxel g, -1 where the block is missing"""
        q = loc + off
        k = (np.floor_divide(q[:, 0], RES) + 1) + 3 * (np.floor_divide(q[:, 1], RES) + 1) + 9 * (np.floor_divide(q[:, 2], RES) + 1)
        j = nbr[bi, k]
        qi = q % RES
        return np.where(j >= 0, j * BV + qi[:, 0] + RES * qi[:, 1] + RES * RES * qi[:, 2], -1)

    def valid_at(idx):
        return (idx >= 0) & valid[np.maximum(idx, 0)]

    case = np.zeros(N * BV, np.int64)
    cell_ok = np.ones(N * BV, bool)
    for c in range(8):
        idx = fetch(CORNERS[c])
        cell_ok &= valid_at(idx)
        case |= (inside[np.maximum(idx, 0)] & (idx >= 0)).astype(np.int64) << c

    def cell_ok_at(off):
        idx = fetch(np.asarray(off))
        return (idx >= 0) & cell_ok[np.maximum(idx, 0)]

    vmask = np.zeros(N * BV, np.int64)
    nxt = {}
    for a in range(3):
        e = np.zeros(3, int)
        e[a] = 1
        nxt[a] = fetch(e)
        b, c = _other(a)
        near = np.zeros(N * BV, bool)
        for ob in (0, 1):
            for oc in (0, 1):
                off = np.zeros(3, int)
                off[b], off[c] = -ob, -oc
                near |= cell_ok_at(off)
        j = nxt[a]
        change = (j >= 0) & (inside != inside[np.maximum(j, 0)])
        vmask |= (near & change).astype(np.int64) << a
    vcnt = (vmask & 1) + (vmask >> 1 & 1) + (vmask >> 2 & 1)
    voff = np.cumsum(vcnt) - vcnt
    V = int(vcnt.sum())
    verts = np.zeros((V, 3), F)
    vcol = np.zeros((V, 3), F)
    gp = (blocks[bi] * RES + loc).astype(F) * vs              # grid point positions
    for a in range(3):
        m = (vmask >> a & 1).astype(bool)
        r = voff + ((vmask & ((1 << a) - 1)) & 1) + ((vmask & ((1 << a) - 1)) >> 1 & 1)
        j = nxt[a][m]
        f0, f1 = ts[m], ts[j]
        t = f0 / (f0 - f1)
        p = gp[m].copy()
        p[:, a] = p[:, a] + t * vs
        verts[r[m]] = p
        c0, c1 = col[m], col[j]
        vcol[r[m]] = c0 + t[:, None] * (c1 - c0)
    # triangles in (voxel, table order)
    ntri = np.array([len(t) for t in TABLE])
    tab = np.full((256, MAX_TRI, 3), -1, np.int64)
    for cs, tl in enumerate(TABLE):
        if tl:
            tab[cs, :len(tl)] = tl
    cells = np.flatnonzero(cell_ok & (ntri[case] > 0))
    edges = tab[case[cells]]                                  # [n, MAX_TRI, 3]
    vid = np.full(edges.shape, -1, np.int64)
    for e in range(12):
        p, _ = edge_ends(e)
        a = e // 4
        own = fetch(p)[cells]
        idx = voff[own] + ((vmask[own] & ((1 << a) - 1)) & 1) + ((vmask[own] & ((1 << a) - 1)) >> 1 & 1)
        assert np.all(np.broadcast_to((vmask[own] >> a & 1)[:, None, None], edges.shape)[edges == e] == 1)
        vid = np.where(edges == e, idx[:, None, None], vid)
    tris = vid[np.arange(MAX_TRI)[None, :] < ntri[case[cells]][:, None]].astype(np.int32)
    return verts, vcol, tris.reshape(-1, 3)


def vertex_normals(verts, tris):
    verts = np.asarray(verts, F)
    tris = np.asarray(tris, np.int64)
    v0, v1, v2 = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    a, b = v1 - v0, v2 - v0
    nf = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    acc = np.zeros((len(verts), 3), F)
    np.add.at(acc, tris.reshape(-1), np.repeat(nf, 3, axis=0))  # unbuffered, in index order: ascending triangle per vertex
    ln = np.sqrt((acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        out = acc / ln[:, None]
    out[ln == 0] = 0
    return out.astype(F)
