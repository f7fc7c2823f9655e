"""numpy model of the Tanks and Temples cull contracts (include/rgs_b200.h, rgs_tnt_mesh_depth and
rgs_tnt_visibility_count), bit for bit: every operation is one float32 numpy operation, rounded on its own, in the order
the header writes it.  numpy never fuses a multiply and an add, so these arrays are what the kernels must store."""
import numpy as np

f32 = np.float32
SMALL_AREA, MEDIUM_AREA = 16, 4096


def w2c_rows(c2w) -> np.ndarray:
    """[n, 12]: rows 0..2 of the fp64 inverse of the fp32-rounded pose, rounded to fp32 (rade_gs_b200.tnt_cull._w2c)."""
    c = np.asarray(c2w, np.float64).astype(np.float32).astype(np.float64).reshape(-1, 4, 4)
    return np.linalg.inv(c)[:, :3, :].astype(np.float32).reshape(-1, 12)


def to_camera(m, p):
    """m [12] float32, p [..., 3] float32 -> X, Y, Z: ((m_r0 x + m_r1 y) + m_r2 z) + m_r3."""
    m = np.asarray(m, f32)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return [((m[4 * r] * x + m[4 * r + 1] * y) + m[4 * r + 2] * z) + m[4 * r + 3] for r in range(3)]


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _sub(a, b):
    return tuple(a[k] - b[k] for k in range(3))


def _add(a, b):
    return tuple(a[k] + b[k] for k in range(3))


def _edge(c, dx, dy):
    return (c[0] * dx + c[1] * dy) + c[2]


def _tie(c):
    return (c[0] > 0) | ((c[0] == 0) & ((c[1] > 0) | ((c[1] == 0) & (c[2] > 0))))


def setup(vertices, faces, m, fx, fy, cx, cy, H, W, znear, zfar):
    """Per face: (draws bool [F], box int [F, 4] = x0, y0, x1, y1, edges [3][3] arrays, n [3] arrays, num)."""
    v = np.asarray(vertices, f32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    fx, fy, cx, cy, znear, zfar = (f32(a) for a in (fx, fy, cx, cy, znear, zfar))
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("face index outside [0, V)")
    with np.errstate(all="ignore"):
        X, Y, Z = to_camera(m, v)
        P = [(X[f[:, k]], Y[f[:, k]], Z[f[:, k]]) for k in range(3)]
        finite = np.ones(len(f), bool)
        for k in range(3):
            finite &= np.isfinite(P[k][0]) & np.isfinite(P[k][1]) & np.isfinite(P[k][2])
        zs = np.stack([P[k][2] for k in range(3)])
        all_near, all_far = (zs < znear).all(0), (zs > zfar).all(0)
        draws = finite & ~all_near & ~all_far
        us, ws = [], []
        for k in range(3):   # the face clipped at Z = znear: front vertices and edge crossings, in edge order
            a, b = P[k], P[(k + 1) % 3]
            front = ~(a[2] < znear)
            us.append(np.where(front, (fx * a[0]) / a[2] + cx, np.nan))
            ws.append(np.where(front, (fy * a[1]) / a[2] + cy, np.nan))
            cross = (a[2] < znear) != (b[2] < znear)
            s = (znear - a[2]) / (b[2] - a[2])
            q = [a[i] + s * (b[i] - a[i]) for i in range(3)]
            us.append(np.where(cross, (fx * q[0]) / q[2] + cx, np.nan))
            ws.append(np.where(cross, (fy * q[1]) / q[2] + cy, np.nan))
        u, w = np.stack(us), np.stack(ws)
        clamp = lambda a, hi: np.fmin(np.fmax(a, f32(-1)), f32(hi))  # noqa: E731
        umin, umax = clamp(np.fmin.reduce(u, 0), W), clamp(np.fmax.reduce(u, 0), W)
        vmin, vmax = clamp(np.fmin.reduce(w, 0), H), clamp(np.fmax.reduce(w, 0), H)
        box = np.stack([np.maximum(np.floor(umin - f32(0.5)), 0), np.maximum(np.floor(vmin - f32(0.5)), 0),
                        np.minimum(np.ceil(umax - f32(0.5)), W - 1), np.minimum(np.ceil(vmax - f32(0.5)), H - 1)], 1)
        box = np.where(np.isfinite(box), box, 0).astype(np.int64)
        draws &= (box[:, 0] <= box[:, 2]) & (box[:, 1] <= box[:, 3])
        n = _cross(_sub(P[1], P[0]), _sub(P[2], P[0]))
        num = (n[0] * P[0][0] + n[1] * P[0][1]) + n[2] * P[0][2]
        draws &= num != 0
        sgn = np.where(num < 0, f32(-1), f32(1))
        edges = []
        for k in range(3):
            a, b = P[k], P[(k + 1) % 3]
            c = _cross(_add(a, b), _sub(b, a))
            edges.append(tuple(c[i] * sgn for i in range(3)))   # negation: exact
    return draws, box, edges, n, num


def _fragments(idx, px, py, edges, n, num, fx, fy, cx, cy, znear, zfar, W):
    """Pixel (px, py) of face idx: (flat pixel index, depth) of the fragments that draw."""
    dx = ((px.astype(f32) + f32(0.5)) - f32(cx)) / f32(fx)
    dy = ((py.astype(f32) + f32(0.5)) - f32(cy)) / f32(fy)
    with np.errstate(all="ignore"):
        inside = np.ones(len(idx), bool)
        for c in edges:
            cc = tuple(c[i][idx] for i in range(3))
            e = _edge(cc, dx, dy)
            inside &= (e > 0) | ((e == 0) & _tie(cc))
        z = num[idx] / _edge(tuple(n[i][idx] for i in range(3)), dx, dy)
        keep = inside & (z >= f32(znear)) & (z <= f32(zfar))
    return py[keep].astype(np.int64) * W + px[keep], z[keep]


def split(vertices, faces, m, fx, fy, cx, cy, H, W, znear=0.01, zfar=20.0):
    """Faces on each side of the work split: (small, medium, large) counts of the faces that reach the pixel stage."""
    draws, box, *_ = setup(vertices, faces, m, fx, fy, cx, cy, H, W, znear, zfar)
    area = (box[:, 2] - box[:, 0] + 1) * (box[:, 3] - box[:, 1] + 1)
    a = area[draws]
    return int((a <= SMALL_AREA).sum()), int(((a > SMALL_AREA) & (a <= MEDIUM_AREA)).sum()), int((a > MEDIUM_AREA).sum())


def mesh_depth(vertices, faces, m, fx, fy, cx, cy, H, W, znear=0.01, zfar=20.0, chunk=1 << 20):
    """float32 [H, W]: rgs_tnt_mesh_depth."""
    draws, box, edges, n, num = setup(vertices, faces, m, fx, fy, cx, cy, H, W, znear, zfar)
    out = np.full(H * W, np.inf, f32)
    ids = np.nonzero(draws)[0]
    bw = box[ids, 2] - box[ids, 0] + 1
    area = bw * (box[ids, 3] - box[ids, 1] + 1)
    # enumerate every pixel of every box, in bounded chunks of (face, pixel) pairs
    ends = np.cumsum(area)
    start = 0
    while start < len(ids):
        base = ends[start] - area[start]
        stop = max(int(np.searchsorted(ends, base + chunk, side="right")), start + 1)
        sel, a, b = ids[start:stop], area[start:stop], bw[start:stop]
        rep = np.repeat(np.arange(len(sel)), a)
        p = np.arange(rep.size) - np.repeat(np.cumsum(a) - a, a)
        px = box[sel[rep], 0] + p % b[rep]
        py = box[sel[rep], 1] + p // b[rep]
        pix, z = _fragments(sel[rep], px, py, edges, n, num, fx, fy, cx, cy, znear, zfar, W)
        np.minimum.at(out, pix, z)
        start = stop
    out[np.isinf(out)] = 0
    return out.reshape(H, W)


def visibility(points, depth, m, fx, fy, cx, cy, eps=0.005):
    """(seen bool [N], in_frustum bool [N], z, s): rgs_tnt_visibility_count for one view, with the quantities its decisions
    compare (z and the sample s), for margin checks."""
    p = np.asarray(points, f32).reshape(-1, 3)
    D = np.asarray(depth, f32)
    H, W = D.shape
    fx, fy, cx, cy, eps = (f32(a) for a in (fx, fy, cx, cy, eps))
    with np.errstate(all="ignore"):
        X, Y, Z = to_camera(m, p)
        z = Z + f32(1e-8)
        u = (fx * X + cx * Z) / z
        v = (fy * Y + cy * Z) / z
        Wm1, Hm1 = f32(W - 1), f32(H - 1)
        fr = (u >= 0) & (u <= Wm1) & (v >= 0) & (v <= Hm1) & (z > 0)
        uu, vv = np.where(fr, u, f32(0)), np.where(fr, v, f32(0))
        gx = (uu * (f32(1) / Wm1)) * f32(2) - f32(1)
        gy = (vv * (f32(1) / Hm1)) * f32(2) - f32(1)
        ix = np.minimum(Wm1, np.maximum(((gx + f32(1)) / f32(2)) * Wm1, f32(0)))
        iy = np.minimum(Hm1, np.maximum(((gy + f32(1)) / f32(2)) * Hm1, f32(0)))
        x0, y0 = np.floor(ix), np.floor(iy)
        x1, y1 = x0 + f32(1), y0 + f32(1)
        xi, yi = x0.astype(np.int64), y0.astype(np.int64)
        xr, yb = xi + 1 < W, yi + 1 < H
        at = lambda yy, xx, ok: np.where(ok, D[np.minimum(yy, H - 1), np.minimum(xx, W - 1)], f32(0))  # noqa: E731
        s = np.zeros(len(p), f32)
        s = s + at(yi, xi, True) * ((x1 - ix) * (y1 - iy))
        s = np.where(xr, s + at(yi, xi + 1, xr) * ((ix - x0) * (y1 - iy)), s)
        s = np.where(yb, s + at(yi + 1, xi, yb) * ((x1 - ix) * (iy - y0)), s)
        s = np.where(xr & yb, s + at(yi + 1, xi + 1, xr & yb) * ((ix - x0) * (iy - y0)), s)
        seen = fr & np.where(s > 0, z < s + eps, True)
    return seen, fr, z, s


def visibility_count(points, depths, ms, fx, fy, cx, cy, eps=0.005) -> np.ndarray:
    """int32 [N]: the counts after one rgs_tnt_visibility_count per view, from zero."""
    counts = np.zeros(len(np.asarray(points).reshape(-1, 3)), np.int32)
    for D, m in zip(depths, ms):
        counts += visibility(points, D, m, fx, fy, cx, cy, eps)[0]
    return counts
