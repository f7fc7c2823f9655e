"""fp64 evaluation of `integrate_gaussians_to_points` with per-element bounds on what an fp32 evaluation may differ by.

The integrate kernels (csrc/rgs_integrate.cu) and the CPU oracle (oracle/oracle.c, `orc_inte_geometry` / `orc_integrate`)
evaluate in fp32 what the reference does in forward.cu:187-235, 857-900 and 938-1372:
  * invray: the inverse covariance in (pixel x, pixel y, ray depth) space of every Gaussian, from the stored fp32 Sigma^-1;
  * phase A: every pixel walks its tile's list with five samples (centre and four corners), each with its own transmittance.
    `test_T < 1e-4` SKIPS the entry for that sample and the walk goes on; an entry is *used* by the pixel when any sample takes
    it, and the pixel stops after its 2048th used entry.  The centre sample writes colour, depth, median depth and alpha; every
    sample feeds the maximum depth;
  * phase B: every query point that projects into the image composites, with the 3D ray-space Gaussian, the used entries of
    its pixel, and reads its SDF off the plane of the pixel's median contributor.

This module evaluates the same in fp64 from the same fp32 inputs (this build's decoded buffers or the oracle's state) and
carries a rigorous bound next to every value, the way tests/blend_f64.py does for the blend.  A decision whose fp32 value may
fall on either side of its threshold is *ambiguous*: `power > 0`, `alpha < 1/255`, `test_T < 1e-4`, `T > 0.5` in phase A; the
near plane, the image borders and the `qd < depth` skip in phase B.  `depth > Cmax` needs no classification: Cmax is a running
maximum, which moves by at most the largest error of its arguments whichever way a tie is decided.

Phase A is a skip recurrence, so blend's cumprod-until-stop does not apply.  It is scanned in blocks of BLOCK list positions:
within a block every candidate is speculatively taken, the first entry whose test fails is dropped, and the block is rescanned
(once a transmittance is below 1e-4 / (1 - 1/255) every later entry fails, and the rest of the block is dropped at once).  Memory
is O(tiles x 256 x 5 x BLOCK), whatever the list length.  Phase B runs inside the same scan: every point gathers its pixel's
used entries of the block, so no used set is ever stored.

alpha_integrated = 1 - prod (1 - alpha_j) over the used entries j of the pixel whose alpha >= 1/255 is monotone in the set and in
every alpha_j, so each point gets an envelope [set surely taken with the lowest alphas, set possibly taken with the highest],
and needs no outlier budget.  Everything is torch: it runs on the CPU (host tests) and on the GPU.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from blend_f64 import ALPHA_MAX, ALPHA_MIN, K_EXPF, K_POWER, PAIR_BUDGET, T_MEDIAN, T_STOP, U, _f32, _np64, _ratio, focal

MAX_CONTRIB = 2048           # MAX_NUM_CONTRIBUTORS * 4 (auxiliary.h:31, forward.cu:1126)
NEAR = _f32(0.2)             # v.z > 0.2f (auxiliary.h:170)
EPS_Z = _f32(0.0000001)      # v.z + 0.0000001f in the point projection
BLOCK = 256                  # list positions scanned at once
OFFSETS = ((0.0, 0.0), (-0.5, -0.5), (0.5, -0.5), (-0.5, 0.5), (0.5, 0.5))   # centre, then the corners in the kernel's order

# invray = S T2^T Sigma^-1 T2 S in fp32.  t = V p carries 3 roundings (or 2 fused), u/v = t/t_z clamped and re-divided 3 more;
# each entry of `full` (sums of products of u, v, 1/l, l_tz and f) adds at most 6, so every entry of T2 = W full^T (3-term
# sums) is within ~12u of |W| |full|^T.  T2 enters the quadratic form twice (24u), the two 3-term products add 6u and the
# 1/focal scaling (a rounded reciprocal and two products) 4u: 34u of |T2|^T |Sigma^-1| |T2|, scaled.  40 leaves margin for
# the second-order terms.
K_INVRAY = 40.0
# Phase B power = -0.5 d.(M d) with d = (dx, dy, dz) and M the six stored entries: the inner 3-term sums and the outer one
# round at most 3u each of the magnitudes |M||d||d|; 8u leaves room for second-order terms.  Errors of M and d come on top.
K_POW3 = 8.0
# Recursive fp32 sums / products of n terms: (n - 1)u for the sum, 2u per layer for the transmittance, a few per term.
KAPPA = 4.0
# xform4x3: three products and three sums (or fused) of magnitude sum |V_ij p_j| + |V_i3|.
K_XF = 4.0

# At most this fraction of a family's pixels, or of its in-image points, may be ambiguous, unless the family states its own
# ceiling (tests/test_gpu_integrate_exact.py records the fractions measured on an H100).
AMBIGUOUS_CEILING = 0.05


@dataclass
class Integrate:
    """One integrate problem: fp32 per-Gaussian state (phase A records, Sigma^-1 and its flags, radii, centres), the sorted
    tile lists and the camera."""
    means2D: torch.Tensor        # [P,2]
    conic_opacity: torch.Tensor  # [P,4] (A, B, C, opacity)
    rgb: torch.Tensor            # [P,3]
    ts: torch.Tensor             # [P]
    ray_planes: torch.Tensor     # [P,2]
    sigma_inv: torch.Tensor      # [P,9] column-major (symmetric up to rounding)
    flags: torch.Tensor          # [P] int: bit 0 well-conditioned, bit 1 solver converged
    radii: torch.Tensor          # [P]
    means3D: torch.Tensor        # [P,3]
    ranges: torch.Tensor         # [tiles,2]
    point_list: torch.Tensor     # [R]
    V: torch.Tensor              # [16] view matrix as passed (x_view_j = sum_i x_i V[4i + j] + V[12 + j])
    bg: torch.Tensor             # [3]
    W: int
    H: int
    tanfovx: float
    tanfovy: float
    focal_x: float
    focal_y: float

    @property
    def device(self):
        return self.means2D.device


def make_integrate(st: dict, W, H, tanfovx, tanfovy, bg, viewmatrix, means3D, device="cpu") -> Integrate:
    """From plain arrays: means2D, conic_opacity, rgb, ts, ray_planes, radii, ranges, point_list, sigma_inv ([P,9] or [P,12]
    with the flag bits in float 9) and optionally flags."""
    def t(v, integer=False):
        v = np.ascontiguousarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v)
        if integer:
            if v.dtype in (np.int32, np.uint32):
                v = v.view(np.uint32).astype(np.int64)
            return torch.as_tensor(v.astype(np.int64)).to(device)
        return torch.as_tensor(v).to(device, torch.float64)
    si = st["sigma_inv"]
    si = si.detach().cpu().numpy() if isinstance(si, torch.Tensor) else np.asarray(si)
    si = np.ascontiguousarray(si, np.float32)
    flags = st.get("flags")
    if flags is None:
        flags = si[:, 9].view(np.int32).copy()
    return Integrate(t(st["means2D"]), t(st["conic_opacity"]), t(st["rgb"]), t(st["ts"]).reshape(-1), t(st["ray_planes"]),
                     t(si[:, :9]), t(np.asarray(flags, np.int64), True), t(st["radii"], True), t(means3D),
                     t(st["ranges"], True).reshape(-1, 2), t(st["point_list"], True).reshape(-1),
                     t(np.asarray(viewmatrix, np.float32).reshape(-1)), t(np.asarray(bg, np.float32)), int(W), int(H),
                     float(tanfovx), float(tanfovy), focal(W, tanfovx), focal(H, tanfovy))


# ---- invray (inte_geometry_kernel) -------------------------------------------------------------------------------------

def _xform(V, p):
    """x_view = p (V rows 0-2) + V row 3, with the magnitude its fp32 evaluation errs against."""
    Vm = V.view(4, 4)
    v = p @ Vm[:3, :3] + Vm[3, :3]
    mag = p.abs() @ Vm[:3, :3].abs() + Vm[3, :3].abs()
    return v, mag


def invray(it: Integrate) -> dict:
    """The six stored entries (xx, xy, xz, yy, yz, zz) of every Gaussian's ray-space inverse covariance, their bound and the
    `condition` flag.  Zero where !solved, where Sigma^-1 W (u, v, 1) has no direction (NaN in the kernel) or radii == 0."""
    P, dev = it.means3D.shape[0], it.device
    well = (it.flags & 1) != 0
    solved = (it.flags & 2) != 0
    t, _ = _xform(it.V, it.means3D)
    limx, limy = _f32(np.float32(1.3) * np.float32(it.tanfovx)), _f32(np.float32(1.3) * np.float32(it.tanfovy))
    tz = t[:, 2]
    u = (t[:, 0] / tz).clamp(-limx, limx)
    v = (t[:, 1] / tz).clamp(-limy, limy)
    tx, ty = u * tz, v * tz
    S = it.sigma_inv.view(P, 3, 3).transpose(1, 2)          # column-major storage: S[i][j] = stored[3 j + i]
    Wm = it.V.view(4, 4)[:3, :3].expand(P, 3, 3)
    cci = Wm.transpose(1, 2) @ S @ Wm
    uvh = torch.stack([u, v, torch.ones_like(u)], 1)
    um = (cci @ uvh[:, :, None])[:, :, 0]
    nrm = um.norm(dim=1)
    finite = torch.isfinite(nrm) & (nrm > 0)
    u2, v2, uv = u * u, v * v, u * v
    l = torch.sqrt(tx * tx + ty * ty + tz * tz)
    ltz = u2 + v2 + 1
    f = tz / ltz
    z0 = torch.zeros_like(u)
    # columns of `full` (rgs_integrate.cu: m3(...) is column-major) -> full[i][j] = column j, row i
    c0 = torch.stack([v2 + 1, -uv, u / l * ltz], 1)
    c1 = torch.stack([-uv, u2 + 1, v / l * ltz], 1)
    c2 = torch.stack([-u, -v, 1 / l * ltz], 1)
    full = torch.stack([c0, c1, c2], 2) * f[:, None, None]
    T2 = Wm @ full.transpose(1, 2)
    inv = T2.transpose(1, 2) @ S @ T2
    T2a = Wm.abs() @ full.abs().transpose(1, 2)
    mag = T2a.transpose(1, 2) @ S.abs() @ T2a
    sc = torch.tensor([1.0 / it.focal_x, 1.0 / it.focal_y, 1.0], dtype=torch.float64, device=dev)
    inv = inv * sc[None, :, None] * sc[None, None, :]
    mag = mag * sc[None, :, None] * sc[None, None, :]
    live = (it.radii > 0) & solved & well & finite
    ii, jj = [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]
    M = torch.where(live[:, None], inv[:, ii, jj], z0[:, None])
    bM = torch.where(live[:, None], K_INVRAY * U * mag[:, ii, jj], z0[:, None])
    return dict(M=torch.nan_to_num(M), b_M=torch.nan_to_num(bM, nan=0.0), condition=well & (it.radii > 0), live=live)


# ---- query points (integrate_points_project_kernel) ----------------------------------------------------------------------

def project(it: Integrate, points3D) -> dict:
    """fp64 image coordinate, view depth and distance of every point, their bounds, the in-image decision and its ambiguity."""
    p = torch.as_tensor(np.asarray(points3D, np.float32)).to(it.device, torch.float64)
    v, mag = _xform(it.V, p)
    ev = K_XF * U * mag
    vz = v[:, 2]
    den = vz + EPS_Z
    out = {}
    for ax, (fc, size) in enumerate(((it.focal_x, it.W), (it.focal_y, it.H))):
        a = fc * v[:, ax] / den
        ea = abs(fc) * ev[:, ax] / den.abs() + a.abs() * ev[:, 2] / den.abs() + 3 * U * a.abs()
        im = a + size / 2.0
        out["im" + "xy"[ax]] = im
        out["e_im" + "xy"[ax]] = ea + U * im.abs()
    qd = v.norm(dim=1)
    e_qd = (v.abs() * ev).sum(1) / qd.clamp(min=1e-300) + 3 * U * qd
    front = vz > NEAR
    amb = (vz - NEAR).abs() <= ev[:, 2]
    ix, iy, ex, ey = out["imx"], out["imy"], out["e_imx"], out["e_imy"]
    inside = (ix >= 0) & (ix < it.W) & (iy >= 0) & (iy < it.H)
    amb_in = ((ix.abs() <= ex) | ((ix - it.W).abs() <= ex) | (iy.abs() <= ey) | ((iy - it.H).abs() <= ey)) & front
    out.update(vz=vz, e_vz=ev[:, 2], qd=qd, e_qd=e_qd, inside=front & inside, ambiguous=amb | amb_in)
    return out


# ---- phase A + phase B ----------------------------------------------------------------------------------------------------

def _tile_chunks(it: Integrate, tiles_subset=None):
    n = (it.ranges[:, 1] - it.ranges[:, 0]).cpu()
    order = torch.argsort(n, descending=True) if tiles_subset is None else torch.as_tensor(tiles_subset)
    budget = PAIR_BUDGET["cuda" if it.device.type == "cuda" else "cpu"]
    i, T = 0, order.numel()
    while i < T:
        L = max(int(n[order[i]]), 1)
        k = max(1, min(T - i, budget // (256 * 5 * min(L, BLOCK))))
        yield order[i:i + k].to(it.device), max(int(n[order[i:i + k]].max()), 1)
        i += k


def _excl_cumprod(f):
    c = torch.cumprod(f, -1)
    return torch.cat([torch.ones_like(c[..., :1]), c[..., :-1]], -1)


def _first(mask, pos, none):
    return torch.where(mask, pos, torch.full_like(pos, none)).min(-1).values


PIXEL_KEYS = ("color0", "color1", "color2", "color3", "color4", "color6", "color7")
POINT_CHUNK = 1 << 14


def integrate(it: Integrate, points3D, coord_given, in_given, tiles_subset=None, trace=None) -> dict:
    """The fp64 model of one call.  `coord_given` [PN,2] and `in_given` [PN] are the point coordinates and in-image decisions
    of the implementation under test: phase B evaluates every point it placed in the image at the pixel it reports (the
    coordinate itself is checked against `project` by `check`).

    Returns per pixel ([H,W]): the channels `color{0,1,2,3,4,6,7}` with bounds `b_*` (inf where an ambiguous decision makes
    the channel unconstrained), `n_used`, `last`, `overflow`, `ambiguous`; per point: `alpha` (fp64), `alpha_lo`/`alpha_hi`
    (the envelope), `sdf`, `b_sdf` (inf = unchecked), `point_ambiguous`; and `overflow_count`.  With `trace` = (y, x) the
    per-position decisions of that pixel are returned under `trace` (used by the host tests to plant defects)."""
    H, W, dev = it.H, it.W, it.device
    HW = H * W
    gx = (W + 15) // 16
    inv = invray(it)
    M, bM, cond = inv["M"], inv["b_M"], inv["condition"]
    pr = project(it, points3D)
    PN = pr["qd"].shape[0]
    cg = torch.as_tensor(np.asarray(coord_given, np.float32)).to(dev, torch.float64).reshape(PN, 2)
    ing = torch.as_tensor(np.asarray(in_given, bool)).to(dev)
    qpix = torch.where(ing, cg[:, 1].floor().long().clamp(0, H - 1) * W + cg[:, 0].floor().long().clamp(0, W - 1), torch.full_like(ing, -1, dtype=torch.long))
    qtile = torch.where(ing, (qpix // W // 16) * gx + (qpix % W) // 16, torch.full_like(qpix, -1))
    qloc = ((qpix // W) % 16) * 16 + (qpix % W) % 16

    res = {k: torch.zeros(HW, dtype=torch.float64, device=dev) for k in PIXEL_KEYS}
    bnd = {k: torch.zeros(HW, dtype=torch.float64, device=dev) for k in PIXEL_KEYS}
    n_used_px = torch.zeros(HW, dtype=torch.int64, device=dev)
    last_px = torch.zeros(HW, dtype=torch.int64, device=dev)
    over_px = torch.zeros(HW, dtype=torch.bool, device=dev)
    amb_px = torch.zeros(HW, dtype=torch.bool, device=dev)
    logT64 = torch.zeros(PN, dtype=torch.float64, device=dev)
    logT_lo = torch.zeros(PN, dtype=torch.float64, device=dev)   # over the possible set with the highest alphas
    logT_hi = torch.zeros(PN, dtype=torch.float64, device=dev)   # over the sure set with the lowest alphas
    n_pt = torch.zeros(PN, dtype=torch.float64, device=dev)
    sdf = torch.zeros(PN, dtype=torch.float64, device=dev)
    b_sdf = torch.full((PN,), float("inf"), dtype=torch.float64, device=dev)
    pt_amb = pr["ambiguous"].clone()
    kap = KAPPA * U
    tr = None
    offx = torch.tensor([o[0] for o in OFFSETS], dtype=torch.float64, device=dev).view(1, 1, 5, 1)
    offy = torch.tensor([o[1] for o in OFFSETS], dtype=torch.float64, device=dev).view(1, 1, 5, 1)

    for tiles, L in _tile_chunks(it, tiles_subset):
        nt = tiles.numel()
        loc = torch.arange(256, device=dev)
        px = (tiles % gx)[:, None] * 16 + loc % 16
        py = (tiles // gx)[:, None] * 16 + loc // 16
        inside = (px < W) & (py < H)
        pix = py.clamp(max=H - 1) * W + px.clamp(max=W - 1)
        start, n = it.ranges[tiles, 0], it.ranges[tiles, 1] - it.ranges[tiles, 0]
        # the chunk's points, grouped by (tile in chunk, pixel in tile)
        tpos = torch.full((it.ranges.shape[0],), -1, dtype=torch.long, device=dev)
        tpos[tiles] = torch.arange(nt, device=dev)
        sel = (qtile >= 0) & (tpos[qtile.clamp(min=0)] >= 0)
        pts = torch.nonzero(sel).flatten()
        p_t, p_l = tpos[qtile[pts]], qloc[pts]
        # per-pixel state, per sample: transmittance, its relative error bound
        T = torch.ones(nt, 256, 5, dtype=torch.float64, device=dev)
        eT = torch.zeros_like(T)
        n_used = torch.zeros(nt, 256, dtype=torch.int64, device=dev)
        stopped = ~inside
        first_amb = torch.full((nt, 256), 1 << 40, dtype=torch.int64, device=dev)
        T_a = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
        acc = {k: torch.zeros(nt, 256, dtype=torch.float64, device=dev) for k in ("c0", "c1", "c2", "d", "a")}
        accb = {k: torch.zeros(nt, 256, dtype=torch.float64, device=dev) for k in acc}     # sum w |v| r_w
        accm = {k: torch.zeros(nt, 256, dtype=torch.float64, device=dev) for k in acc}     # sum w |v|abs
        vmax = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
        n0 = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
        cmax = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
        b_cmax = torch.zeros(nt, 256, dtype=torch.float64, device=dev)
        med = torch.full((nt, 256), -1, dtype=torch.int64, device=dev)     # list position of the median contributor
        med_amb = torch.zeros(nt, 256, dtype=torch.bool, device=dev)
        last = torch.zeros(nt, 256, dtype=torch.int64, device=dev)
        overflow = torch.zeros(nt, 256, dtype=torch.bool, device=dev)
        tq = None
        if trace is not None:
            ty_, tx_ = trace
            tq = ((tiles == (ty_ // 16) * gx + tx_ // 16).nonzero().flatten(), (ty_ % 16) * 16 + tx_ % 16)
            if tq[0].numel() == 0:
                tq = None
            else:
                tr = dict(used=[], used_centre=[], used_corner_only=[], ids=[], amb=[], pt_id=[], pt_pos=[], pt_alpha=[])

        for b0 in range(0, L, BLOCK):
            B = min(BLOCK, L - b0)
            pos = b0 + torch.arange(B, device=dev)                                   # list position in the tile
            valid_l = pos[None, :] < n[:, None]                                      # [nt,B]
            ids = it.point_list[(start[:, None] + pos).clamp(max=max(it.point_list.numel() - 1, 0))] if it.point_list.numel() else \
                torch.zeros(nt, B, dtype=torch.long, device=dev)
            ids = torch.where(valid_l, ids, torch.zeros_like(ids))
            g = lambda a: a[ids][:, None, None, :]                                   # [nt,1,1,B]  # noqa: E731
            mx, my = g(it.means2D[:, 0]), g(it.means2D[:, 1])
            A, Bc, C, o = (g(it.conic_opacity[:, k]) for k in range(4))
            tc, rx, ry = g(it.ts), g(it.ray_planes[:, 0]), g(it.ray_planes[:, 1])
            d1x = mx - (px[:, :, None, None] + 0.5)
            d1y = my - (py[:, :, None, None] + 0.5)
            dx, dy = d1x - offx, d1y - offy                                          # [nt,256,5,B]
            edx, edy = U * (d1x.abs() + dx.abs()), U * (d1y.abs() + dy.abs())
            t1, t2, t3 = A * dx * dx, C * dy * dy, Bc * dx * dy
            power = -0.5 * (t1 + t2) - t3
            e_pow = K_POWER * U * (0.5 * t1.abs() + 0.5 * t2.abs() + t3.abs()) + \
                (A * dx).abs() * edx + (Bc * dy).abs() * edx + (C * dy).abs() * edy + (Bc * dx).abs() * edy
            alpha = (o * torch.exp(power.clamp(max=80.0))).clamp(max=ALPHA_MAX)
            a_lo = (o * torch.exp((power - e_pow).clamp(max=80.0)) * (1 - K_EXPF * U)).clamp(max=ALPHA_MAX)
            a_hi = (o * torch.exp((power + e_pow).clamp(max=80.0)) * (1 + K_EXPF * U)).clamp(max=ALPHA_MAX)
            e_alpha = torch.maximum(a_hi - alpha, alpha - a_lo)
            depth = tc + (rx * dx + ry * dy)
            dabs = tc.abs() + (rx * dx).abs() + (ry * dy).abs()
            e_depth = 3 * U * dabs + rx.abs() * edx + ry.abs() * edy
            valid = valid_l[:, None, None, :] & ~stopped[:, :, None, None]
            cand = valid & (power <= 0) & (alpha >= ALPHA_MIN)
            certain_out = (power - e_pow > 0) | (a_hi < ALPHA_MIN)
            possible_all = valid_l[:, None, None, :] & inside[:, :, None, None] & ~certain_out   # also past the fp64 stop
            possible = valid & ~certain_out
            amb_c = possible & ((power.abs() <= e_pow) | ((a_lo < ALPHA_MIN) & (a_hi >= ALPHA_MIN)))
            f = 1 - alpha
            # speculate and repair: the skip recurrence of each sample
            take = cand.clone()
            posb = torch.arange(B, device=dev).expand_as(take)
            while True:
                Tb = T[..., None] * _excl_cumprod(torch.where(take, f, torch.ones_like(f)))
                fail = take & (Tb * f < T_STOP)
                if not bool(fail.any()):
                    break
                fst = _first(fail, posb, B)
                has = fst < B
                Ts = torch.gather(Tb, -1, fst.clamp(max=B - 1)[..., None]).squeeze(-1)
                dead = has & (Ts * (1 - ALPHA_MIN) < T_STOP)
                clear = has[..., None] & ((posb == fst[..., None]) | (dead[..., None] & (posb >= fst[..., None])))
                take = take & ~clear
            # the 2048-entry stop: the pixel ends after its MAX_CONTRIB-th used entry
            used = take.any(2)                                                        # [nt,256,B]
            cum = n_used[..., None] + torch.cumsum(used.long(), -1)
            hit = used & (cum >= MAX_CONTRIB)
            stop_at = _first(hit, posb[:, :, 0, :], B)                                # [nt,256]
            keep = posb[:, :, 0, :] <= stop_at[..., None]
            take = take & keep[:, :, None, :]
            used = used & keep
            Tb = T[..., None] * _excl_cumprod(torch.where(take, f, torch.ones_like(f)))
            inc = torch.where(take, e_alpha / f + 2 * U, torch.zeros_like(f))
            eTb = eT[..., None] + torch.cumsum(inc, -1) - inc
            # ambiguous decisions among the positions the pixel reaches
            reach = valid & keep[:, :, None, :]
            test_T = Tb * f
            rel = (Tb * (1 - a_lo) * (1 + eTb + e_alpha / f.clamp(min=1e-300) + 2 * U) >= T_STOP)   # the T test could pass
            amb_t = reach & (cand | amb_c) & ((test_T - T_STOP).abs() <= (eTb + e_alpha / f + 2 * U) * test_T)
            amb_m = take[:, :, 0, :] & ((Tb[:, :, 0, :] - T_MEDIAN).abs() <= eTb[:, :, 0, :] * Tb[:, :, 0, :] + 1e-300)
            amb_here = (amb_c & reach & rel).any(2) | amb_t.any(2) | amb_m
            fa = _first(amb_here, pos.expand(nt, 256, B), 1 << 40)
            newamb = (fa < first_amb) & (first_amb == (1 << 40))
            T_fa = torch.gather(Tb[:, :, 0, :], -1, (fa - b0).clamp(0, B - 1)[..., None]).squeeze(-1)
            T_a = torch.where(newamb, T_fa, T_a)
            first_amb = torch.minimum(first_amb, fa)
            med_amb = med_amb | amb_m.any(-1)
            # centre accumulations
            t0 = take[:, :, 0, :]
            w = torch.where(t0, alpha[:, :, 0, :] * Tb[:, :, 0, :], torch.zeros_like(Tb[:, :, 0, :]))
            r_w = eTb[:, :, 0, :] + e_alpha[:, :, 0, :] / alpha[:, :, 0, :].clamp(min=ALPHA_MIN)
            dep0, dabs0, edep0 = depth[:, :, 0, :], dabs[:, :, 0, :], e_depth[:, :, 0, :]
            for k, (val, vabs) in (("c0", (g(it.rgb[:, 0])[:, :, 0, :], None)), ("c1", (g(it.rgb[:, 1])[:, :, 0, :], None)),
                                   ("c2", (g(it.rgb[:, 2])[:, :, 0, :], None)), ("d", (dep0, dabs0)), ("a", (None, None))):
                if val is None:
                    val = torch.ones_like(w)
                val = val.expand_as(w)
                va = val.abs() if vabs is None else vabs
                acc[k] += (w * val).sum(-1)
                accb[k] += (w * val.abs() * r_w).sum(-1) + (w * edep0).sum(-1) * (k == "d")
                accm[k] += (w * va).sum(-1)
            n0 += t0.sum(-1)
            vmax = torch.maximum(vmax, torch.where(possible[:, :, 0, :], dabs0 + g(it.rgb.abs().amax(1))[:, :, 0, :] + 1, torch.zeros_like(w)).amax(-1))
            # maximum depth over every sample
            dm = torch.where(take, depth, torch.full_like(depth, -float("inf")))
            dmax = dm.amax((-1, -2))
            bmx = torch.where(take, e_depth, torch.zeros_like(depth)).amax((-1, -2))
            cmax = torch.maximum(cmax, dmax)
            b_cmax = torch.maximum(b_cmax, bmx)
            # median contributor: last centre entry taken with T > 0.5
            mpos = torch.where(t0 & (Tb[:, :, 0, :] > T_MEDIAN), pos.expand(nt, 256, B), torch.full_like(posb[:, :, 0, :], -1)).amax(-1)
            med = torch.maximum(med, mpos)
            last = torch.maximum(last, torch.where(used, pos + 1, torch.zeros_like(pos)).amax(-1))
            # phase B for the chunk's points: the sure set and the possible set of their pixel's entries in this block
            amb_sofar = pos.expand(nt, 256, B) >= first_amb[..., None]
            sure = used & ~amb_sofar
            maybe = used | (amb_sofar & possible_all.any(2))
            if trace is not None and tq is not None:
                ti, li = tq
                tr["used"].append(used[ti, li].flatten().cpu())
                tr["used_centre"].append(t0[ti, li].flatten().cpu())
                tr["used_corner_only"].append((used & ~t0)[ti, li].flatten().cpu())
                tr["ids"].append(ids[ti].flatten().cpu())
                tr["amb"].append(amb_here[ti, li].flatten().cpu())
            for c0 in range(0, pts.numel(), POINT_CHUNK):
                q = pts[c0:c0 + POINT_CHUNK]
                qt, ql = p_t[c0:c0 + POINT_CHUNK], p_l[c0:c0 + POINT_CHUNK]
                um = maybe[qt, ql]
                if not bool(um.any()):
                    continue
                us = sure[qt, ql]
                u64 = used[qt, ql]
                gid = ids[qt]                                                         # [np,B]
                qx, qy = cg[q, 0:1], cg[q, 1:2]
                qd, eqd = pr["qd"][q, None], pr["e_qd"][q, None]
                pdx, pdy = it.means2D[gid, 0] - qx, it.means2D[gid, 1] - qy
                epx, epy = U * pdx.abs(), U * pdy.abs()
                ptc, prx, pry = it.ts[gid], it.ray_planes[gid, 0], it.ray_planes[gid, 1]
                pdep = ptc + (prx * pdx + pry * pdy)
                epd = 3 * U * (ptc.abs() + (prx * pdx).abs() + (pry * pdy).abs()) + prx.abs() * epx + pry.abs() * epy
                cd = cond[gid]
                mn = torch.minimum(qd.expand_as(pdep), pdep)
                dz = torch.where(cd, ptc - mn, ptc)
                edz = torch.where(cd, torch.maximum(eqd.expand_as(epd), epd) + U * dz.abs(), torch.zeros_like(dz))
                skip = ~cd & (qd < pdep)
                amb_skip = ~cd & ((qd - pdep).abs() <= eqd + epd)
                Mg, bMg = M[gid], bM[gid]                                             # [np,B,6]
                d = (pdx, pdy, dz)
                e = (epx, epy, edz)
                idx = ((0, 1, 2), (1, 3, 4), (2, 4, 5))
                quad = torch.zeros_like(pdx)
                emag = torch.zeros_like(pdx)
                for a_ in range(3):
                    for b_ in range(3):
                        m, bm = Mg[..., idx[a_][b_]], bMg[..., idx[a_][b_]]
                        quad = quad + d[a_] * m * d[b_]
                        da, db = d[a_].abs(), d[b_].abs()
                        emag = emag + K_POW3 * U * m.abs() * da * db + bm * da * db + (m.abs() + bm) * (da * e[b_] + e[a_] * db + e[a_] * e[b_])
                pw = -0.5 * quad
                epw = 0.5 * emag
                po = it.conic_opacity[gid, 3]
                al = (po * torch.exp(pw.clamp(max=80.0))).clamp(max=ALPHA_MAX)
                al_lo = (po * torch.exp((pw - epw).clamp(max=80.0)) * (1 - K_EXPF * U)).clamp(max=ALPHA_MAX)
                al_hi = (po * torch.exp((pw + epw).clamp(max=80.0)) * (1 + K_EXPF * U)).clamp(max=ALPHA_MAX)
                in64 = u64 & ~skip & (al >= ALPHA_MIN)
                insure = us & ~skip & ~amb_skip & (al_lo >= ALPHA_MIN)
                inmaybe = um & (~skip | amb_skip) & (al_hi >= ALPHA_MIN)
                logT64[q] += torch.where(in64, torch.log1p(-al), torch.zeros_like(al)).sum(-1)
                logT_hi[q] += torch.where(insure, torch.log1p(-al_lo), torch.zeros_like(al)).sum(-1)
                logT_lo[q] += torch.where(inmaybe, torch.log1p(-al_hi), torch.zeros_like(al)).sum(-1)
                n_pt[q] += inmaybe.sum(-1).double()
                if tq is not None:
                    mine = (qt == tq[0][0]) & (ql == tq[1])
                    k_, j_ = torch.nonzero(in64 & mine[:, None], as_tuple=True)
                    tr["pt_id"].append(q[k_].cpu())
                    tr["pt_pos"].append((b0 + j_).cpu())
                    tr["pt_alpha"].append(al[k_, j_].cpu())
            n_used = n_used + used.sum(-1)
            ov = stop_at < B
            overflow = overflow | ov
            stopped = stopped | ov
            T = Tb[..., -1] * torch.where(take[..., -1], f[..., -1], torch.ones_like(f[..., -1]))
            eT = eTb[..., -1] + inc[..., -1]

        # ---- pixel outputs
        amb = first_amb < (1 << 40)
        T0 = T[:, :, 0]
        n0f = n0
        bg = it.bg
        inf = torch.full_like(T0, float("inf"))
        for ch in range(3):
            k = f"c{ch}"
            val = acc[k] + T0 * float(bg[ch])
            bb = accb[k] + kap * (n0f + 2) * (accm[k] + T0 * abs(float(bg[ch]))) + T0 * abs(float(bg[ch])) * eT[:, :, 0]
            al = 2 * T_a * torch.maximum(vmax, torch.full_like(vmax, abs(float(bg[ch]))))
            _put(res, bnd, f"color{ch}", pix, inside, val, bb + torch.where(amb, al, torch.zeros_like(al)))
        _put(res, bnd, "color3", pix, inside, acc["d"], accb["d"] + kap * (n0f + 2) * accm["d"] + torch.where(amb, 2 * T_a * vmax, torch.zeros_like(vmax)))
        _put(res, bnd, "color7", pix, inside, acc["a"], accb["a"] + kap * (n0f + 2) * accm["a"] + torch.where(amb, 2 * T_a, torch.zeros_like(vmax)))
        _put(res, bnd, "color6", pix, inside, cmax, torch.where(amb, inf, b_cmax))
        # median depth and the mid-plane of the SDF
        mid = _median_state(it, start, med)
        mdx, mdy = mid["mx"] - (px + 0.5), mid["my"] - (py + 0.5)
        cmed = mid["ts"] + (mid["rx"] * mdx + mid["ry"] * mdy)
        b_med = 3 * U * (mid["ts"].abs() + (mid["rx"] * mdx).abs() + (mid["ry"] * mdy).abs()) + U * (mid["rx"].abs() * mdx.abs() + mid["ry"].abs() * mdy.abs())
        # an ambiguous decision while the centre transmittance is still above 0.5 may move the median
        med_bad = (amb & (T_a >= T_MEDIAN * (1 - 1e-5))) | med_amb
        _put(res, bnd, "color4", pix, inside, cmed, torch.where(med_bad, inf, b_med))
        n_used_px[pix[inside]] = n_used[inside]
        last_px[pix[inside]] = last[inside]
        over_px[pix[inside]] = overflow[inside]
        amb_px[pix[inside]] = amb[inside]
        if pts.numel():
            qx, qy = cg[pts, 0], cg[pts, 1]
            qd, eqd = pr["qd"][pts], pr["e_qd"][pts]
            m_ = {k: v[p_t, p_l] for k, v in mid.items()}
            sdx, sdy = m_["mx"] - qx, m_["my"] - qy
            pl_ = m_["ts"] + (m_["rx"] * sdx + m_["ry"] * sdy)
            sdf[pts] = pl_ - qd
            bs = 3 * U * (m_["ts"].abs() + (m_["rx"] * sdx).abs() + (m_["ry"] * sdy).abs()) + U * (m_["rx"].abs() * sdx.abs() + m_["ry"].abs() * sdy.abs()) \
                + eqd + U * (pl_ - qd).abs()
            bad = med_bad[p_t, p_l]
            b_sdf[pts] = torch.where(bad, torch.full_like(bs, float("inf")), bs)
            pt_amb[pts] = pt_amb[pts] | amb[p_t, p_l]
        if tr is not None and tq is not None:
            tr = {k: (torch.cat(v) if v else torch.zeros(0)) if isinstance(v, list) else v for k, v in tr.items()}
            tr.update(median=int(med[tq[0], tq[1]]), last=int(last[tq[0], tq[1]]))
            tq = None

    alpha64 = -torch.expm1(logT64)
    lo = -torch.expm1(logT_hi)
    hi = -torch.expm1(logT_lo)
    slack = kap * (n_pt + 2) * hi
    shp = lambda v: v.view(H, W)  # noqa: E731
    out = {k: shp(v) for k, v in res.items()}
    out.update({"b_" + k: shp(v) for k, v in bnd.items()})
    out.update(n_used=shp(n_used_px), last=shp(last_px), overflow=shp(over_px), ambiguous=shp(amb_px), overflow_count=int(over_px.sum()),
               alpha=alpha64, alpha_lo=lo - slack, alpha_hi=hi + slack, sdf=sdf, b_sdf=b_sdf, point_ambiguous=pt_amb, proj=pr, invray=inv,
               in_given=ing, coord_given=cg, pixel=qpix, trace=tr)
    return out


def _put(res, bnd, key, pix, inside, val, b):
    res[key][pix[inside]] = val[inside]
    bnd[key][pix[inside]] = b[inside]


def _median_state(it: Integrate, start, med):
    """(ts, ray plane, mean2D) of each pixel's median entry; zeros where there is none (the kernel's initial values)."""
    has = med >= 0
    gid = it.point_list[(start[:, None] + med.clamp(min=0)).clamp(max=max(it.point_list.numel() - 1, 0))] if it.point_list.numel() else torch.zeros_like(med)
    z = lambda v: torch.where(has, v[gid], torch.zeros_like(v[gid]))  # noqa: E731
    return dict(ts=z(it.ts), rx=z(it.ray_planes[:, 0]), ry=z(it.ray_planes[:, 1]), mx=z(it.means2D[:, 0]), my=z(it.means2D[:, 1]))


# ---- the check ------------------------------------------------------------------------------------------------------------

def culled(alpha, color_int, coord, sdf):
    """The fill values of a point the kernel did not place in the image."""
    a, c, q, s = (_np64(x) for x in (alpha, color_int, coord, sdf))
    return (a == 1.0) & (c.reshape(-1, 3) == 0).all(1) & (q.reshape(-1, 2) == 0).all(1) & (s == -1000.0)


def check(ref: dict, given: dict, it: Integrate, name="", max_report=8) -> dict:
    """`given`: color [9,H,W], alpha_integrated [PN], color_integrated [PN,3], point_coordinate [PN,2], point_sdf [PN] and
    optionally overflow_count.  Raises AssertionError naming the pixels and points out of bound; returns the worst
    error/bound ratio per output and the ambiguous fractions."""
    H, W = it.H, it.W
    errors, stats = [], {}
    color = _np64(given["color"]).reshape(9, H, W)
    amb = ref["ambiguous"].cpu().numpy()
    stats["ambiguous_pixels"] = float(amb.mean()) if amb.size else 0.0
    for ch in (0, 1, 2, 3, 4, 6, 7):
        r, b = ref[f"color{ch}"].cpu().numpy(), ref[f"b_color{ch}"].cpu().numpy()
        d = np.abs(color[ch] - r)
        rt = np.where(np.isinf(b), 0.0, _ratio(d, b))
        rt = np.where(np.isnan(color[ch]), np.inf, rt)
        stats[f"color[{ch}]"] = float(rt.max()) if rt.size else 0.0
        bad = np.argwhere(rt > 1)
        for y, x in bad[:max_report]:
            errors.append(f"{name}: color[{ch}] at pixel (y={y}, x={x}): {color[ch, y, x]!r} vs fp64 {r[y, x]!r}, bound {b[y, x]:.3e}"
                          f"{' (ambiguous pixel)' if amb[y, x] else ''}")
        if len(bad) > max_report:
            errors.append(f"{name}: color[{ch}]: {len(bad)} pixels out of bound")
    if color[5].any():
        y, x = np.argwhere(color[5] != 0)[0]
        errors.append(f"{name}: color[5] at pixel (y={y}, x={x}) is {color[5, y, x]!r}, must be 0")
    alpha, cint, coord, sdf = (_np64(given[k]) for k in ("alpha_integrated", "color_integrated", "point_coordinate", "point_sdf"))
    cint, coord = cint.reshape(-1, 3), coord.reshape(-1, 2)
    ing = ref["in_given"].cpu().numpy()
    pr = {k: v.cpu().numpy() for k, v in ref["proj"].items()}
    pamb = pr["ambiguous"]
    # in-image decisions and coordinates against the fp64 projection
    bad = np.nonzero((ing != pr["inside"]) & ~pamb)[0]
    for i in bad[:max_report]:
        errors.append(f"{name}: point {i}: {'placed in' if ing[i] else 'culled from'} the image, the fp64 projection "
                      f"({pr['imx'][i]!r}, {pr['imy'][i]!r}) at view z {pr['vz'][i]!r} says otherwise")
    if len(bad) > max_report:
        errors.append(f"{name}: {len(bad)} points with the wrong in-image decision")
    dq = np.abs(coord - np.stack([pr["imx"], pr["imy"]], 1))
    bq = np.stack([pr["e_imx"], pr["e_imy"]], 1)
    rq = np.where(ing[:, None], _ratio(dq, bq), 0.0)
    stats["point_coordinate"] = float(rq.max()) if rq.size else 0.0
    for i in np.nonzero((rq > 1).any(1))[0][:max_report]:
        errors.append(f"{name}: point {i}: coordinate {tuple(coord[i])} vs fp64 ({pr['imx'][i]!r}, {pr['imy'][i]!r}), bound {tuple(bq[i])}")
    # culled points: the fill values exactly
    cul = ~ing
    notfill = cul & ~culled(alpha, cint, coord, sdf)
    for i in np.nonzero(notfill)[0][:max_report]:
        errors.append(f"{name}: culled point {i}: ({alpha[i]!r}, {tuple(cint[i])}, {tuple(coord[i])}, {sdf[i]!r}) instead of (1, 0, 0, -1000)")
    # points per pixel: exactly the points the kernel placed there
    pix = ref["pixel"].cpu().numpy()
    cnt = np.bincount(pix[ing], minlength=H * W).reshape(H, W) if ing.any() else np.zeros((H, W))
    badc = np.argwhere(color[8] != cnt)
    for y, x in badc[:max_report]:
        errors.append(f"{name}: color[8] at pixel (y={y}, x={x}) is {color[8, y, x]!r}, {cnt[y, x]} points report that pixel")
    # color_integrated: the kernel's own channels 0-2 at the point's pixel, bit for bit
    if ing.any():
        ci = np.stack([color[ch].reshape(-1)[pix[ing]] for ch in range(3)], 1)
        badi = np.nonzero((ci != cint[ing]).any(1))[0]
        for j in badi[:max_report]:
            i = np.nonzero(ing)[0][j]
            errors.append(f"{name}: point {i}: color_integrated {tuple(cint[i])} differs from color[0:3] {tuple(ci[j])} at its pixel {divmod(pix[i], W)}")
    # alpha envelope and SDF bound of every in-image point
    lo, hi, a64 = (ref[k].cpu().numpy() for k in ("alpha_lo", "alpha_hi", "alpha"))
    out = ing & ((alpha < lo) | (alpha > hi) | np.isnan(alpha))
    width = np.maximum(hi - a64, a64 - lo)
    ra = np.where(ing, _ratio(np.abs(alpha - a64), np.where(width > 0, width, 1e-300)), 0.0)
    stats["alpha_integrated"] = float(ra.max()) if ra.size else 0.0
    for i in np.nonzero(out)[0][:max_report]:
        y, x = divmod(int(pix[i]), W)
        errors.append(f"{name}: point {i} (pixel y={y}, x={x}): alpha_integrated {alpha[i]!r} outside [{lo[i]!r}, {hi[i]!r}] (fp64 {a64[i]!r})"
                      f"{' (ambiguous point)' if ref['point_ambiguous'][i] else ''}")
    if out.sum() > max_report:
        errors.append(f"{name}: {int(out.sum())} points outside their alpha envelope")
    s64, bs = ref["sdf"].cpu().numpy(), ref["b_sdf"].cpu().numpy()
    rs = np.where(ing & np.isfinite(bs), _ratio(np.abs(sdf - s64), bs), 0.0)
    rs = np.where(ing & np.isnan(sdf), np.inf, rs)
    stats["point_sdf"] = float(rs.max()) if rs.size else 0.0
    for i in np.nonzero(rs > 1)[0][:max_report]:
        y, x = divmod(int(pix[i]), W)
        errors.append(f"{name}: point {i} (pixel y={y}, x={x}): point_sdf {sdf[i]!r} vs fp64 {s64[i]!r}, bound {bs[i]:.3e}")
    if (rs > 1).sum() > max_report:
        errors.append(f"{name}: {int((rs > 1).sum())} points with point_sdf out of bound")
    if "overflow_count" in given and given["overflow_count"] is not None:
        n_amb_over = int((ref["overflow"].cpu().numpy() & amb).sum())
        n = int(given["overflow_count"])
        if not (ref["overflow_count"] - n_amb_over <= n <= ref["overflow_count"] + int(amb.sum())):
            errors.append(f"{name}: {n} pixels met the contributor cap, the fp64 model counts {ref['overflow_count']}")
        stats["overflow_count"] = n
    ptamb = ref["point_ambiguous"].cpu().numpy()
    stats["ambiguous_points"] = float(ptamb[ing].mean()) if ing.any() else 0.0
    if errors:
        raise AssertionError("\n".join(errors))
    return stats
