"""fp64 evaluation of the tile alpha blend (forward and backward) with per-element bounds on what an fp32 evaluation may differ by.

The blend kernels (csrc/rgs_render_fwd.cu, csrc/rgs_render_bwd.cu), the CPU oracle (oracle/oracle.c) and the reference build
all evaluate the same per-pixel recurrence in fp32 (reference: forward.cu:428-693, backward.cu:631-1016).  This module evaluates
it in fp64 from the same fp32 per-Gaussian records, and carries alongside every value a rigorous bound on how far an fp32
evaluation of the same expression can land from it.  So a checker needs no outlier budget: every pixel and every accumulator
row must be within its own bound, and n_contrib must be exact wherever no decision is ambiguous.

Decisions.  Four comparisons steer the recurrence: `power > 0`, `alpha < 1/255`, `test_T < 1e-4` and `T > 0.5` (the median
contributor).  Each is evaluated in fp64 and classified *ambiguous* when the fp32 value's error bound straddles the threshold.
A pixel is ambiguous when an ambiguous decision occurs at or before its fp64 stop; such pixels are not held to exact n_contrib,
and their maps get the allowance of everything from the first ambiguous decision on (see `forward`).

Everything is torch, so the same code runs on the CPU (host tests) and on the GPU (tile-chunked, lists padded per chunk).
It reads plain arrays only: this build's decoded buffers (rawapi.ours_views), the oracle's state, or a fixture's `st_*` arrays.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

U = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)


def _f32(x):
    return float(np.float32(x))


ALPHA_MIN = _f32(1.0 / 255.0)   # 1.0f / 255.0f as the kernels compare it
ALPHA_MAX = _f32(0.99)          # min(0.99f, ...)
T_STOP = _f32(0.0001)           # test_T < 0.0001f
T_MEDIAN = 0.5                  # T > 0.5 (a double literal: the fp32 T is compared exactly)
NLEN_MIN = _f32(1.0e-12)        # normal renormalisation floor

# power = -0.5 (A dx dx + C dy dy) - B dx dy in fp32: dx, dy are rounded once (centre - pixel), each product chain adds at most two
# roundings, the two sums one each: every term carries at most 6u of its own magnitude; 8u leaves room for second-order terms.
K_POWER = 8.0
# expf is within 2 ulp of exp (CUDA C++ Programming Guide, single-precision mathematical functions; glibc is within 1 ulp):
# at most 4u relative.  One more rounding for o * G.
K_EXPF = 5.0
# Forward maps: a recursive fp32 sum of n terms errs by at most (n-1)u of the sum of |terms|, each term (value x alpha x T, the
# value itself a 3-term plane evaluation) carries a few more roundings; the divisions and the square root of the normalised maps
# a few more.  4 covers (n + 2) per sum with a margin of ~2 for the per-term roundings.
KAPPA_FWD = 4.0
# Backward rows: each pair term is a product chain of up to ~8 roundings on top of the fp32 running sum B (one rounding per layer
# behind), the warp reduction adds 5 levels and the float atomics one rounding per partial (at most one per pair).  8 covers
# (n_behind + n_row + 16) per term with a margin of 2.
KAPPA_BWD = 8.0

# At most this fraction of a scene's pixels may be ambiguous (not held to exact n_contrib).  Needles without a kernel filter
# (scale ratios up to 1e4, conic entries ~1e6 with B^2 ~ A C) are the worst family at 9.2e-2 on an H100; every other family,
# C1 included, stays below 1e-3.
AMBIGUOUS_CEILING = 0.12

PAIR_BUDGET = {"cpu": 1 << 21, "cuda": 1 << 23}  # (pixel, list entry) pairs evaluated at once


@dataclass
class Blend:
    """One blend problem: fp32 per-Gaussian records, the sorted tile lists and the camera constants."""
    means2D: torch.Tensor        # [P,2]
    conic_opacity: torch.Tensor  # [P,4] (A, B, C, opacity)
    rgb: torch.Tensor            # [P,3]
    ts: torch.Tensor | None      # [P]
    ray_planes: torch.Tensor | None     # [P,2]
    normals: torch.Tensor | None        # [P,3]
    camera_planes: torch.Tensor | None  # [P,6] reference layout: (x row: dx, dy), (y row), (z row)
    view_points: torch.Tensor | None    # [P,3]
    ranges: torch.Tensor         # [tiles,2]
    point_list: torch.Tensor     # [R]
    bg: torch.Tensor             # [3]
    W: int
    H: int
    focal_x: float               # fp32 values, as the kernels compute them: W / (2.0f * tan_fovx)
    focal_y: float
    coord: bool
    depth: bool

    @property
    def geo(self):
        return self.coord or self.depth

    @property
    def device(self):
        return self.means2D.device


def focal(size, tan_fov):
    return _f32(np.float32(size) / (np.float32(2.0) * np.float32(tan_fov)))


def make_blend(st: dict, W, H, tanfovx, tanfovy, bg, coord, depth, device="cpu") -> Blend:
    """Blend from a dict of plain arrays named as oracle.preprocess / rawapi.ours_views / a fixture's `st_*` entries."""
    def t(k, required=True):
        v = st.get(k)
        if v is None:
            assert not required, k
            return None
        v = torch.as_tensor(np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v)).to(device)
        return v.to(torch.float64) if v.is_floating_point() else v.to(torch.int64)
    geo = coord or depth
    ranges = t("ranges")
    return Blend(t("means2D"), t("conic_opacity"), t("rgb"), t("ts", geo), t("ray_planes", geo), t("normals", geo),
                 t("camera_planes", coord), t("view_points", coord), ranges.reshape(-1, 2), t("point_list").reshape(-1),
                 torch.as_tensor(np.asarray(bg, np.float32)).to(device, torch.float64), int(W), int(H),
                 focal(W, tanfovx), focal(H, tanfovy), bool(coord), bool(depth))


# ---- tile-chunked pair evaluation ------------------------------------------------------------------------------------

def _chunks(bl: Blend):
    """Tiles grouped so that (tiles x 256 pixels x longest list) stays within the pair budget; lists padded per chunk."""
    n = (bl.ranges[:, 1] - bl.ranges[:, 0]).cpu()
    order = torch.argsort(n, descending=True)
    budget = PAIR_BUDGET["cuda" if bl.device.type == "cuda" else "cpu"]
    i, T = 0, order.numel()
    while i < T:
        L = max(int(n[order[i]]), 1)
        k = max(1, min(T - i, budget // (256 * L)))
        yield order[i:i + k].to(bl.device), L
        i += k


def _pixels(bl: Blend, tiles):
    gx = (bl.W + 15) // 16
    loc = torch.arange(256, device=bl.device)
    px = (tiles % gx)[:, None] * 16 + loc % 16
    py = (tiles // gx)[:, None] * 16 + loc // 16
    inside = (px < bl.W) & (py < bl.H)
    return px, py, inside, py.clamp(max=bl.H - 1) * bl.W + px.clamp(max=bl.W - 1)


def _pairs(bl: Blend, tiles, L, last=None):
    """Per-(pixel, list position) quantities of a chunk, [nt, 256, L], and the fp32-rounding-aware decisions."""
    pos = torch.arange(L, device=bl.device)
    start, n = bl.ranges[tiles, 0], bl.ranges[tiles, 1] - bl.ranges[tiles, 0]
    valid_l = pos[None, :] < n[:, None]                                              # [nt, L]
    ids = bl.point_list[(start[:, None] + pos).clamp(max=max(bl.point_list.numel() - 1, 0))] if bl.point_list.numel() else \
        torch.zeros(tiles.numel(), L, dtype=torch.int64, device=bl.device)
    ids = torch.where(valid_l, ids, torch.zeros_like(ids))
    px, py, inside, pix = _pixels(bl, tiles)
    valid = valid_l[:, None, :] & inside[:, :, None]
    if last is not None:
        valid = valid & (pos[None, None, :] < last[:, :, None])
    e = dict(ids=ids, pos=pos, valid=valid, px=px, py=py, inside=inside, pix=pix)
    g = lambda a: a[ids][:, None]                                                    # [nt, 1, L, ...]
    dx = g(bl.means2D[:, 0]) - px[:, :, None].double()
    dy = g(bl.means2D[:, 1]) - py[:, :, None].double()
    A, B, C, o = (g(bl.conic_opacity[:, k]) for k in range(4))
    t1, t2, t3 = A * dx * dx, C * dy * dy, B * dx * dy
    power = -0.5 * (t1 + t2) - t3
    e_pow = K_POWER * U * (0.5 * t1.abs() + 0.5 * t2.abs() + t3.abs())
    G = torch.exp(power.clamp(max=80.0))  # power > 0 never blends; the clamp keeps o G finite (o = 0 splats with indefinite conics)
    a_raw = o * G
    alpha = a_raw.clamp(max=ALPHA_MAX)
    a_lo = (o * torch.exp((power - e_pow).clamp(max=80.0)) * (1 - K_EXPF * U)).clamp(max=ALPHA_MAX)
    a_hi = (o * torch.exp((power + e_pow).clamp(max=80.0)) * (1 + K_EXPF * U)).clamp(max=ALPHA_MAX)
    contrib = valid & (power <= 0) & (alpha >= ALPHA_MIN)
    certain_out = (power - e_pow > 0) | (a_hi < ALPHA_MIN)
    amb = valid & ~certain_out & ((power.abs() <= e_pow) | ((a_lo < ALPHA_MIN) & (a_hi >= ALPHA_MIN)))
    e.update(dx=dx, dy=dy, A=A, B=B, C=C, o=o, G=G, alpha=alpha, a_hi=a_hi, contrib=contrib, amb=amb,
             e_alpha=torch.maximum(a_hi - alpha, alpha - a_lo),                       # |fp32 alpha - alpha| bound
             r_G=torch.expm1(e_pow.clamp(max=80.0)) + K_EXPF * U)                     # relative bound on fp32 G
    e["g"] = g
    return e


def _plane_values(bl: Blend, e):
    """t = t_centre + ray . d and the camera-plane coordinates, with the magnitudes their fp32 evaluation errs against."""
    g, dx, dy = e["g"], e["dx"], e["dy"]
    out = {}
    if bl.depth:
        a, b = g(bl.ray_planes[:, 0]) * dx, g(bl.ray_planes[:, 1]) * dy
        tc = g(bl.ts)
        out["t"] = (tc + (a + b), tc.abs() + a.abs() + b.abs())
    if bl.coord:
        out["c"] = []
        for ch in range(3):
            vp, a, b = g(bl.view_points[:, ch]), g(bl.camera_planes[:, 2 * ch]) * dx, g(bl.camera_planes[:, 2 * ch + 1]) * dy
            out["c"].append((vp + a + b, vp.abs() + a.abs() + b.abs()))
    return out


def _ln(bl: Blend, px, py):
    pnx = (px.double() - bl.W / 2.0) / bl.focal_x
    pny = (py.double() - bl.H / 2.0) / bl.focal_y
    return torch.sqrt(pnx * pnx + pny * pny + 1)


def _excl_cumprod(f):
    c = torch.cumprod(f, -1)
    return torch.cat([torch.ones_like(c[..., :1]), c[..., :-1]], -1)


def _excl_cumsum(f):
    c = torch.cumsum(f, -1)
    return c - f


MAP_KEYS = ("color", "alpha", "depth", "mdepth", "normal", "coord", "mcoord", "accum_depth", "accum_coord", "normal_length")


# ---- forward ---------------------------------------------------------------------------------------------------------

def forward(bl: Blend) -> dict:
    """fp64 maps ([C,H,W]), n_contrib ([2,H,W], int64), per-element bounds `b_<map>`, ambiguity flags and allowances.

    Bound of an accumulated map value sum_k v_k w_k (w_k = alpha_k T_k, T_k = prod_{j<k} (1 - alpha_j)):
      * sum_k |v_k| w_k r_w,k        -- r_w,k = e_T,k + e_alpha,k / alpha_k is the relative bound on the fp32 weight, where
                                        e_T,k = sum_{j<k} (e_alpha,j / (1 - alpha_j) + 2u) covers the fp32 product for T (one
                                        subtraction and one product per layer) and e_alpha the fp32 alpha (power, expf, o*G);
      * KAPPA_FWD u (n + 2) sum_k |v|_k w_k -- the recursive fp32 sum of n terms and the roundings inside each term, where |v|_k
                                        is the sum of the magnitudes of the value's own terms (t = t_c + r.d, camera planes);
      * the background layer T_final bg with its e_T.
    Normalised maps (depth = accum / weight, normal = N / |N|) propagate these first-order through the division.
    An ambiguous pixel (a flippable decision at or before its fp64 stop, at transmittance T_a) adds the allowance
    2 T_a max|v| to accumulated maps -- whatever is blended from there on weighs T_a in total in either outcome -- and the whole
    value range to the normalised and median maps."""
    H, W, dev = bl.H, bl.W, bl.device
    HW = H * W
    res = {k: torch.zeros(c, HW, dtype=torch.float64, device=dev) for k, c in
           (("color", 3), ("alpha", 1), ("depth", 1), ("mdepth", 1), ("normal", 3), ("coord", 3), ("mcoord", 3), ("accum_depth", 1),
            ("accum_coord", 3), ("normal_length", 1))}
    bnd = {k: torch.zeros_like(v) for k, v in res.items()}
    allow = {k: torch.zeros_like(v) for k, v in res.items()}
    n_contrib = torch.zeros(2, HW, dtype=torch.int64, device=dev)
    ambiguous = torch.zeros(HW, dtype=torch.bool, device=dev)
    kap = KAPPA_FWD * U
    for tiles, L in _chunks(bl):
        e = _pairs(bl, tiles, L)
        pos, inside, pix = e["pos"], e["inside"], e["pix"]
        alpha, contrib = e["alpha"], e["contrib"]
        one_m = 1 - alpha
        T_before = _excl_cumprod(torch.where(contrib, one_m, torch.ones_like(one_m)))
        inc = torch.where(contrib, e["e_alpha"] / one_m + 2 * U, torch.zeros_like(one_m))
        eT = _excl_cumsum(inc)
        test_T = T_before * one_m
        stop_here = contrib & (test_T < T_STOP)
        amb_stop = contrib & ((test_T - T_STOP).abs() <= (eT + e["e_alpha"] / one_m + 2 * U) * test_T)
        stop = torch.where(stop_here, pos, torch.full_like(pos, L)).min(-1).values          # [nt,256]
        upto = pos[None, None, :] <= stop[..., None]
        blended = contrib & (pos[None, None, :] < stop[..., None])
        amb_any = (e["amb"] | amb_stop) & upto
        if bl.geo:
            med_ok = blended & (T_before > T_MEDIAN)
            amb_any = amb_any | (blended & ((T_before - T_MEDIAN).abs() <= eT * T_before + 1e-300))
        last = torch.where(blended, pos + 1, torch.zeros_like(pos)).max(-1).values
        if bl.geo:
            maxc = torch.where(med_ok, pos + 1, torch.zeros_like(pos)).max(-1).values
            maxc = torch.where(maxc > 0, maxc, torch.full_like(maxc, 0xFFFFFFFF))
        else:
            maxc = torch.full_like(last, 0xFFFFFFFF)
        amb_pix = amb_any.any(-1) & inside
        first_amb = torch.where(amb_any, pos, torch.full_like(pos, L)).min(-1).values
        T_a = torch.gather(torch.cat([T_before, T_before[..., -1:] * 0], -1), -1, first_amb[..., None]).squeeze(-1)
        T_a = torch.where(amb_pix, torch.where(first_amb < L, T_a, torch.zeros_like(T_a)), torch.zeros_like(T_a))

        w = torch.where(blended, alpha * T_before, torch.zeros_like(alpha))
        r_w = eT + e["e_alpha"] / alpha.clamp(min=ALPHA_MIN)
        n = blended.sum(-1).double()
        T_fin = torch.where(blended, one_m, torch.ones_like(one_m)).prod(-1)
        eT_fin = inc.mul(blended).sum(-1)
        validmask = e["valid"]

        def acc(v, vabs):
            return (w * v).sum(-1), (w * v.abs() * r_w).sum(-1) + kap * (n + 2) * (w * vabs).sum(-1)

        def vmax(vabs):
            return torch.where(validmask, vabs, torch.zeros_like(vabs)).amax(-1) if L else torch.zeros_like(T_a)

        def put(key, ch, val, b, al):
            sel = inside
            res[key][ch, pix[sel]] = val[sel]
            bnd[key][ch, pix[sel]] = b[sel]
            allow[key][ch, pix[sel]] = torch.where(amb_pix, al, torch.zeros_like(al))[sel]

        g = e["g"]
        for ch in range(3):
            c = g(bl.rgb[:, ch]).expand_as(alpha)
            s, b = acc(c, c.abs())
            bgc = float(bl.bg[ch])
            val = s + T_fin * bgc
            b = b + kap * (n + 2) * T_fin * abs(bgc) + T_fin * abs(bgc) * eT_fin
            put("color", ch, val, b, 2 * T_a * torch.maximum(vmax(c.abs()), torch.full_like(T_a, abs(bgc))))
        weight, b_weight = acc(torch.ones_like(alpha), torch.ones_like(alpha))
        put("alpha", 0, weight, b_weight, 2 * T_a)
        has = last > 0
        wsafe = torch.where(has, weight, torch.ones_like(weight))
        px, py = e["px"], e["py"]
        ln = _ln(bl, px, py)
        planes = _plane_values(bl, e)
        med_sel = (pos[None, None, :] == (maxc - 1)[..., None]) & blended

        def at_median(v):
            return torch.where(med_sel, v, torch.zeros_like(v)).sum(-1)

        if bl.depth:
            t, tabs = planes["t"]
            D, bD = acc(t, tabs)
            ad = D / ln
            b_ad = bD / ln + kap * ad.abs()
            put("accum_depth", 0, ad, b_ad, 2 * T_a * vmax(tabs) / ln)
            dep = torch.where(has, ad / wsafe, torch.zeros_like(ad))
            b_dep = torch.where(has, (b_ad + dep.abs() * b_weight) / wsafe + kap * dep.abs(), torch.zeros_like(ad))
            put("depth", 0, dep, b_dep, 2 * vmax(tabs) / ln)
            md = at_median(t) / ln
            put("mdepth", 0, md, kap * at_median(tabs) / ln + kap * md.abs(), 2 * vmax(tabs) / ln)
        if bl.coord:
            for ch in range(3):
                c, cabs = planes["c"][ch]
                S, bS = acc(c, cabs)
                put("accum_coord", ch, S, bS, 2 * T_a * vmax(cabs))
                co = torch.where(has, S / wsafe, torch.zeros_like(S))
                put("coord", ch, co, torch.where(has, (bS + co.abs() * b_weight) / wsafe + kap * co.abs(), torch.zeros_like(S)), 2 * vmax(cabs))
                mc = at_median(c)
                put("mcoord", ch, mc, kap * at_median(cabs) + kap * mc.abs(), 2 * vmax(cabs))
        if bl.geo:
            N, bN = [], []
            for ch in range(3):
                nv = g(bl.normals[:, ch]).expand_as(alpha)
                s, b = acc(nv, nv.abs())
                N.append(s)
                bN.append(b)
            nlen = torch.sqrt(N[0] ** 2 + N[1] ** 2 + N[2] ** 2)
            b_len = torch.sqrt(bN[0] ** 2 + bN[1] ** 2 + bN[2] ** 2) + kap * nlen
            put("normal_length", 0, torch.where(has, nlen, torch.ones_like(nlen)), torch.where(has, b_len, torch.zeros_like(nlen)),
                2 * T_a * vmax(g(bl.normals.norm(dim=1)).expand_as(alpha)) + (T_a >= 1).double())
            ls = nlen.clamp(min=NLEN_MIN)
            for ch in range(3):
                nv = torch.where(has, N[ch] / ls, torch.zeros_like(ls))
                bn = torch.where(has, bN[ch] / ls + N[ch].abs() * b_len / ls ** 2 + kap * nv.abs(), torch.zeros_like(ls))
                put("normal", ch, nv, bn, torch.full_like(ls, 2.0))
        n_contrib[0, pix[inside]] = last[inside]
        n_contrib[1, pix[inside]] = maxc[inside]
        ambiguous[pix[inside]] = amb_pix[inside]
    shp = lambda v: v.view(v.shape[0], H, W)
    out = {k: shp(v) for k, v in res.items()}
    out.update({"b_" + k: shp(v) for k, v in bnd.items()})
    out.update({"allow_" + k: shp(v) for k, v in allow.items()})
    out["n_contrib"] = n_contrib.view(2, H, W)
    out["ambiguous"] = ambiguous.view(H, W)
    return out


def _np64(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu()
        if x.dtype == torch.int32:
            return x.numpy().view(np.uint32).astype(np.int64)
        return x.double().numpy()
    x = np.asarray(x)
    if x.dtype in (np.int32, np.uint32):
        return x.view(np.uint32).astype(np.int64)
    return x.astype(np.float64)


def _ratio(d, b):
    return np.where(d == 0, 0.0, d / np.where(b > 0, b, 1e-300))


def check_forward(ref: dict, given: dict, bl: Blend, name="", hitmask=None, chunk_base=None, max_report=8) -> dict:
    """Every map in `given` ([C,H,W] or [H,W]) within its bound at every pixel; n_contrib exact on every unambiguous pixel.
    Returns the statistics (worst error/bound per map and channel, ambiguous fraction); raises AssertionError naming the
    pixels otherwise.  With `hitmask` / `chunk_base` (this build's forward ballots) a pair missing from a pixel is reported
    together with whether the ballot culled it."""
    stats, errors = {}, []
    amb = ref["ambiguous"].cpu().numpy()
    stats["ambiguous_frac"] = float(amb.mean()) if amb.size else 0.0
    for k in MAP_KEYS:
        if k not in given:
            continue
        r = ref[k].cpu().numpy()
        a = _np64(given[k]).reshape(r.shape)
        b = (ref["b_" + k] + ref["allow_" + k]).cpu().numpy()
        d = np.abs(a - r)
        rt = _ratio(d, b)
        rt = np.where(np.isnan(a) != np.isnan(r), np.inf, np.nan_to_num(rt, nan=0.0))
        for ch in range(r.shape[0]):
            stats[f"{k}[{ch}]"] = float(rt[ch].max()) if rt[ch].size else 0.0
        bad = np.argwhere(rt > 1)
        for ch, y, x in bad[:max_report]:
            errors.append(f"{name}: {k}[{ch}] at pixel (y={y}, x={x}): {a[ch, y, x]!r} vs fp64 {r[ch, y, x]!r}, bound {b[ch, y, x]:.3e}"
                          f"{' (ambiguous pixel)' if amb[y, x] else ''}")
        if len(bad) > max_report:
            errors.append(f"{name}: {k}: {len(bad)} elements out of bound")
    if "n_contrib" in given:
        nc = _np64(given["n_contrib"]).reshape(2, bl.H, bl.W)
        rn = ref["n_contrib"].cpu().numpy()
        bad = np.argwhere((nc != rn).any(0) & ~amb)
        stats["n_contrib_mismatch"] = int(len(bad))
        for y, x in bad[:max_report]:
            msg = f"{name}: n_contrib at pixel (y={y}, x={x}): {tuple(nc[:, y, x])} vs fp64 {tuple(rn[:, y, x])}"
            msg += explain_pixel(bl, int(y), int(x), int(nc[0, y, x]), hitmask, chunk_base)
            errors.append(msg)
        if len(bad) > max_report:
            errors.append(f"{name}: n_contrib differs on {len(bad)} unambiguous pixels")
    if errors:
        raise AssertionError("\n".join(errors))
    return stats


def explain_pixel(bl: Blend, y, x, given_last, hitmask=None, chunk_base=None) -> str:
    """Which list entries the fp64 blend takes at one pixel, and, at the first entry the given result lacks, the forward ballot."""
    gx = (bl.W + 15) // 16
    tile = torch.tensor([(y // 16) * gx + x // 16], device=bl.device)
    L = int(bl.ranges[tile, 1] - bl.ranges[tile, 0])
    e = _pairs(bl, tile, max(L, 1))
    l = (y % 16) * 16 + x % 16
    contrib = e["contrib"][0, l].cpu().numpy()
    takes = np.nonzero(contrib)[0]
    s = f"; fp64 blends list positions {takes[:6].tolist()}{'...' if len(takes) > 6 else ''} of {L}"
    miss = [p for p in takes if p >= given_last] if given_last < (takes[-1] + 1 if len(takes) else 0) else []
    if hitmask is not None and chunk_base is not None and len(takes):
        warp = ((y % 16) // 4) * 2 + (x % 16) // 8
        p = int(miss[0]) if miss else int(takes[0])
        word = (int(chunk_base[int(tile)]) + p // 32) * 8 + warp
        bit = (int(hitmask[word]) >> (p % 32)) & 1
        s += f"; position {p} (Gaussian {int(e['ids'][0, p])}): forward ballot bit {'set' if bit else 'CLEAR (culled by the box test)'}"
    return s


# ---- backward --------------------------------------------------------------------------------------------------------

SG_KEYS = ("mean2D", "conic", "opacity", "colors", "ts", "camera_planes", "ray_planes", "normals", "view_points")
SG_WIDTH = dict(mean2D=3, conic=4, opacity=1, colors=3, ts=1, camera_planes=6, ray_planes=2, normals=3, view_points=3)


def _pixel_upstream(bl: Blend, state: dict, up: dict):
    """Per-pixel factors of the backward recurrence (backward.cu:704-781) in fp64 from the given fp32 pixel state, each with
    the magnitude its fp32 evaluation errs against (cancellations counted by the sum of |terms|)."""
    dev, H, W = bl.device, bl.H, bl.W
    HW = H * W
    f = lambda v, c: torch.as_tensor(_np64(v)).to(dev).reshape(c, HW)
    w_final = f(state["alpha"], 1)[0]
    nc = f(state["n_contrib"], 2)
    last, maxc = nc[0].long(), nc[1].long()
    gcol = f(up["color"], 3)
    q = dict(last=last, maxc=maxc, w_final=w_final, T_final=1 - w_final, gcol=gcol, gcol_abs=gcol.abs(),
             dalpha=f(up["alpha"], 1)[0].clone())
    q["dalpha_abs"] = q["dalpha"].abs()
    live = (last > 0).double()
    ww = w_final * w_final
    wsafe = torch.where(last > 0, w_final, torch.ones_like(w_final))
    wwsafe = torch.where(last > 0, ww, torch.ones_like(ww))
    gy, gxx = torch.div(torch.arange(HW, device=dev), W, rounding_mode="floor"), torch.arange(HW, device=dev) % W
    if bl.coord:
        gc, acc_c = f(up["coord"], 3), f(state["accum_coord"], 3)
        q["dalpha"] = q["dalpha"] - (gc * acc_c).sum(0) / wwsafe
        q["dalpha_abs"] = q["dalpha_abs"] + (gc * acc_c).abs().sum(0) / wwsafe
        q["dpc"], q["dpmc"] = gc / wsafe, f(up["mcoord"], 3)
    if bl.depth:
        ln = _ln(bl, gxx, gy)
        gd, acc_d = f(up["depth"], 1)[0], f(state["accum_depth"], 1)[0]
        q["dalpha"] = q["dalpha"] - gd * acc_d / wwsafe
        q["dalpha_abs"] = q["dalpha_abs"] + (gd * acc_d).abs() / wwsafe
        q["dpt"], q["dpmt"] = gd / wsafe / ln, f(up["mdepth"], 1)[0] / ln
    if bl.geo:
        gn, nn, nlen = f(up["normal"], 3), f(state["normal"], 3), f(state["normal_length"], 1)[0]
        # normal renormalisation (backward.cu:760-775): below the 1e-12 floor the reference divides by the floor and drops the
        # projection; otherwise (g - (g.n) n) / |N|
        d = (gn * nn).sum(0)
        small = nlen < NLEN_MIN
        q["dpn"] = torch.where(small, gn / NLEN_MIN, (gn - d * nn) / torch.where(small, torch.ones_like(nlen), nlen))
        q["dpn_abs"] = torch.where(small, gn.abs() / NLEN_MIN, (gn.abs() + (gn * nn).abs().sum(0) * nn.abs()) / torch.where(small, torch.ones_like(nlen), nlen))
    # pixels nothing was blended into (last_contributor == 0) contribute nothing: every pair fails `contributor < last`
    for k in ("dalpha", "dalpha_abs", "dpt", "dpmt"):
        if k in q:
            q[k] = q[k] * live
    for k in ("dpc", "dpmc", "dpn", "dpn_abs", "gcol", "gcol_abs"):
        if k in q:
            q[k] = q[k] * live
    bg = bl.bg.view(3, 1)
    q["bg_dot"] = (bg * q["gcol"]).sum(0)
    q["bg_abs"] = (bg.abs() * q["gcol_abs"]).sum(0)
    return q


def backward(bl: Blend, state: dict, up: dict, clamp_keeps_gradient: bool = True) -> dict:
    """fp64 screen-space rows in the oracle's `orc_sgrad` units (mean2D incl. the |.| densification channel, conic (A, B, -, C),
    opacity, colours, t, camera planes, ray planes, normals, view points), each with a bound `b_<key>`.

    `state` is the forward pixel state being differentiated (alpha, n_contrib, normal, accum_depth, accum_coord, normal_length):
    for a kernel under test its own, so that this check isolates the backward kernel.  T is recovered exactly (fp64 division)
    from the given T_final = 1 - alpha.  Semantics restated from backward.cu:631-1016:
      * the 0.99 clamp keeps its unclamped gradient: dL/dG = o dL/dalpha whether or not o G was clamped;
      * the median-contributor terms (mcoord, mdepth) go to list position max_contributor - 1 only;
      * the normal renormalisation as in `_pixel_upstream`, including the |N| < 1e-12 branch;
      * pixels with last_contributor == 0 contribute nothing, and only list positions < last_contributor are visited.
    dL/dalpha_k is written T_k S_k - B_k / (1 - alpha_k), with S_k = sum_ch c_ch g_ch (alpha channel c = 1) and B_k the sum of
    w_j S_j over the layers behind plus T_final bg.g -- algebraically the reference's accum_rec form.

    Bound of row r, channel c, over the pairs k that reach it (M_k = the pair term evaluated on magnitudes: |.| of every factor,
    and T_k S_abs + B_abs / (1 - alpha_k) for dL/dalpha, i.e. the T S - B/(1 - alpha) cancellation counted in full):
      * KAPPA_BWD u (n_behind,k + n_row + 16) M_k -- roundings inside the term, the fp32 running sum B over the n_behind layers,
        the warp reduction and the float atomics over the n_row pairs of the row;
      * r_k M_k with r_k = e_T,k + e_alpha,k (1/alpha_k + 1/(1 - alpha_k)) + r_G,k: e_T,k = u + sum over the layers at or
        behind k of (e_alpha / (1 - alpha) + 3u) is the error growth of T recovered by division (the reciprocal, the product,
        and the fp32 alpha of each layer), r_G the fp32 G;
      * 2 F_k M_k for every pair at or in front of a pair whose decision may flip (`power > 0`, `alpha < 1/255`), where
        F_k = prod 1 / (1 - alpha_hi) over those flippable layers: the flip changes the pair itself by at most its |term|, and
        the T of the layers in front by at most that factor.
    `clamp_keeps_gradient=False` evaluates a wrong variant in which the clamp also cuts dL/dG where o G > 0.99; the host tests
    plant it as a defect."""
    dev = bl.device
    P = bl.means2D.shape[0]
    sg = {k: torch.zeros(P, SG_WIDTH[k], dtype=torch.float64, device=dev) for k in SG_KEYS}
    bA = {k: torch.zeros_like(v) for k, v in sg.items()}     # sum M (kappa u (n_behind + 16) + r)
    bM = {k: torch.zeros_like(v) for k, v in sg.items()}     # sum M
    bF = {k: torch.zeros_like(v) for k, v in sg.items()}     # flip allowance
    n_row = torch.zeros(P, dtype=torch.float64, device=dev)
    q = _pixel_upstream(bl, state, up)
    kap = KAPPA_BWD * U
    hx, hy = 0.5 * bl.W, 0.5 * bl.H
    for tiles, L in _chunks(bl):
        _, _, inside, pix = _pixels(bl, tiles)
        last = torch.where(inside, q["last"][pix], torch.zeros_like(pix))
        e = _pairs(bl, tiles, L, last=last)
        P_ = lambda v: v[pix][..., None]                                                 # per-pixel factor -> [nt,256,1]
        alpha, contrib, amb, pos = e["alpha"], e["contrib"], e["amb"], e["pos"]
        one_m = 1 - alpha
        f = torch.where(contrib, one_m, torch.ones_like(one_m))
        suffix = torch.flip(torch.cumprod(torch.flip(f, [-1]), -1), [-1])               # prod over layers at or behind k
        T = P_(q["T_final"]) / suffix                                                    # T before layer k
        inc = torch.where(contrib, e["e_alpha"] / one_m + 3 * U, torch.zeros_like(one_m))
        eT = U + torch.flip(torch.cumsum(torch.flip(inc, [-1]), -1), [-1])
        n_behind = torch.flip(torch.cumsum(torch.flip(contrib.double(), [-1]), -1), [-1])
        w = alpha * T
        g = e["g"]
        col = [g(bl.rgb[:, ch]) for ch in range(3)]
        S = P_(q["dalpha"]) + sum(col[ch] * P_(q["gcol"][ch]) for ch in range(3))
        Sa = P_(q["dalpha_abs"]) + sum(col[ch].abs() * P_(q["gcol_abs"][ch]) for ch in range(3))
        planes = _plane_values(bl, e)
        is_med = contrib & (pos[None, None, :] == (P_(q["maxc"]) - 1))
        terms = {}   # key -> list of (value, magnitude) per channel

        if bl.coord:
            dco, dco_a = [], []
            for ch in range(3):
                c, cabs = planes["c"][ch]
                S = S + c * P_(q["dpc"][ch])
                Sa = Sa + cabs * P_(q["dpc"][ch]).abs()
                med = torch.where(is_med, P_(q["dpmc"][ch]).expand_as(w), torch.zeros_like(w))
                dco.append(w * P_(q["dpc"][ch]) + med)
                dco_a.append(w * P_(q["dpc"][ch]).abs() + med.abs())
        if bl.depth:
            t, tabs = planes["t"]
            S = S + t * P_(q["dpt"])
            Sa = Sa + tabs * P_(q["dpt"]).abs()
            med = torch.where(is_med, P_(q["dpmt"]).expand_as(w), torch.zeros_like(w))
            dt = w * P_(q["dpt"]) + med
            dt_a = w * P_(q["dpt"]).abs() + med.abs()
        if bl.geo:
            nrm = [g(bl.normals[:, ch]) for ch in range(3)]
            S = S + sum(nrm[ch] * P_(q["dpn"][ch]) for ch in range(3))
            Sa = Sa + sum(nrm[ch].abs() * P_(q["dpn_abs"][ch]) for ch in range(3))
        wS = torch.where(contrib, w * S, torch.zeros_like(w))
        wSa = torch.where(contrib, w * Sa, torch.zeros_like(w))
        Bk = P_(q["T_final"] * q["bg_dot"]) + torch.flip(torch.cumsum(torch.flip(wS, [-1]), -1), [-1]) - wS      # layers behind k
        Bka = P_(q["T_final"] * q["bg_abs"]) + torch.flip(torch.cumsum(torch.flip(wSa, [-1]), -1), [-1]) - wSa
        dopa = T * S - Bk / one_m
        dopa_a = T * Sa + Bka / one_m
        G, o, dx, dy = e["G"], e["o"], e["dx"], e["dy"]
        dG = o * dopa                        # unclamped: dalpha/dG = o even where o G was clamped at 0.99
        dG_a = o.abs() * dopa_a
        if not clamp_keeps_gradient:
            dG = torch.where(o * G > ALPHA_MAX, torch.zeros_like(dG), dG)
        gx_ = -G * dx * e["A"] - G * dy * e["B"]
        gy_ = -G * dy * e["C"] - G * dx * e["B"]
        gx_a = G * ((dx * e["A"]).abs() + (dy * e["B"]).abs())
        gy_a = G * ((dy * e["C"]).abs() + (dx * e["B"]).abs())
        mx, my, mx_a, my_a = dG * gx_, dG * gy_, dG_a * gx_a, dG_a * gy_a
        mabs = (dG * gx_ * hx).abs() + (dG * gy_ * hy).abs()
        mabs_a = mx_a * hx + my_a * hy
        if bl.coord:
            for ch in range(3):
                cpx, cpy = g(bl.camera_planes[:, 2 * ch]), g(bl.camera_planes[:, 2 * ch + 1])
                mx, my = mx + dco[ch] * cpx, my + dco[ch] * cpy
                mx_a, my_a = mx_a + dco_a[ch] * cpx.abs(), my_a + dco_a[ch] * cpy.abs()
        if bl.depth:
            rx, ry = g(bl.ray_planes[:, 0]), g(bl.ray_planes[:, 1])
            mx, my = mx + dt * rx, my + dt * ry
            mx_a, my_a = mx_a + dt_a * rx.abs(), my_a + dt_a * ry.abs()
        terms["mean2D"] = [(mx * hx, mx_a * hx), (my * hy, my_a * hy), (mabs, mabs_a)]
        zero = torch.zeros_like(w)
        terms["conic"] = [(-0.5 * G * dx * dx * dG, 0.5 * G * dx * dx * dG_a), (-0.5 * G * dx * dy * dG, 0.5 * G * (dx * dy).abs() * dG_a),
                          (zero, zero), (-0.5 * G * dy * dy * dG, 0.5 * G * dy * dy * dG_a)]
        terms["opacity"] = [(G * dopa, G * dopa_a)]
        terms["colors"] = [(w * P_(q["gcol"][ch]), w * P_(q["gcol_abs"][ch])) for ch in range(3)]
        if bl.depth:
            terms["ts"] = [(dt, dt_a)]
            terms["ray_planes"] = [(dt * dx / bl.focal_x, dt_a * dx.abs() / bl.focal_x), (dt * dy / bl.focal_y, dt_a * dy.abs() / bl.focal_y)]
        if bl.geo:
            terms["normals"] = [(w * P_(q["dpn"][ch]), w * P_(q["dpn_abs"][ch])) for ch in range(3)]
        if bl.coord:
            terms["view_points"] = [(dco[ch], dco_a[ch]) for ch in range(3)]
            terms["camera_planes"] = [v for ch in range(3) for v in ((dco[ch] * dx / bl.focal_x, dco_a[ch] * dx.abs() / bl.focal_x),
                                                                      (dco[ch] * dy / bl.focal_y, dco_a[ch] * dy.abs() / bl.focal_y))]
        r = eT + e["e_alpha"] * (1 / alpha.clamp(min=1e-300) + 1 / one_m) + e["r_G"]
        rel = kap * (n_behind + 16) + r
        # flippable layers: every pair at or in front of one gets 2 F |term|
        Fl = torch.where(amb, 1 / (1 - e["a_hi"]), torch.ones_like(alpha))
        F = torch.flip(torch.cumprod(torch.flip(Fl, [-1]), -1), [-1])
        amb_behind = torch.flip(torch.cummax(torch.flip(amb.int(), [-1]), -1).values, [-1]).bool()
        flip = (contrib | amb) & amb_behind
        ids = e["ids"][:, None, :].expand_as(contrib)
        sel = contrib
        rows = ids[sel]
        n_row.index_add_(0, rows, torch.ones_like(rows, dtype=torch.float64))
        fsel = flip
        frows = ids[fsel]
        for k, chans in terms.items():
            for ch, (v, va) in enumerate(chans):
                v, va = v.expand_as(w), va.expand_as(w)
                sg[k][:, ch].index_add_(0, rows, v[sel])
                bA[k][:, ch].index_add_(0, rows, (va * rel)[sel])
                bM[k][:, ch].index_add_(0, rows, va[sel])
                bF[k][:, ch].index_add_(0, frows, (2 * F * va)[fsel])
    out = dict(sg)
    for k in SG_KEYS:
        out["b_" + k] = bA[k] + kap * n_row[:, None] * bM[k] + bF[k]
    out["n_row"] = n_row
    return out


def accumulator_to_sg(acc, bl: Blend) -> dict:
    """This build's packed accumulator rows (`_C.rasterize_gaussians_backward_render`, layout G_* in rgs_common.cuh) in the
    oracle's units: mean2D x/y take 0.5 W / 0.5 H, the plane rows 1/focal (backward-preprocess applies them the same way)."""
    a = torch.as_tensor(acc).double().cpu()
    P = a.shape[0]
    fx, fy = bl.focal_x, bl.focal_y
    z = lambda c: torch.zeros(P, c, dtype=torch.float64)
    sg = dict(mean2D=torch.stack([a[:, 0] * (0.5 * bl.W), a[:, 1] * (0.5 * bl.H), a[:, 15]], 1),
              conic=torch.stack([a[:, 12], a[:, 13], torch.zeros(P, dtype=torch.float64), a[:, 14]], 1),
              opacity=a[:, 11:12], colors=a[:, 4:7], ts=a[:, 7:8], ray_planes=torch.stack([a[:, 2] / fx, a[:, 3] / fy], 1),
              normals=a[:, 8:11], view_points=z(3), camera_planes=z(6))
    if a.shape[1] >= 25:
        sg["view_points"] = a[:, 16:19]
        sg["camera_planes"] = a[:, 19:25] / torch.tensor([fx, fy, fx, fy, fx, fy], dtype=torch.float64)
    return sg


def check_backward(ref: dict, given: dict, name="", max_report=8) -> dict:
    """Every row and channel of `given` (orc_sgrad units) within its bound; rows that received nothing must be exactly zero
    (their bound is zero).  The unit conversion of `accumulator_to_sg` adds one rounding: 2u |value| is allowed for it."""
    stats, errors = {}, []
    for k in SG_KEYS:
        r = ref[k].cpu().numpy()
        a = _np64(given[k]).reshape(r.shape)
        b = ref["b_" + k].cpu().numpy() + 2 * U * np.abs(r)
        d = np.abs(a - r)
        rt = np.where(np.isnan(a), np.inf, _ratio(d, b))
        for ch in range(r.shape[1]):
            stats[f"{k}[{ch}]"] = float(rt[:, ch].max()) if rt.shape[0] else 0.0
        bad = np.argwhere(rt > 1)
        for row, ch in bad[:max_report]:
            what = "received nothing in fp64, must be exactly 0" if b[row, ch] == 0 else f"bound {b[row, ch]:.3e}"
            errors.append(f"{name}: {k}[{ch}] of row {row}: {a[row, ch]!r} vs fp64 {r[row, ch]!r}, {what} "
                          f"({int(ref['n_row'][row])} pairs)")
        if len(bad) > max_report:
            errors.append(f"{name}: {k}: {len(bad)} elements out of bound")
    if errors:
        raise AssertionError("\n".join(errors))
    return stats
