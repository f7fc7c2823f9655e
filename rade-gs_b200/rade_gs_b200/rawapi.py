"""Thin helpers that call a `_C`-style module (this build or the reference build) on a synthetic Scene.

Both modules export the reference's `rasterize_gaussians` / `rasterize_gaussians_backward`
(reference: rasterize_points.h:18-76), so the same two functions drive either one -- this is what the parity
tests and `bench.py` time (SURVEY.md 8d: t_fwd = `_C.rasterize_gaussians`, t_bwd = `_C.rasterize_gaussians_backward`).
"""
from __future__ import annotations

import torch

FWD_KEYS = ("num_rendered", "color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth", "radii", "geom", "binning", "img")
BWD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")


def _absent():
    return torch.Tensor([])


def forward(C, sc, require_coord: bool, require_depth: bool, kernel_size: float = 0.0, sh_degree: int = 3,
            scale_modifier: float = 1.0, colors_precomp=None, cov3D_precomp=None, debug: bool = False) -> dict:
    shs = _absent() if colors_precomp is not None else sc.shs
    cols = colors_precomp if colors_precomp is not None else _absent()
    scales = _absent() if cov3D_precomp is not None else sc.scales
    rots = _absent() if cov3D_precomp is not None else sc.rotations
    cov = cov3D_precomp if cov3D_precomp is not None else _absent()
    out = C.rasterize_gaussians(sc.bg, sc.means3D, cols, sc.opacities, scales, rots, scale_modifier, cov,
                                sc.viewmatrix, sc.projmatrix, sc.tanfovx, sc.tanfovy, kernel_size, sc.height, sc.width,
                                shs, sh_degree, sc.campos, False, require_coord, require_depth, debug)
    res = dict(zip(FWD_KEYS, out))
    res["_call"] = dict(require_coord=require_coord, require_depth=require_depth, kernel_size=kernel_size, sh_degree=sh_degree,
                        scale_modifier=scale_modifier, shs=shs, cols=cols, scales=scales, rots=rots, cov=cov, debug=debug)
    return res


def backward(C, sc, fwd: dict, grads: dict) -> dict:
    c = fwd["_call"]
    out = C.rasterize_gaussians_backward(sc.bg, sc.means3D, fwd["radii"], c["cols"], c["scales"], c["rots"], c["scale_modifier"], c["cov"],
                                         sc.viewmatrix, sc.projmatrix, sc.tanfovx, sc.tanfovy, c["kernel_size"],
                                         grads["color"], grads["coord"], grads["mcoord"], grads["depth"], grads["mdepth"], grads["alpha"],
                                         grads["normal"], fwd["normal"], c["shs"], c["sh_degree"], sc.campos, fwd["geom"], fwd["num_rendered"],
                                         fwd["binning"], fwd["img"], fwd["alpha"], c["require_coord"], c["require_depth"], c["debug"])
    return dict(zip(BWD_KEYS, out))


# ---- views into the private buffers (parity tests only) ----------------------------------------------------------

def _align(x, a=128):
    return (x + a - 1) // a * a


class _Cursor:
    def __init__(self, buf):
        self.buf, self.off = buf, 0

    def take(self, count, dtype, itemsize):
        self.off = _align(self.off)
        v = self.buf[self.off:self.off + count * itemsize].view(dtype)
        self.off += count * itemsize
        return v


def ours_views(fwd: dict, sc) -> dict:
    """Decode this build's buffers (layout: rgs_api.cu carve_geom / carve_bin / carve_img)."""
    P = sc.means3D.shape[0]
    R = int(fwd["num_rendered"])
    coord, depth = fwd["_call"]["require_coord"], fwd["_call"]["require_depth"]
    RF = 24 if coord else 16
    N = sc.width * sc.height
    tiles = ((sc.width + 15) // 16) * ((sc.height + 15) // 16)
    g = _Cursor(fwd["geom"])
    rec = g.take(P * RF, torch.float32, 4).view(P, RF)
    depths = g.take(P, torch.float32, 4)
    tiles_touched = g.take(P, torch.int32, 4)
    g.take(P, torch.int32, 4)  # backward preprocess's row list
    clamped = g.take(P, torch.uint8, 1)
    g.take(P * 12, torch.float32, 4)  # Sigma^-1 kept for backward
    b = _Cursor(fwd["binning"])
    point_list = b.take(R, torch.int32, 4)
    keys = b.take(R, torch.int64, 8)
    # forward-render's ballots: word (chunk_base[tile] + k) * 8 + warp holds, for list positions [32k, 32k + 32) of the tile, the
    # entries that warp's 8x4 pixel block did not cull (warp w covers tile columns 8 (w & 1) .. +7, rows 4 (w >> 1) .. +3)
    hitmask = b.take((R // 32 + tiles + 1) * 8, torch.int32, 4)
    i = _Cursor(fwd["img"])
    ranges = i.take(tiles * 2, torch.int32, 4).view(tiles, 2)
    i.take(tiles, torch.int32, 4)   # tile_count (counted back down to zero by the scatter)
    totals = i.take(2, torch.int32, 4)
    chunk_base = i.take(tiles, torch.int32, 4)  # first 32-entry chunk of each tile's list, in hit-mask words / 8
    n_contrib = i.take(2 * N, torch.int32, 4).view(2, sc.height, sc.width)
    accum_depth = i.take(N if depth else 0, torch.float32, 4).view(-1, sc.width)
    normal_length = i.take(N if (coord or depth) else 0, torch.float32, 4).view(-1, sc.width)
    accum_coord = i.take(3 * N if coord else 0, torch.float32, 4).view(-1, sc.height, sc.width)
    return dict(totals=totals, records=rec, depths=depths, tiles_touched=tiles_touched, clamped=clamped, point_list=point_list,
                keys=keys, hitmask=hitmask, ranges=ranges, chunk_base=chunk_base, n_contrib=n_contrib,
                accum_depth=(accum_depth if depth else None), normal_length=(normal_length if (coord or depth) else None),
                accum_coord=(accum_coord if coord else None),
                means2D=rec[:, 0:2], conic_opacity=torch.stack([rec[:, 2], rec[:, 3], rec[:, 4], rec[:, 5]], 1), ts=rec[:, 11],
                ray_planes=rec[:, 6:8], rgb=rec[:, 8:11], normals=rec[:, 12:15],
                camera_planes=(torch.cat([rec[:, 19:24], rec[:, 15:16]], 1) if coord else None),
                view_points=(rec[:, 16:19] if coord else None))


def ref_views(fwd: dict, sc) -> dict:
    """Decode the reference build's buffers (reference: cuda_rasterizer/rasterizer_impl.cu:190-250; SURVEY.md app. B)."""
    P = sc.means3D.shape[0]
    R = int(fwd["num_rendered"])
    N = sc.width * sc.height
    tiles = ((sc.width + 15) // 16) * ((sc.height + 15) // 16)
    g = _Cursor(fwd["geom"])
    v = {}
    v["depths"] = g.take(P, torch.float32, 4)
    v["camera_planes"] = g.take(P * 6, torch.float32, 4).view(P, 6)
    v["ray_planes"] = g.take(P * 2, torch.float32, 4).view(P, 2)
    v["ts"] = g.take(P, torch.float32, 4)
    v["normals"] = g.take(P * 3, torch.float32, 4).view(P, 3)
    v["clamped"] = g.take(P * 3, torch.uint8, 1).view(P, 3)
    v["internal_radii"] = g.take(P, torch.int32, 4)
    v["means2D"] = g.take(P * 2, torch.float32, 4).view(P, 2)
    v["view_points"] = g.take(P * 3, torch.float32, 4).view(P, 3)
    v["cov3D"] = g.take(P * 6, torch.float32, 4).view(P, 6)
    v["conic_opacity"] = g.take(P * 4, torch.float32, 4).view(P, 4)
    v["rgb"] = g.take(P * 3, torch.float32, 4).view(P, 3)
    v["tiles_touched"] = g.take(P, torch.int32, 4)
    b = _Cursor(fwd["binning"])
    v["point_list"] = b.take(R, torch.int32, 4)
    b.take(R, torch.int32, 4)
    v["keys"] = b.take(R, torch.int64, 8)
    i = _Cursor(fwd["img"])
    v["n_contrib"] = i.take(2 * N, torch.int32, 4).view(2, sc.height, sc.width)
    v["ranges"] = i.take(N * 2, torch.int32, 4).view(N, 2)[:tiles]
    return v
