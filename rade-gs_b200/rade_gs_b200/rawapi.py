"""Thin helpers that call a `_C`-style module (this build or the reference build) on a synthetic Scene.

Both modules export the reference's `rasterize_gaussians` / `rasterize_gaussians_backward`
(reference: rasterize_points.h:18-76), so the same two functions drive either one -- this is what the parity
tests and `bench.py` time (SURVEY.md 8d: t_fwd = `_C.rasterize_gaussians`, t_bwd = `_C.rasterize_gaussians_backward`).
This build's extras -- the tile-row slab forward and the two stages of the multi-GPU backward -- are driven the same way
(`forward(..., tile_rows=...)`, `backward_render`, `backward_preprocess`).  `forward_args`, `backward_args` and `preprocess_args`
spell each call's argument order once, for these helpers and the autograd wrappers; this module imports no extension.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

FWD_KEYS = ("num_rendered", "color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth", "radii", "geom", "binning", "img")
BWD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")
_CALL_SETTINGS = ("kernel_size", "scale_modifier", "sh_degree", "require_coord", "require_depth", "debug")


def _absent():
    return torch.Tensor([])


def forward_args(s, means3D, colors_precomp, opacities, scales, rotations, cov3D_precomp, sh, sh_rest=None) -> tuple:
    """The forward's arguments in the order of RasterizeGaussiansCUDA (reference: rasterize_points.h:18-41), from raster settings
    `s` (the fields of `GaussianRasterizationSettings`) and the Gaussians.  The split-SH symbol takes `sh_rest` after `sh`."""
    return (s.bg, means3D, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3D_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.image_height, s.image_width,
            *((sh,) if sh_rest is None else (sh, sh_rest)), s.sh_degree, s.campos, s.prefiltered, s.require_coord, s.require_depth, s.debug)


def backward_args(s, means3D, radii, colors_precomp, scales, rotations, cov3D_precomp, grads, normal, sh, geom, num_rendered, binning, img,
                  alpha, sh_rest=None) -> tuple:
    """The backward's arguments in the order of RasterizeGaussiansBackwardCUDA (reference: rasterize_points.h:43-76); `grads` are the
    gradients of the maps color, coord, mcoord, depth, mdepth, alpha, normal.  The split-SH symbol takes `sh_rest` after `sh`."""
    return (s.bg, means3D, radii, colors_precomp, scales, rotations, s.scale_modifier, cov3D_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, *grads, normal,
            *((sh,) if sh_rest is None else (sh, sh_rest)), s.sh_degree, s.campos, geom, num_rendered, binning, img, alpha,
            s.require_coord, s.require_depth, s.debug)


def preprocess_args(s, acc, means3D, radii, colors_precomp, opacities, scales, rotations, cov3D_precomp, sh, geom) -> tuple:
    """The arguments of stage 2 (`rasterize_gaussians_backward_preprocess`) for the summed accumulator rows `acc`."""
    return (acc, s.bg, means3D, radii, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3D_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.image_height, s.image_width, sh, s.sh_degree, s.campos,
            geom, s.require_coord, s.require_depth, s.debug)


def _settings(sc, c: dict) -> SimpleNamespace:  # the raster settings of call `c` on scene `sc`
    return SimpleNamespace(image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, bg=sc.bg, viewmatrix=sc.viewmatrix,
                           projmatrix=sc.projmatrix, campos=sc.campos, prefiltered=False, **{k: c[k] for k in _CALL_SETTINGS})


def _forward_args(sc, c: dict) -> tuple:
    return forward_args(_settings(sc, c), sc.means3D, c["cols"], sc.opacities, c["scales"], c["rots"], c["cov"], c["shs"])


def _backward_args(sc, fwd: dict, grads: dict) -> tuple:
    c = fwd["_call"]
    return backward_args(_settings(sc, c), sc.means3D, fwd["radii"], c["cols"], c["scales"], c["rots"], c["cov"],
                         [grads[k] for k in ("color", "coord", "mcoord", "depth", "mdepth", "alpha", "normal")], fwd["normal"], c["shs"],
                         fwd["geom"], fwd["num_rendered"], fwd["binning"], fwd["img"], fwd["alpha"])


def forward(C, sc, require_coord: bool, require_depth: bool, kernel_size: float = 0.0, sh_degree: int = 3,
            scale_modifier: float = 1.0, colors_precomp=None, cov3D_precomp=None, debug: bool = False,
            tile_rows: tuple | None = None, compact: bool = False) -> dict:
    """The whole image, or with ``tile_rows=(begin, end)`` only the tile rows of that slab (`rasterize_gaussians_slab`; with
    ``compact`` the maps hold only the slab's pixel rows)."""
    c = dict(require_coord=require_coord, require_depth=require_depth, kernel_size=kernel_size, sh_degree=sh_degree,
             scale_modifier=scale_modifier, debug=debug, tile_rows=tile_rows, compact=compact,
             shs=_absent() if colors_precomp is not None else sc.shs,
             cols=colors_precomp if colors_precomp is not None else _absent(),
             scales=_absent() if cov3D_precomp is not None else sc.scales,
             rots=_absent() if cov3D_precomp is not None else sc.rotations,
             cov=cov3D_precomp if cov3D_precomp is not None else _absent())
    args = _forward_args(sc, c)
    out = C.rasterize_gaussians(*args) if tile_rows is None else C.rasterize_gaussians_slab(*args, *tile_rows, compact)
    res = dict(zip(FWD_KEYS, out))
    res["_call"] = c
    return res


def backward(C, sc, fwd: dict, grads: dict) -> dict:
    return dict(zip(BWD_KEYS, C.rasterize_gaussians_backward(*_backward_args(sc, fwd, grads))))


def backward_render(C, sc, fwd: dict, grads: dict) -> torch.Tensor:
    """Stage 1 of the two-stage backward over the forward's slab (the whole image without one): the packed gradient
    accumulator rows [P, stride], additive across slabs.  For compact maps ``grads`` hold the slab's rows only."""
    c = fwd["_call"]
    b, e = c["tile_rows"] if c["tile_rows"] is not None else (0, -1)
    return C.rasterize_gaussians_backward_render(*_backward_args(sc, fwd, grads), b, e, c["compact"], sc.height)


def backward_preprocess(C, sc, fwd: dict, acc: torch.Tensor) -> dict:
    """Stage 2: the (summed) accumulator rows -> the parameter gradients of `backward`."""
    c = fwd["_call"]
    args = preprocess_args(_settings(sc, c), acc, sc.means3D, fwd["radii"], c["cols"], sc.opacities, c["scales"], c["rots"], c["cov"], c["shs"], fwd["geom"])
    return dict(zip(BWD_KEYS, C.rasterize_gaussians_backward_preprocess(*args)))


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
    sigma_inv = g.take(P * 12, torch.float32, 4).view(P, 12)  # Sigma^-1 kept for backward: 9 floats column-major, flag bits in float 9
    b = _Cursor(fwd["binning"])
    point_list = b.take(R, torch.int32, 4)
    keys = b.take(R, torch.int64, 8)
    # forward-render's ballots: word (chunk_base[tile] + k) * 8 + s holds, for list positions [32k, 32k + 32) of the tile, the
    # entries the box test kept for the 8x8 pixel block holding 8x4 half s (half s covers tile columns 8 (s & 1) .. +7, rows
    # 4 (s >> 1) .. +3); the two halves of a block, s and s + 2 with s & 2 == 0, hold the same word
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
    return dict(totals=totals, records=rec, sigma_inv=sigma_inv, depths=depths, tiles_touched=tiles_touched, clamped=clamped, point_list=point_list,
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
