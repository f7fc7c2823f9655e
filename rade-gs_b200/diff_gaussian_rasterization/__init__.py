"""Drop-in ``diff_gaussian_rasterization`` package backed by the H100-native (sm_90a) rasterizer.

Public surface kept identical to the reference wrapper
(reference: submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py):

* ``GaussianRasterizationSettings`` -- NamedTuple, same 15 fields in the same order (ref :171-186);
* ``GaussianRasterizer(raster_settings)`` with ``forward(means3D, means2D, opacities, shs, colors_precomp,
  scales, rotations, cov3D_precomp)`` returning ``(color, radii, coord, mcoord, depth, mdepth, alpha, normal)``
  (ref :101, :204-237), ``markVisible(positions)`` (ref :193-202) and ``integrate(...)`` (ref :239-306, the
  opacity integration at query points used by mesh extraction);
* ``rasterize_gaussians(...)`` functional form (ref :20-42);
* gradient order of the autograd function ``(means3D, means2D, sh, colors_precomp, opacities, scales,
  rotations, cov3Ds_precomp, None)`` (ref :157-167), followed by that of the split-SH extension's ``sh_rest``;
  ``means2D.grad`` receives ``(d/dx, d/dy, sum |.|)``.

So ``gaussian_renderer.render()``, ``train.py`` and ``render.py`` of the reference import this package unchanged.
The compiled module ``_C`` exports the reference's four symbols; there is no CPU or eager fallback -- importing
this package without the built extension raises.
"""
from __future__ import annotations

import os as _os
from typing import NamedTuple

import torch
import torch.nn as nn
from rade_gs_b200.rawapi import backward_args, forward_args

try:
    from . import _C
except ImportError as _exc:  # fail loudly: a silent fallback would void every parity claim
    raise ImportError(
        "diff_gaussian_rasterization._C (sm_90a build) is missing or failed to load: run "
        "`python rade-gs_b200/build.py` (needs nvcc, sm_90a).  Original error: %s" % (_exc,)
    ) from _exc

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians"]


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    kernel_size: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    require_depth: bool
    require_coord: bool
    debug: bool


def _snapshot(args):
    """CPU copies of a call's arguments, taken before the call so a crash cannot corrupt them (ref :17-19)."""
    return tuple(a.detach().cpu().clone() if isinstance(a, torch.Tensor) else a for a in args)


def _call_with_dump(fn, args, debug: bool, dump_name: str, what: str):
    """Run ``fn(*args)``; with ``debug`` set, dump the arguments to ``dump_name`` if it throws (ref :86-95,146-155)."""
    if not debug:
        return fn(*args)
    saved = _snapshot(args)
    try:
        return fn(*args)
    except Exception:
        torch.save(saved, dump_name)
        print("\nAn error occured in %s. Please forward %s for debugging." % (what, dump_name))
        raise


class _RasterizeGaussians(torch.autograd.Function):
    """The reference's autograd function, plus one input: a non-empty ``sh_rest`` keeps the SH coefficients in the model's two
    tensors (``sh`` = ``_features_dc`` [P,1,3], ``sh_rest`` = ``_features_rest`` [P,M-1,3]; reference
    scene/gaussian_model.py:133-136 concatenates them every iteration).  Opt-in extension (SURVEY.md 8f row 1): pass
    ``shs=(features_dc, features_rest)`` to ``GaussianRasterizer.forward``."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, sh_rest,
                reserve=None):
        s = raster_settings
        rest = sh_rest if sh_rest.numel() else None
        if reserve is None:
            args = forward_args(s, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh, rest)
            fn = _C.rasterize_gaussians if rest is None else _C.rasterize_gaussians_split_sh
            out = _call_with_dump(fn, args, s.debug, "snapshot_fw.dump", "forward")
        else:
            out = _forward_into_reserve(forward_args(s, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh) + (sh_rest,),
                                        reserve)
        (num_rendered, color, coord, mcoord, alpha, normal, depth, mdepth, radii, geom_buf, binning_buf, img_buf) = out
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh,
                              geom_buf, binning_buf, img_buf, alpha, sh_rest)
        return color, radii, coord, mcoord, depth, mdepth, alpha, normal

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal):
        s = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh,
         geom_buf, binning_buf, img_buf, alpha, sh_rest) = ctx.saved_tensors
        rest = sh_rest if sh_rest.numel() else None
        args = backward_args(s, means3D, radii, colors_precomp, scales, rotations, cov3Ds_precomp,
                             (grad_color, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal), normal, sh,
                             geom_buf, ctx.num_rendered, binning_buf, img_buf, alpha, rest)
        fn = _C.rasterize_gaussians_backward if rest is None else _C.rasterize_gaussians_backward_split_sh
        # the split-SH symbol returns the gradient of sh_rest after that of sh
        (g_means2D, g_colors, g_opacities, g_means3D, g_cov3D, g_sh, *g_sh_rest, g_scales, g_rotations) = _call_with_dump(
            fn, args, s.debug, "snapshot_bw.dump", "backward")
        return (g_means3D, g_means2D, g_sh, g_colors, g_opacities, g_scales, g_rotations, g_cov3D, None, (g_sh_rest[0] if g_sh_rest else None),
                None)


def _forward_into_reserve(args, reserve):
    """The forward binned into `reserve`'s capacities (`_C._graph`, no host read).  Under stream capture: the call only; the caller
    reads the reserve's status after the step.  Eagerly: the status is read at once, and a frame that did not fit grows the
    reserve and runs again."""
    def call():
        return _C._graph.rasterize_gaussians(*args, reserve.instances, reserve.longest_list, reserve.status)

    if torch.cuda.is_current_stream_capturing():
        return call()
    reserve.clear()
    out = call()
    if reserve.overflowed():
        reserve.clear()
        out = call()
    return out


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                                     _absent())


def _absent():
    # the C++ side reads "no tensor" from an empty CPU tensor (reference: :214-224, rasterize_points.cu:104-112)
    return torch.Tensor([])


def _inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's exactly-one-of checks, then every input not given as the absent tensor, in argument order."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    pair_missing = scales is None or rotations is None
    pair_any = scales is not None or rotations is not None
    if (pair_missing and cov3D_precomp is None) or (pair_any and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    return tuple(_absent() if t is None else t for t in (shs, colors_precomp, scales, rotations, cov3D_precomp))


class GaussianRasterizer(nn.Module):
    """``reserve`` (extension, a ``rade_gs_b200.graphs.BinningReserve``): bin every forward into the reserve's capacities without
    reading the frame's instance count on the host, so that the call can be captured in a CUDA graph (``rade_gs_b200.graphs``).
    Whole image only; not with ``debug``."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, reserve=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.reserve = reserve

    def markVisible(self, positions):
        """Boolean mask of the points in front of the near plane (reference :193-202)."""
        with torch.no_grad():
            s = self.raster_settings
            return _C.mark_visible(positions, s.viewmatrix, s.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp = _inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
        sh_rest = _absent()
        if isinstance(shs, (tuple, list)):  # extension: (features_dc [P,1,3], features_rest [P,M-1,3])
            if len(shs) != 2:
                raise ValueError("split SH layout: shs must be the pair (features_dc, features_rest)")
            shs, sh_rest = shs  # a degree-0 model's empty features_rest takes the reference path
        return _RasterizeGaussians.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, self.raster_settings,
                                         sh_rest, self.reserve)

    def integrate(self, points3D, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                  cov3D_precomp=None, view2gaussian_precomp=None):
        """GOF-style opacity integration at query points (reference :239-306), used by marching-tetrahedra mesh
        extraction.  Returns ``(color [9,H,W], alpha_integrated [PN], color_integrated [PN,3], point_coordinate [PN,2],
        point_sdf [PN], radii [P])``; like the reference the call is not differentiable and runs with kernel_size 0."""
        s = self.raster_settings
        shs, colors_precomp, scales, rotations, cov3D_precomp = _inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
        view2gaussian_precomp = _absent() if view2gaussian_precomp is None else view2gaussian_precomp
        subpixel_offset = _absent()  # the reference allocates an [H,W,2] zero tensor that its kernel never uses (:265)
        args = (
            s.bg, points3D, means3D, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3D_precomp, view2gaussian_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, 0.0, subpixel_offset, s.image_height, s.image_width, shs, s.sh_degree,
            s.campos, s.prefiltered, s.debug,
        )
        with torch.no_grad():
            (_num_rendered, color, alpha_integrated, color_integrated, point_coordinate, point_sdf, radii,
             _geom, _binning, _img) = _call_with_dump(_C.integrate_gaussians_to_points, args, s.debug, "snapshot_fw.dump", "forward")
        return color, alpha_integrated, color_integrated, point_coordinate, point_sdf, radii
