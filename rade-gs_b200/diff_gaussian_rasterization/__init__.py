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
  rotations, cov3Ds_precomp, None)`` (ref :157-167); ``means2D.grad`` receives ``(d/dx, d/dy, sum |.|)``.

So ``gaussian_renderer.render()``, ``train.py`` and ``render.py`` of the reference import this package unchanged.
The compiled module ``_C`` exports the reference's four symbols; there is no CPU or eager fallback -- importing
this package without the built extension raises.
"""
from __future__ import annotations

import os as _os
from typing import NamedTuple

import torch
import torch.nn as nn

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


def _forward_args(s: GaussianRasterizationSettings, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh):
    # order of RasterizeGaussiansCUDA (reference: rasterize_points.h:18-41)
    return (
        s.bg, means3D, colors_precomp, opacities, scales, rotations, s.scale_modifier, cov3Ds_precomp,
        s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.image_height, s.image_width,
        sh, s.sh_degree, s.campos, s.prefiltered, s.require_coord, s.require_depth, s.debug,
    )


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        s = raster_settings
        args = _forward_args(s, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh)
        (num_rendered, color, coord, mcoord, alpha, normal, depth, mdepth, radii,
         geom_buf, binning_buf, img_buf) = _call_with_dump(_C.rasterize_gaussians, args, s.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh,
                              geom_buf, binning_buf, img_buf, alpha)
        return color, radii, coord, mcoord, depth, mdepth, alpha, normal

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal):
        s = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh,
         geom_buf, binning_buf, img_buf, alpha) = ctx.saved_tensors
        # order of RasterizeGaussiansBackwardCUDA (reference: rasterize_points.h:43-76)
        args = (
            s.bg, means3D, radii, colors_precomp, scales, rotations, s.scale_modifier, cov3Ds_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size,
            grad_color, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal, normal,
            sh, s.sh_degree, s.campos, geom_buf, ctx.num_rendered, binning_buf, img_buf, alpha,
            s.require_coord, s.require_depth, s.debug,
        )
        (g_means2D, g_colors, g_opacities, g_means3D, g_cov3D, g_sh, g_scales, g_rotations) = _call_with_dump(
            _C.rasterize_gaussians_backward, args, s.debug, "snapshot_bw.dump", "backward")
        return g_means3D, g_means2D, g_sh, g_colors, g_opacities, g_scales, g_rotations, g_cov3D, None


class _RasterizeGaussiansSplitSh(torch.autograd.Function):
    """Same op with the SH coefficients left in the model's two tensors (``_features_dc`` [P,1,3], ``_features_rest``
    [P,M-1,3]; reference scene/gaussian_model.py:133-136 concatenates them every iteration).  Opt-in extension
    (SURVEY.md 8f row 1): pass ``shs=(features_dc, features_rest)`` to ``GaussianRasterizer.forward``."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh_dc, sh_rest, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        s = raster_settings
        none = _absent()
        args = (
            s.bg, means3D, none, opacities, scales, rotations, s.scale_modifier, cov3Ds_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size, s.image_height, s.image_width,
            sh_dc, sh_rest, s.sh_degree, s.campos, s.prefiltered, s.require_coord, s.require_depth, s.debug,
        )
        (num_rendered, color, coord, mcoord, alpha, normal, depth, mdepth, radii,
         geom_buf, binning_buf, img_buf) = _call_with_dump(_C.rasterize_gaussians_split_sh, args, s.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh_dc, sh_rest, geom_buf, binning_buf, img_buf, alpha)
        return color, radii, coord, mcoord, depth, mdepth, alpha, normal

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal):
        s = ctx.raster_settings
        (means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh_dc, sh_rest, geom_buf, binning_buf, img_buf, alpha) = ctx.saved_tensors
        args = (
            s.bg, means3D, radii, _absent(), scales, rotations, s.scale_modifier, cov3Ds_precomp,
            s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.kernel_size,
            grad_color, grad_coord, grad_mcoord, grad_depth, grad_mdepth, grad_alpha, grad_normal, normal,
            sh_dc, sh_rest, s.sh_degree, s.campos, geom_buf, ctx.num_rendered, binning_buf, img_buf, alpha,
            s.require_coord, s.require_depth, s.debug,
        )
        (g_means2D, _g_colors, g_opacities, g_means3D, g_cov3D, g_sh_dc, g_sh_rest, g_scales, g_rotations) = _call_with_dump(
            _C.rasterize_gaussians_backward_split_sh, args, s.debug, "snapshot_bw.dump", "backward")
        return g_means3D, g_means2D, g_sh_dc, g_sh_rest, g_opacities, g_scales, g_rotations, g_cov3D, None


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings)


def _absent():
    # the C++ side reads "no tensor" from an empty CPU tensor (reference: :214-224, rasterize_points.cu:104-112)
    return torch.Tensor([])


def _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp):
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    pair_missing = scales is None or rotations is None
    pair_any = scales is not None or rotations is not None
    if (pair_missing and cov3D_precomp is None) or (pair_any and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of the points in front of the near plane (reference :193-202)."""
        with torch.no_grad():
            s = self.raster_settings
            return _C.mark_visible(positions, s.viewmatrix, s.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp)
        split_sh = isinstance(shs, (tuple, list))  # extension: (features_dc [P,1,3], features_rest [P,M-1,3])
        shs = _absent() if shs is None else shs
        colors_precomp = _absent() if colors_precomp is None else colors_precomp
        scales = _absent() if scales is None else scales
        rotations = _absent() if rotations is None else rotations
        cov3D_precomp = _absent() if cov3D_precomp is None else cov3D_precomp
        if split_sh:
            if len(shs) != 2:
                raise ValueError("split SH layout: shs must be the pair (features_dc, features_rest)")
            if shs[1].numel() == 0:  # degree-0 model: nothing to split
                shs = shs[0]
            else:
                return _RasterizeGaussiansSplitSh.apply(means3D, means2D, shs[0], shs[1], opacities, scales, rotations, cov3D_precomp,
                                                        self.raster_settings)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, self.raster_settings)

    def integrate(self, points3D, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                  cov3D_precomp=None, view2gaussian_precomp=None):
        """GOF-style opacity integration at query points (reference :239-306), used by marching-tetrahedra mesh
        extraction.  Returns ``(color [9,H,W], alpha_integrated [PN], color_integrated [PN,3], point_coordinate [PN,2],
        point_sdf [PN], radii [P])``; like the reference the call is not differentiable and runs with kernel_size 0."""
        s = self.raster_settings
        _check_exclusive(shs, colors_precomp, scales, rotations, cov3D_precomp)
        shs = _absent() if shs is None else shs
        colors_precomp = _absent() if colors_precomp is None else colors_precomp
        scales = _absent() if scales is None else scales
        rotations = _absent() if rotations is None else rotations
        cov3D_precomp = _absent() if cov3D_precomp is None else cov3D_precomp
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
