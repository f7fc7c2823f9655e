"""GaussianModel.densify_and_prune and reset_opacity (reference scene/gaussian_model.py:495-513, :662-741) on the GPU.

``densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size)`` and ``reset_opacity(gaussians)`` take the
reference's ``GaussianModel`` (duck-typed: ``_xyz``, ``_features_dc``, ``_features_rest``, ``_opacity``, ``_scaling``,
``_rotation``, the densification statistics, ``filter_3D``, ``percent_dense`` and ``optimizer``) and mutate it as the methods
do, with the same result: the same rows in the same order, the Adam moments following their rows, zero moments on new rows,
``step`` and every other state key kept, a new ``nn.Parameter`` per group, the appearance groups untouched.

Where the reference concatenates and mask-indexes every parameter and moment three times, the kernels in csrc/rgs_densify.cu
select once, read five counts back once, and write every output row once from its source row.  The quantile threshold is
exact at any size (torch.quantile refuses more than 2^24 Gaussians).  The random offsets of new rows are drawn through
``torch.normal`` with the reference's shapes and order ([C, 3] for the clones, then [2S, 3] for the split children), so a
seeded run consumes the same random numbers.  No ``torch.cuda.empty_cache()``.  No CPU path: CUDA tensors only.
"""
from __future__ import annotations

import torch
from torch import nn

from diff_gaussian_rasterization import _C

__all__ = ["densify_and_prune", "reset_opacity"]

# optimizer group name -> GaussianModel attribute, in the reference's group order
_GROUPS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
           "rotation": "_rotation"}
_UNTOUCHED = ("appearance_embeddings", "appearance_network")


def _param_groups(gaussians):
    groups = {}
    for group in gaussians.optimizer.param_groups:
        if group["name"] in _UNTOUCHED:
            continue
        if len(group["params"]) != 1:
            raise ValueError(f"densify: optimizer group {group['name']!r} must hold one parameter")
        groups[group["name"]] = group
    missing = [name for name in _GROUPS if name not in groups]
    if missing:
        raise ValueError(f"densify: the optimizer has no group for {missing}")
    for name, attr in _GROUPS.items():
        if not groups[name]["params"][0].is_cuda or not getattr(gaussians, attr).is_cuda:
            raise RuntimeError("densify: the model must be on a CUDA device: there is no CPU path")
    return groups


def _replace(gaussians, group, param, moments=None):
    """Install `param` as the group's new parameter; the optimizer state (if any) moves to it with `moments` replacing
    exp_avg and exp_avg_sq (scene/gaussian_model.py:561-596)."""
    optimizer = gaussians.optimizer
    old = group["params"][0]
    state = optimizer.state.get(old, None)
    new = nn.Parameter(param.requires_grad_(True))
    if state is not None:
        state["exp_avg"], state["exp_avg_sq"] = moments
        del optimizer.state[old]
    group["params"][0] = new
    if state is not None:
        optimizer.state[new] = state
    setattr(gaussians, _GROUPS[group["name"]], new)


@torch.no_grad()
def densify_and_prune(gaussians, max_grad, min_opacity, extent, max_screen_size):
    """scene/gaussian_model.py:717-741.  Returns the reference's (cloned, split, pruned) counts."""
    groups = _param_groups(gaussians)
    p = {name: groups[name]["params"][0] for name in _GROUPS}
    flags, offsets, _, counts = _C._densify.select(
        gaussians.xyz_gradient_accum, gaussians.xyz_gradient_accum_abs, gaussians.denom, p["scaling"], p["opacity"], float(max_grad),
        gaussians.percent_dense * extent, float(min_opacity), bool(max_screen_size), float(max_screen_size or 0), 0.1 * extent)
    C, S = counts[0], counts[1]
    src, draw, std_clone, std_split = _C._densify.plan(flags, offsets, counts, p["scaling"])
    dev = p["xyz"].device
    sample_clone = torch.normal(mean=torch.zeros((C, 3), device=dev), std=std_clone)
    sample_split = torch.normal(mean=torch.zeros((2 * S, 3), device=dev), std=std_split)

    columns, slots = [], {}
    for name in _GROUPS:
        state = gaussians.optimizer.state.get(p[name], None)
        if name not in ("xyz", "scaling"):        # xyz and scaling of new rows are computed, not copied
            slots[name] = len(columns)
            columns.append((p[name].detach(), False))
        if state is not None:
            slots[name + ".moments"] = len(columns)
            columns += [(state["exp_avg"], True), (state["exp_avg_sq"], True)]
    xyz, scaling, outs = _C._densify.gather(src, draw, C, p["xyz"].detach(), p["rotation"].detach(), p["scaling"].detach(), sample_clone,
                                           sample_split, columns)
    for name in _GROUPS:
        param = {"xyz": xyz, "scaling": scaling}.get(name)
        if param is None:
            param = outs[slots[name]]
        k = slots.get(name + ".moments")
        _replace(gaussians, groups[name], param, None if k is None else (outs[k], outs[k + 1]))

    N = xyz.shape[0]
    gaussians.xyz_gradient_accum = torch.zeros((N, 1), device=dev)
    gaussians.xyz_gradient_accum_abs = torch.zeros((N, 1), device=dev)
    gaussians.xyz_gradient_accum_abs_max = torch.zeros((N, 1), device=dev)
    gaussians.denom = torch.zeros((N, 1), device=dev)
    gaussians.max_radii2D = torch.zeros((N,), device=dev)
    P = flags.shape[0]
    return C, S, P + C + S - N


@torch.no_grad()
def reset_opacity(gaussians):
    """scene/gaussian_model.py:495-513: opacity := inverse_sigmoid(min(opacity_with_3D_filter, 0.01) / coef), zero moments."""
    groups = _param_groups(gaussians)
    if not gaussians.filter_3D.is_cuda:
        raise RuntimeError("reset_opacity: the model must be on a CUDA device: there is no CPU path")
    new = _C._densify.reset_opacity(groups["scaling"]["params"][0].detach(), groups["opacity"]["params"][0].detach(), gaussians.filter_3D)
    _replace(gaussians, groups["opacity"], new, (torch.zeros_like(new), torch.zeros_like(new)))
