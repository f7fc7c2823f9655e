"""DTU mesh evaluation on the GPU: the reference's ``dtu_eval/eval.py`` (chamfer distances against the DTU ground truth)
and the mask culling of ``evaluate_dtu_mesh.py`` (``cull_mesh``), without Open3D, trimesh, scikit-image or scikit-learn.

    from rade_gs_b200 import dtu_eval, ply_io
    vertices, faces = ply_io.load_triangle_mesh_ply("recon.ply")
    vertices, faces, _ = dtu_eval.cull_mesh(scene.getTrainCameras(), vertices, faces)
    ...                                                    # the reference's alignment, in numpy
    r = dtu_eval.evaluate((vertices, faces), **dtu_eval.load_scan(dtu_dir, scan), mode="mesh", seed=0)
    print(r.mean_d2s, r.mean_s2d, r.overall)

or, for files, ``python -m rade_gs_b200.dtu_eval`` with eval.py's arguments (plus ``--seed``).

All arithmetic is fp64 and follows the reference's expressions; the contract is stated at ``rgs_dtu_*`` in
include/rgs_b200.h and the kernels are in csrc/rgs_dtu_eval.cu.  Sampling, the kept set of the radius downsample and the
nearest-neighbour distances are bit-identical to the reference's for the same shuffle; the means agree to the last few
bits (their summation order differs).  Deliberate differences:

* the shuffle: eval.py shuffles with an unseeded ``np.random.default_rng()``, so its own numbers change from run to run.
  Here the order is ``torch.randperm`` on the device, seeded by ``seed``, or an explicit ``perm``;
* culling takes ``world_view_transform.T`` as the world->camera matrix as given, and evaluates the projection in fp64 with
  fx, fy unrounded; the reference inverts that matrix twice and projects in fp32, so a vertex whose projection lies within
  about 1e-3 px of a pixel-rounding or image-border boundary may fall the other way;
* an empty query set yields empty distances and a NaN mean (scikit-learn refuses 0 queries).

Inputs with a NaN or infinite coordinate raise ``ValueError`` (scikit-learn's ``fit`` does too), and so does an empty
reference set.  There is no CPU path: the work runs on a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import math
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from diff_gaussian_rasterization import _C

from . import ply_io


def _device(device) -> torch.device:
    d = torch.device(device)
    if d.type != "cuda":
        raise RuntimeError("mesh evaluation runs on a CUDA device: there is no CPU path")
    return d


def _points(x, device, name: str) -> torch.Tensor:
    t = x.detach() if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))
    t = t.to(device=device, dtype=torch.float64)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be [N, 3], got {tuple(t.shape)}")
    if t.numel() and not bool(torch.isfinite(t).all()):
        raise ValueError(f"{name} has NaN or infinite coordinates")
    return t.contiguous()


def sample_mesh_points(vertices, faces, density: float = 0.2, device="cuda") -> torch.Tensor:
    """eval.py's ``data_pcd`` before the shuffle (eval.py:54-71): every vertex in order, then the samples of every triangle
    of nonzero area in triangle order, float64 [V + S, 3] on the device."""
    dev = _device(device)
    v = _points(vertices, dev, "vertices")
    f = faces.detach() if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces))
    f = f.to(dev).reshape(-1, 3)
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError("face index out of [0, V)")
    return _C.dtu_sample_mesh(v, f.to(torch.int32).contiguous(), float(density))


def shuffle_permutation(n: int, seed: Optional[int] = None, device="cuda") -> torch.Tensor:
    """The processing order of the downsample: ``torch.randperm(n)`` on the device, seeded when ``seed`` is given."""
    dev = _device(device)
    if seed is None:
        return torch.randperm(n, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(int(seed))
    return torch.randperm(n, device=dev, generator=g)


@dataclass
class Downsampled:
    points: torch.Tensor    # float64 [K, 3]: the kept points, in shuffled order (eval.py's data_down)
    perm: torch.Tensor      # int64 [N]: shuffled[i] = input[perm[i]]
    kept: torch.Tensor      # bool [N] over the shuffled order
    rounds: int             # decision rounds the GPU needed


def radius_downsample(points, radius: float, seed: Optional[int] = None, perm=None, device="cuda") -> Downsampled:
    """eval.py:80-94: shuffle, then keep each point that no earlier kept point lies within ``radius`` of (d <= radius).
    The kept set is exactly the reference's for the same order."""
    dev = _device(device)
    p = _points(points, dev, "points")
    n = p.shape[0]
    if perm is None:
        perm = shuffle_permutation(n, seed, dev)
    else:
        perm = torch.as_tensor(perm).to(device=dev, dtype=torch.int64).reshape(-1)
        if perm.numel() != n or not torch.equal(torch.sort(perm).values, torch.arange(n, device=dev)):
            raise ValueError("perm must be a permutation of range(len(points))")
    shuffled = p[perm].contiguous()
    kept, rounds = _C.dtu_radius_downsample(shuffled, float(radius))
    return Downsampled(shuffled[kept], perm, kept, int(rounds))


def nearest_distances(reference, query, device="cuda"):
    """(distance float64 [N], index int64 [N]): for each query point its exact Euclidean distance to the nearest reference
    point (eval.py's ``kneighbors(n_neighbors=1)``) and the index of one such point."""
    dev = _device(device)
    r, q = _points(reference, dev, "reference"), _points(query, dev, "query")
    if r.shape[0] == 0:
        raise ValueError("the reference set is empty")
    return _C.dtu_nearest(r, q)


# ---- culling (evaluate_dtu_mesh.py:82-138) ------------------------------------------------------------------------------

def _fov2focal(fov: float, pixels: int) -> float:
    return pixels / (2 * math.tan(fov / 2))


def cull_projections(cameras) -> np.ndarray:
    """float64 [n, 3, 4]: rows 0..2 of K @ w2c per camera, with the reference's K (fx, fy, W / 2, H / 2) and
    w2c = world_view_transform.T, each entry summed left to right."""
    out = np.zeros((len(cameras), 3, 4), np.float64)
    for n, cam in enumerate(cameras):
        wvt = cam.world_view_transform
        w2c = (wvt.detach().cpu().double().numpy() if isinstance(wvt, torch.Tensor) else np.asarray(wvt, np.float64)).T
        K = np.eye(4)
        K[0, 0] = _fov2focal(cam.FoVx, cam.image_width)
        K[1, 1] = _fov2focal(cam.FoVy, cam.image_height)
        K[0, 2] = cam.image_width / 2.0
        K[1, 2] = cam.image_height / 2.0
        for r in range(3):
            out[n, r] = ((K[r, 0] * w2c[0] + K[r, 1] * w2c[1]) + K[r, 2] * w2c[2]) + K[r, 3] * w2c[3]
    return out


def cull_masks(cameras, device="cuda") -> torch.Tensor:
    """uint8 [n, H, W]: each camera's ``gt_mask[0] > 0``."""
    dev = _device(device)
    ms = []
    for cam in cameras:
        m = cam.gt_mask if isinstance(cam.gt_mask, torch.Tensor) else torch.as_tensor(np.asarray(cam.gt_mask))
        ms.append((m.reshape(-1, m.shape[-2], m.shape[-1])[0] > 0).to(dev, torch.uint8))
    if len({tuple(m.shape) for m in ms}) > 1:
        raise ValueError("every camera's mask must have the same size")
    return torch.stack(ms)


def cull_mesh(cameras, vertices, faces, device="cuda"):
    """The reference's ``cull_mesh``: keep the vertices that every camera either does not see or sees inside its mask
    dilated by disk(6), and the faces whose three vertices are all kept, both renumbered in their original order.
    ``cameras`` carry ``world_view_transform``, ``FoVx``, ``FoVy``, ``image_width``, ``image_height`` and ``gt_mask``
    (the reference's Camera objects).  Returns (vertices float64 [V', 3], faces int64 [F', 3], keep bool [V])."""
    dev = _device(device)
    v = _points(vertices, dev, "vertices")
    f = (faces.detach() if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces))).to(dev, torch.int64).reshape(-1, 3)
    if len(cameras):
        for cam in cameras:
            if (cam.image_height, cam.image_width) != tuple(cam.gt_mask.shape[-2:]):
                raise ValueError("gt_mask must be [.., image_height, image_width]")
        dil = _C.dtu_dilate_masks(cull_masks(cameras, dev))
        keep = _C.dtu_cull_vertices(v, torch.as_tensor(cull_projections(cameras), device=dev), dil)
    else:
        keep = torch.ones(v.shape[0], dtype=torch.bool, device=dev)
    new_index = torch.cumsum(keep.to(torch.int64), 0) - 1
    face_keep = keep[f].all(dim=1) if f.numel() else torch.zeros(0, dtype=torch.bool, device=dev)
    return v[keep], new_index[f[face_keep]], keep


# ---- evaluation (eval.py:96-166) ----------------------------------------------------------------------------------------

@dataclass
class DTUResult:
    mean_d2s: float
    mean_s2d: float
    overall: float
    dist_d2s: torch.Tensor      # float64 [K]: each ObsMask point of the data to the STL cloud
    dist_s2d: torch.Tensor      # float64 [L]: each STL point above the ground plane to the in-box data
    data_down: torch.Tensor     # float64 [D, 3] downsampled data (shuffled order)
    data_color: torch.Tensor    # float64 [D, 3] eval.py's visualisation colours
    stl: torch.Tensor           # float64 [M, 3]
    stl_color: torch.Tensor     # float64 [M, 3]
    perm: torch.Tensor          # int64: the shuffle
    kept: torch.Tensor          # bool over the shuffled order
    in_obs: torch.Tensor        # int64: indices into data_down of the points scored by dist_d2s
    above: torch.Tensor         # bool [M]: STL points above the ground plane


def load_scan(dataset_dir: str, scan: int) -> dict:
    """The ground truth eval.py reads: ObsMask{scan}_10.mat (ObsMask, BB, Res), Plane{scan}.mat (P) and the STL cloud."""
    from scipy.io import loadmat
    m = loadmat(f"{dataset_dir}/ObsMask/ObsMask{scan}_10.mat")
    plane = loadmat(f"{dataset_dir}/ObsMask/Plane{scan}.mat")["P"]
    stl = ply_io.load_point_cloud_ply(f"{dataset_dir}/Points/stl/stl{scan:03}_total.ply")
    return {"stl": stl, "obs_mask": m["ObsMask"], "bb": m["BB"], "res": m["Res"], "plane": plane}


def _blend(alpha: torch.Tensor) -> torch.Tensor:
    """R * alpha + W * (1 - alpha) as numpy evaluates it, with R = (1, 0, 0) and W = (1, 1, 1)."""
    a = alpha[:, None]
    R = torch.tensor([[1.0, 0.0, 0.0]], dtype=torch.float64, device=a.device)
    return R * a + 1.0 * (1 - a)


def evaluate(data, stl, obs_mask, bb, res, plane, *, mode: str = "mesh", downsample_density: float = 0.2, patch_size: float = 60,
             max_dist: float = 20, visualize_threshold: float = 10, seed: Optional[int] = None, perm=None, device="cuda") -> DTUResult:
    """eval.py from its inputs.  ``data`` is (vertices, faces) for mode "mesh" and an [N, 3] cloud for mode "pcd"; ``stl``,
    ``obs_mask``, ``bb``, ``res`` and ``plane`` are the ground truth (``load_scan``)."""
    dev = _device(device)
    if mode == "mesh":
        vertices, faces = data
        pcd = sample_mesh_points(vertices, faces, downsample_density, dev)
    elif mode == "pcd":
        pcd = _points(data, dev, "data")
    else:
        raise ValueError(f"mode must be 'mesh' or 'pcd', got {mode!r}")
    ds = radius_downsample(pcd, downsample_density, seed=seed, perm=perm, device=dev)
    down = ds.points

    # masking (eval.py:96-110): BB is cast to float32 and the patch bounds are float32 arithmetic, as numpy does
    bb32 = torch.as_tensor(np.asarray(bb, dtype=np.float32).reshape(2, 3), device=dev)
    patch = float(patch_size)
    lo, hi = (bb32[:1] - patch).double(), (bb32[1:] + patch * 2).double()
    inbound = ((down >= lo) & (down < hi)).all(dim=-1)
    data_in = down[inbound]
    res64 = torch.as_tensor(np.asarray(res, dtype=np.float64), device=dev)
    grid = torch.round((data_in - bb32[:1].double()) / res64).to(torch.int32)
    mask = torch.as_tensor(np.asarray(obs_mask).astype(bool), device=dev)
    shape = torch.tensor(mask.shape, dtype=torch.int32, device=dev)
    grid_inbound = ((grid >= 0) & (grid < shape)).all(dim=-1)
    g = grid[grid_inbound].long()
    in_obs = mask[g[:, 0], g[:, 1], g[:, 2]]
    data_in_obs = data_in[grid_inbound][in_obs]

    stl_t = _points(stl, dev, "stl")
    md = float(max_dist)
    dist_d2s = nearest_distances(stl_t, data_in_obs, dev)[0] if data_in_obs.shape[0] else torch.zeros(0, dtype=torch.float64, device=dev)
    mean_d2s = float(dist_d2s[dist_d2s < md].mean())

    # ground plane (eval.py:126-130): (P * [x, y, z, 1]).sum(-1), summed left to right
    P = torch.as_tensor(np.asarray(plane, dtype=np.float64).reshape(4), device=dev)
    above = (((P[0] * stl_t[:, 0] + P[1] * stl_t[:, 1]) + P[2] * stl_t[:, 2]) + P[3] * 1.0) > 0
    stl_above = stl_t[above]
    if data_in.shape[0] == 0:
        raise ValueError("no downsampled point lies inside the bounding box: the stl -> data reference set is empty")
    dist_s2d = nearest_distances(data_in, stl_above, dev)[0]
    mean_s2d = float(dist_s2d[dist_s2d < md].mean())

    # visualisation colours (eval.py:136-152)
    vis = float(visualize_threshold)
    vis_t = torch.tensor(vis, dtype=torch.float64, device=dev)   # a device divisor: torch divides by a host scalar through its reciprocal
    B = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64, device=dev)
    G = torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64, device=dev)
    idx = torch.nonzero(inbound).flatten()[grid_inbound][in_obs]
    data_color = B.repeat(down.shape[0], 1)
    data_color[idx] = _blend(dist_d2s.clamp(max=vis) / vis_t)
    data_color[idx[dist_d2s >= md]] = G
    stl_color = B.repeat(stl_t.shape[0], 1)
    aidx = torch.nonzero(above).flatten()
    stl_color[aidx] = _blend(dist_s2d.clamp(max=vis) / vis_t)
    stl_color[aidx[dist_s2d >= md]] = G
    return DTUResult(mean_d2s, mean_s2d, (mean_d2s + mean_s2d) / 2, dist_d2s, dist_s2d, down, data_color, stl_t, stl_color, ds.perm, ds.kept, idx,
                     above)


def main(argv=None) -> dict:
    parser = argparse.ArgumentParser(description="DTU chamfer evaluation on the GPU (dtu_eval/eval.py)")
    parser.add_argument("--data", type=str, default="data_in.ply")
    parser.add_argument("--scan", type=int, default=1)
    parser.add_argument("--mode", type=str, default="mesh", choices=["mesh", "pcd"])
    parser.add_argument("--dataset_dir", type=str, default=".")
    parser.add_argument("--vis_out_dir", type=str, default=".")
    parser.add_argument("--downsample_density", type=float, default=0.2)
    parser.add_argument("--patch_size", type=float, default=60)
    parser.add_argument("--max_dist", type=float, default=20)
    parser.add_argument("--visualize_threshold", type=float, default=10)
    parser.add_argument("--seed", type=int, default=None, help="seed of the downsample's shuffle (default: unseeded, as eval.py)")
    args = parser.parse_args(argv)

    data = ply_io.load_triangle_mesh_ply(args.data) if args.mode == "mesh" else ply_io.load_point_cloud_ply(args.data)
    r = evaluate(data, **load_scan(args.dataset_dir, args.scan), mode=args.mode, downsample_density=args.downsample_density,
                 patch_size=args.patch_size, max_dist=args.max_dist, visualize_threshold=args.visualize_threshold, seed=args.seed)
    os.makedirs(args.vis_out_dir, exist_ok=True)
    ply_io.save_point_cloud_ply(f"{args.vis_out_dir}/vis_{args.scan:03}_d2s.ply", r.data_down, r.data_color)
    ply_io.save_point_cloud_ply(f"{args.vis_out_dir}/vis_{args.scan:03}_s2d.ply", r.stl, r.stl_color)
    print(r.mean_d2s, r.mean_s2d, r.overall)
    out = {"mean_d2s": r.mean_d2s, "mean_s2d": r.mean_s2d, "overall": r.overall}
    with open(f"{args.vis_out_dir}/results.json", "w") as fp:
        json.dump(out, fp, indent=True)
    return out


if __name__ == "__main__":
    main()
