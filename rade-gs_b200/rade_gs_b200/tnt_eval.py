"""Tanks and Temples mesh evaluation on the GPU: the reference's ``eval_tnt/run.py`` (trajectory alignment, three ICP
refinement stages, precision / recall / F-score against the ground-truth cloud), without Open3D, trimesh or matplotlib.

    from rade_gs_b200 import ply_io, tnt_eval
    scene = tnt_eval.load_scene(dataset_dir)                   # <scene>.ply, .json, _trans.txt, _COLMAP_SfM.log, tau
    vertices, faces = ply_io.load_triangle_mesh_ply("recon.ply")
    traj = tnt_eval.load_trajectory("traj.log")
    r = tnt_eval.evaluate(tnt_eval.mesh_points(vertices, faces), traj=traj, seed=0, **scene)
    print(r.precision, r.recall, r.fscore)

or, for files, ``python -m rade_gs_b200.tnt_eval`` with run.py's arguments (plus ``--seed``).

The contracts of the device steps (crop, voxel downsample, ICP moments, in-place transform) are stated at ``rgs_tnt_*``
in include/rgs_b200.h; the kernels are in csrc/rgs_tnt_eval.cu, and every nearest-neighbour query goes through
``rgs_dtu_nearest`` (exact fp64 1-NN).  The 3x3 SVD of each ICP update and the RANSAC of the trajectory alignment run on
the host in numpy fp64.  Deliberate differences from the reference:

* the RANSAC of the trajectory alignment is seeded (``seed``) and always runs all ``max_iteration`` hypotheses with no
  early stop on confidence and no refinement; Open3D seeds its own and its result changes from run to run;
* voxel-downsampled clouds come out in ascending voxel-key order (Open3D's follow its hash map), which moves only the last
  bits of the ICP sums; each voxel's mean is Open3D's bit for bit;
* the crop's boundary rule and the strict correspondence test (``d < threshold``) are stated in the header; Open3D was not
  available to confirm either, so points exactly on a polygon edge, or exactly at the threshold, may be decided otherwise;
* the precision / recall PLYs carry no normals (``estimate_normals`` feeds no number);
* the mesh is taken as read: duplicate vertices are not merged (trimesh merges them on load);
* when precision and recall are both 0 the F-score is 0 (the reference divides by zero);
* the ``hot_r`` colour table is derived here from matplotlib's segment data (``_hot_r_table``) and was not checked
  against matplotlib itself;
* the reference's ``.json`` trajectory branch (broken there: it calls names it never imports) is not supported.

Inputs with a NaN or infinite coordinate raise ``ValueError``.  There is no CPU path: the work runs on a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from diff_gaussian_rasterization import _C

from . import ply_io
from .dtu_eval import _device, _points, nearest_distances  # noqa: F401  (nearest_distances is part of this module's API)

# eval_tnt/config.py: the scenes' distance threshold tau (metres)
SCENES_TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Church": 0.025, "Courthouse": 0.025, "Ignatius": 0.003, "Meetingroom": 0.01, "Truck": 0.005}
MAX_POINT_NUMBER = 4e6   # registration.py: the last stage keeps every k-th point above this many
PLOT_STRETCH = 5


def _transform(T, name: str = "transform") -> np.ndarray:
    T = np.asarray(T, np.float64)
    if T.shape != (4, 4):
        raise ValueError(f"{name} must be 4x4, got {T.shape}")
    if not np.isfinite(T).all():
        raise ValueError(f"{name} has NaN or infinite entries")
    if not np.array_equal(T[3], [0.0, 0.0, 0.0, 1.0]):
        raise ValueError(f"{name}'s last row must be (0 0 0 1)")
    return T


def apply_transform(T, points) -> np.ndarray:
    """numpy: the header's transform, p'_r = ((T_r0 x + T_r1 y) + T_r2 z) + T_r3 (Open3D's PointCloud.transform)."""
    p = np.asarray(points, np.float64)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)


# ---- inputs ---------------------------------------------------------------------------------------------------------------

def mesh_points(vertices, faces, device="cuda") -> torch.Tensor:
    """run.py:95-108: the mesh's vertices followed by every face's centroid ((v0 + v1) + v2) / 3, float64 [V + F, 3]."""
    dev = _device(device)
    v = _points(vertices, dev, "vertices")
    f = (faces.detach() if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces))).to(dev, torch.int64).reshape(-1, 3)
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError("face index out of [0, V)")
    three = torch.tensor(3.0, dtype=torch.float64, device=dev)   # a device divisor: torch divides by a host scalar through its reciprocal
    return torch.cat([v, ((v[f[:, 0]] + v[f[:, 1]]) + v[f[:, 2]]) / three]).contiguous()


def read_trajectory(path: str) -> np.ndarray:
    """A ``.log`` trajectory (trajectory_io.read_trajectory): per camera one metadata line and four matrix rows.
    Returns float64 [n, 4, 4]."""
    poses = []
    with open(path, "r") as f:
        lines = f.read().splitlines()
    k = 0
    while k < len(lines):
        if not lines[k].strip():
            k += 1
            continue
        if k + 5 > len(lines):
            raise ValueError(f"{path}: truncated pose at line {k + 1}")
        rows = [np.array(lines[k + 1 + i].replace("\t", " ").split(), dtype=np.float64) for i in range(4)]
        if any(r.shape != (4,) for r in rows):
            raise ValueError(f"{path}: a pose row does not hold 4 numbers near line {k + 2}")
        poses.append(np.stack(rows))
        k += 5
    return np.array(poses, dtype=np.float64).reshape(-1, 4, 4)


def load_trajectory(path: str) -> np.ndarray:
    """run.py's estimated trajectory: ``.npy`` (np.load, [n, 4, 4]) or ``.log``; float64 [n, 4, 4]."""
    if path.endswith(".json"):
        raise ValueError("the .json trajectory format is not supported (the reference's branch for it does not run either)")
    t = np.load(path) if path.endswith(".npy") else read_trajectory(path)
    t = np.asarray(t, np.float64)
    if t.ndim != 3 or t.shape[1:] != (4, 4):
        raise ValueError(f"{path}: a trajectory must be [n, 4, 4], got {t.shape}")
    return t


@dataclass
class CropVolume:
    orthogonal_axis: int        # 0 / 1 / 2 for X / Y / Z
    axis_min: float
    axis_max: float
    polygon: np.ndarray         # float64 [K, 2]: the two other axes in increasing order


def load_crop_volume(path: str) -> CropVolume:
    """An Open3D ``SelectionPolygonVolume`` JSON file (the reference's <scene>.json)."""
    with open(path) as f:
        d = json.load(f)
    try:
        axis = "XYZ".index(str(d["orthogonal_axis"]).upper())
        poly = np.asarray(d["bounding_polygon"], np.float64).reshape(-1, 3)
        lo, hi = float(d["axis_min"]), float(d["axis_max"])
    except (KeyError, ValueError) as e:
        raise ValueError(f"{path}: not a SelectionPolygonVolume ({e})") from None
    if len(poly) < 3 or not np.isfinite(poly).all():
        raise ValueError(f"{path}: the bounding polygon needs at least 3 finite vertices")
    uv = [a for a in range(3) if a != axis]
    return CropVolume(axis, lo, hi, np.ascontiguousarray(poly[:, uv]))


def load_scene(dataset_dir: str, scene: Optional[str] = None) -> dict:
    """What run.py reads from a dataset directory named after the scene: the GT cloud (<scene>.ply), the crop volume
    (<scene>.json), the GT alignment (<scene>_trans.txt), the COLMAP trajectory (<scene>_COLMAP_SfM.log) and tau."""
    scene = scene or os.path.basename(os.path.normpath(dataset_dir))
    if scene not in SCENES_TAU:
        raise ValueError(f"{dataset_dir}: scene {scene!r} is not one of {sorted(SCENES_TAU)}")
    j = lambda suffix: os.path.join(dataset_dir, scene + suffix)  # noqa: E731
    return {"gt": ply_io.load_point_cloud_ply(j(".ply")), "crop_volume": load_crop_volume(j(".json")), "gt_trans": np.loadtxt(j("_trans.txt")),
            "gt_traj": read_trajectory(j("_COLMAP_SfM.log")), "tau": SCENES_TAU[scene], "scene": scene}


# ---- device steps -----------------------------------------------------------------------------------------------------------

def crop(points, volume: Optional[CropVolume], transform=None, device="cuda"):
    """Transform (optional 4x4), then crop by ``volume`` (None: keep all).  Returns (cropped float64 [n, 3] in input order,
    kept bool [N] over the input)."""
    dev = _device(device)
    p = _points(points, dev, "points")
    T = torch.as_tensor(_transform(transform)) if transform is not None else torch.zeros(0, dtype=torch.float64)
    if volume is None:
        kept, out = _C.tnt_crop(p, T, 0, 0.0, 0.0, torch.zeros(0, dtype=torch.float64, device=dev))
    else:
        poly = torch.as_tensor(np.asarray(volume.polygon, np.float64).reshape(-1, 2), device=dev)
        if not (3 <= poly.shape[0] <= 2048):
            raise ValueError("the crop polygon needs 3 to 2048 vertices")
        kept, out = _C.tnt_crop(p, T, int(volume.orthogonal_axis), float(volume.axis_min), float(volume.axis_max), poly)
    return out, kept


def voxel_down_sample(points, voxel_size: float, device="cuda"):
    """Open3D's voxel_down_sample: (means float64 [V, 3] in ascending voxel-key order, counts int64 [V])."""
    dev = _device(device)
    if not (np.isfinite(voxel_size) and voxel_size > 0):
        raise ValueError("voxel_size must be positive and finite")
    p = _points(points, dev, "points")
    try:
        return _C.tnt_voxel_downsample(p, float(voxel_size))
    except RuntimeError as e:
        if "2^21" in str(e):
            raise ValueError(str(e)) from None
        raise


def uniform_down_sample(points, every_k: int) -> torch.Tensor:
    """Open3D's uniform_down_sample: points 0, k, 2k, ... in order."""
    if int(every_k) < 1:
        raise ValueError("every_k must be at least 1")
    out = points[::int(every_k)]
    return out.contiguous() if isinstance(out, torch.Tensor) else out


def uniform_for_registration(points) -> torch.Tensor:
    """registration.py's "uniform" branch: every k-th point, k = int(round(n / 4e6)), only above 4e6 points."""
    n = len(points)
    return uniform_down_sample(points, int(round(n / float(MAX_POINT_NUMBER)))) if n > MAX_POINT_NUMBER else points


def icp_moments(source, target, dist, index, threshold: float) -> np.ndarray:
    """The 18 moments of the header's rgs_tnt_icp_moments (float64 numpy)."""
    return _C.tnt_icp_moments(source, target, dist, index, float(threshold)).numpy()


def umeyama(moments) -> np.ndarray:
    """Eigen's umeyama with scaling from the moments: SVD of sigma = U D V^T, S = diag(1, 1, -1) when det(U) det(V) < 0,
    R = U S V^T, c = (1 / var_s) * (D . S), t = mt - (c R) ms.  No correspondence: the identity."""
    m = np.asarray(moments, np.float64)
    T = np.eye(4)
    if m[0] == 0:
        return T
    ms, mt, sigma, var = m[2:5], m[5:8], m[8:17].reshape(3, 3), m[17]
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    c = (1.0 / var) * D.dot(S)
    T[:3, 3] = mt - (c * R) @ ms
    T[:3, :3] = c * R
    return T


@dataclass
class ICPResult:
    transformation: np.ndarray
    fitness: float
    inlier_rmse: float
    iterations: int
    history: List[np.ndarray] = field(default_factory=list)   # the transformation after each iteration


def _evaluate(src, target, threshold):
    d, idx = _C.dtu_nearest(target, src)
    m = icp_moments(src, target, d, idx, threshold)
    n = m[0]
    fitness = n / src.shape[0] if src.shape[0] else 0.0
    rmse = float(np.sqrt(m[1] / n)) if n else 0.0
    return m, fitness, rmse


def icp(source, target, threshold: float, init=None, max_iteration: int = 30, relative_fitness: float = 1e-6, relative_rmse: float = 1e-6,
        device="cuda") -> ICPResult:
    """Open3D's registration_icp with TransformationEstimationPointToPoint(True): evaluate once, then per iteration the
    Umeyama update of the current correspondences, T <- update T, the source transformed in place by the update, and a
    new evaluation; stop when both |d fitness| < relative_fitness and |d rmse| < relative_rmse."""
    dev = _device(device)
    src = _points(source, dev, "source").clone()
    tgt = _points(target, dev, "target")
    if tgt.shape[0] == 0:
        raise ValueError("the target cloud is empty")
    T = np.eye(4) if init is None else _transform(init, "init").copy()
    if not np.array_equal(T, np.eye(4)):
        _C.tnt_transform(src, torch.as_tensor(T))
    m, fitness, rmse = _evaluate(src, tgt, threshold)
    history, it = [], 0
    for it in range(1, int(max_iteration) + 1):
        update = umeyama(m)
        T = update @ T
        history.append(T.copy())
        _C.tnt_transform(src, torch.as_tensor(update))
        prev = (fitness, rmse)
        m, fitness, rmse = _evaluate(src, tgt, threshold)
        if abs(prev[0] - fitness) < relative_fitness and abs(prev[1] - rmse) < relative_rmse:
            break
    return ICPResult(T, fitness, rmse, it, history)


# ---- trajectory alignment (registration.py:66-110) -----------------------------------------------------------------------

def ransac_hypotheses(n: int, count: int, ransac_n: int, seed: int) -> np.ndarray:
    """int64 [count, ransac_n]: rows of distinct correspondence indices.  numpy's default_rng(seed) draws every row
    uniformly with integers(0, n); rows holding a repeat are redrawn together, in row order, until none is left."""
    if n < ransac_n:
        raise ValueError(f"RANSAC needs at least {ransac_n} correspondences, got {n}")
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, n, (count, ransac_n))
    while True:
        s = np.sort(idx, axis=1)
        dup = (s[:, 1:] == s[:, :-1]).any(axis=1)
        if not dup.any():
            return idx
        idx[dup] = rng.integers(0, n, (int(dup.sum()), ransac_n))


def umeyama_batch(src, dst) -> np.ndarray:
    """Eigen's umeyama with scaling for a batch: src, dst [B, k, 3] -> [B, 4, 4] (degenerate samples give NaN)."""
    k = src.shape[1]
    inv = 1.0 / k
    ms, md = src.sum(axis=1) * inv, dst.sum(axis=1) * inv
    sc, dc = src - ms[:, None], dst - md[:, None]
    var = (sc * sc).sum(axis=(1, 2)) * inv
    sigma = inv * np.einsum("bki,bkj->bij", dc, sc)
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones((len(src), 3))
    S[np.linalg.det(U) * np.linalg.det(Vt) < 0, 2] = -1.0
    R = U @ (S[:, :, None] * Vt)
    with np.errstate(all="ignore"):
        c = (1.0 / var) * (D * S).sum(axis=1)
    T = np.zeros((len(src), 4, 4))
    T[:, 3, 3] = 1.0
    cR = c[:, None, None] * R
    T[:, :3, :3] = cR
    T[:, :3, 3] = md - np.einsum("bij,bj->bi", cR, ms)
    return T


def trajectory_alignment(traj, gt_traj, gt_trans, seed: int = 0, max_iteration: int = 100000, max_distance: float = 0.2, ransac_n: int = 6) -> np.ndarray:
    """registration_ransac_based_on_correspondence of the camera centres: estimated centre i against GT centre i
    (transformed by gt_trans) for every GT camera.  All ``max_iteration`` hypotheses of ``ransac_n`` distinct
    correspondences are fitted with scaled Umeyama; a correspondence is an inlier when |T s - t| < max_distance; the best
    hypothesis has the most inliers, then the lowest inlier RMSE, then the lowest index.  No refinement."""
    traj, gt_traj = np.asarray(traj, np.float64), np.asarray(gt_traj, np.float64)
    n = len(gt_traj)
    if len(traj) < n:
        raise ValueError(f"the estimated trajectory has {len(traj)} cameras, fewer than the {n} of the GT trajectory")
    src = np.ascontiguousarray(traj[:n, :3, 3])
    dst = apply_transform(_transform(gt_trans, "gt_trans"), gt_traj[:, :3, 3]) if gt_trans is not None else gt_traj[:, :3, 3].copy()
    hyp = ransac_hypotheses(n, int(max_iteration), ransac_n, seed)
    best = (-1, np.inf, -1, None)
    chunk = max(1, 2_000_000 // max(n, 1))
    for b0 in range(0, len(hyp), chunk):
        h = hyp[b0:b0 + chunk]
        T = umeyama_batch(src[h], dst[h])
        with np.errstate(all="ignore"):
            moved = np.einsum("bij,nj->bni", T[:, :3, :3], src) + T[:, None, :3, 3]
            d2 = ((moved - dst[None]) ** 2).sum(axis=2)
            inl = np.sqrt(d2) < max_distance
            cnt = inl.sum(axis=1)
            rmse = np.sqrt(np.where(inl, d2, 0.0).sum(axis=1) / np.maximum(cnt, 1))
        order = np.lexsort((np.arange(len(h)), rmse, -cnt))[0]
        if cnt[order] > best[0] or (cnt[order] == best[0] and rmse[order] < best[1]):
            best = (int(cnt[order]), float(rmse[order]), b0 + int(order), T[order])
    if best[0] <= 0:
        return np.eye(4)
    return best[3]


# ---- histogram, F-score and colours (evaluation.py:60-215) -----------------------------------------------------------------

def _segment_lut(data, N=256) -> np.ndarray:
    """matplotlib's _create_lookup_table for segment data (x, y0, y1) with gamma 1."""
    a = np.asarray(data, np.float64)
    x, y0, y1 = a[:, 0], a[:, 1], a[:, 2]
    xind = np.linspace(0, 1, N) ** 1.0
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


# matplotlib's "hot" segment data (_cm.py); "hot_r" reverses every channel as LinearSegmentedColormap.reversed() does:
# (1 - x, y1, y0) over the segments in reverse order, then the 256-entry table is built from the reversed segments.
_HOT = {"red": ((0.0, 0.0416, 0.0416), (0.365079, 1.0, 1.0), (1.0, 1.0, 1.0)),
        "green": ((0.0, 0.0, 0.0), (0.365079, 0.0, 0.0), (0.746032, 1.0, 1.0), (1.0, 1.0, 1.0)),
        "blue": ((0.0, 0.0, 0.0), (0.746032, 0.0, 0.0), (1.0, 1.0, 1.0))}


def _hot_r_table() -> np.ndarray:
    """float64 [256, 3]: matplotlib's hot_r lookup table, derived from the segment data (not checked against matplotlib)."""
    rev = {k: [(1.0 - x, y1, y0) for x, y0, y1 in reversed(v)] for k, v in _HOT.items()}
    return np.stack([_segment_lut(rev[k]) for k in ("red", "green", "blue")], axis=1)


def distance_colors(dist: torch.Tensor, max_distance: float) -> torch.Tensor:
    """evaluation.py's write_color_distances: hot_r(min(d, max_distance) / max_distance), float64 [N, 3].  Colormap
    lookup as matplotlib does it: index floor(v * 256), 256 -> 255."""
    dev = dist.device
    md = torch.tensor(float(max_distance), dtype=torch.float64, device=dev)
    v = torch.minimum(dist, md) / md
    xa = v * 256.0
    xa = torch.where(xa == 256.0, torch.full_like(xa, 255.0), xa)
    idx = xa.clamp(min=0).to(torch.int64).clamp(max=255)
    return torch.as_tensor(_hot_r_table(), device=dev)[idx]


def histogram_edges(tau: float, plot_stretch: float = PLOT_STRETCH) -> np.ndarray:
    return np.arange(0, tau * plot_stretch, tau / 100)


def cumulative_histogram(dist: torch.Tensor, edges: np.ndarray) -> np.ndarray:
    """np.histogram(dist, edges) (bins half-open on the right except the last, which is closed; values outside dropped),
    then np.cumsum(hist).astype(float) / len(dist)."""
    e = torch.as_tensor(edges, device=dist.device)
    nb = len(edges) - 1
    b = torch.searchsorted(e, dist, right=True) - 1
    b = torch.where(dist == e[-1], torch.full_like(b, nb - 1), b)
    ok = (b >= 0) & (b < nb)
    hist = torch.bincount(b[ok], minlength=nb).cpu().numpy()
    return np.cumsum(hist).astype(float) / len(dist)


def f_score(d_source: torch.Tensor, d_target: torch.Tensor, tau: float):
    """get_f1_score_histo2's precision, recall and F (0 when both are 0)."""
    if len(d_source) == 0 or len(d_target) == 0:
        return 0, 0, 0
    recall = float(int((d_target < tau).sum())) / float(len(d_target))
    precision = float(int((d_source < tau).sum())) / float(len(d_source))
    fscore = 2 * recall * precision / (recall + precision) if recall + precision > 0 else 0.0
    return precision, recall, fscore


# ---- the whole evaluation (run.py:58-209) --------------------------------------------------------------------------------

@dataclass
class StageResult:
    transformation: np.ndarray
    fitness: float
    inlier_rmse: float
    iterations: int
    source_points: int
    target_points: int


@dataclass
class TNTResult:
    precision: float
    recall: float
    fscore: float
    transformation: np.ndarray        # the final estimated -> GT transform
    alignment: np.ndarray             # the RANSAC trajectory alignment
    stages: List[StageResult]         # the three ICP stages
    dist_source: torch.Tensor         # float64: each evaluated source point to the GT (precision)
    dist_target: torch.Tensor         # float64: each evaluated GT point to the source (recall)
    edges_source: np.ndarray
    cum_source: np.ndarray
    edges_target: np.ndarray
    cum_target: np.ndarray
    source: torch.Tensor              # float64 [S, 3]: the evaluated source cloud (transformed, cropped, voxel tau / 2)
    target: torch.Tensor              # float64 [G, 3]: the evaluated GT cloud (cropped, voxel tau / 2)


def _stage(source, target, init, volume, voxel, threshold, max_itr, dev):
    s = crop(source, volume, init, dev)[0]
    s = voxel_down_sample(s, voxel, dev)[0] if voxel is not None else uniform_for_registration(s)
    r = icp(s, target, threshold, None, max_itr, device=dev)
    return StageResult(r.transformation @ init, r.fitness, r.inlier_rmse, r.iterations, s.shape[0], target.shape[0])


def evaluate(source, gt, crop_volume: CropVolume, gt_trans, traj, gt_traj, tau: float, *, seed: int = 0, ransac_iterations: int = 100000,
             max_iteration: int = 20, scene: Optional[str] = None, verbose: bool = False, device="cuda") -> TNTResult:
    """run.py's run_evaluation from its inputs.  ``source`` is the reconstruction's cloud (``mesh_points``), ``gt`` the
    GT cloud, ``traj`` / ``gt_traj`` [n, 4, 4] trajectories (``load_scene`` gives the rest)."""
    dev = _device(device)
    src = _points(source, dev, "source")
    gt_t = _points(gt, dev, "gt")
    log = print if verbose else (lambda *a, **k: None)
    T0 = trajectory_alignment(traj, gt_traj, gt_trans, seed=seed, max_iteration=ransac_iterations)
    # the GT crop does not depend on the transform: crop once, reuse the tau / 2 cloud for stage 2 and the histogram
    gt_crop = crop(gt_t, crop_volume, None, dev)[0]
    if gt_crop.shape[0] == 0:
        raise ValueError("no GT point lies inside the crop volume")
    gt_tau = voxel_down_sample(gt_crop, tau, dev)[0]
    gt_half = voxel_down_sample(gt_crop, tau / 2.0, dev)[0]
    stages = []
    for voxel, thr, target in ((tau, tau * 80, gt_tau), (tau / 2.0, tau * 20, gt_half), (None, 2 * tau, uniform_for_registration(gt_crop))):
        if voxel is not None:
            log("[Registration] voxel_size: %f, threshold: %f" % (voxel, thr))
        else:
            log("[Registration] threshold: %f" % thr)
        init = stages[-1].transformation if stages else T0
        stages.append(_stage(src, target, init, crop_volume, voxel, thr, max_iteration, dev))
    T = stages[-1].transformation
    s = voxel_down_sample(crop(src, crop_volume, T, dev)[0], tau / 2.0, dev)[0]
    if s.shape[0] == 0:
        d1 = torch.zeros(0, dtype=torch.float64, device=dev)
        d2 = torch.full((gt_half.shape[0],), float("inf"), dtype=torch.float64, device=dev)
    else:
        d1 = _C.dtu_nearest(gt_half, s)[0]
        d2 = _C.dtu_nearest(s, gt_half)[0]
    precision, recall, fscore = f_score(d1, d2, tau)
    if len(d1) and len(d2):
        edges = histogram_edges(tau)
        es, cs, et, ct = edges, cumulative_histogram(d1, edges), edges, cumulative_histogram(d2, edges)
    else:
        es = cs = et = ct = np.array([0])
    return TNTResult(precision, recall, fscore, T, T0, stages, d1, d2, es, cs, et, ct, s, gt_half)


def write_outputs(r: TNTResult, out_dir: str, scene: str, tau: float) -> None:
    """evaluation.py's files: <scene>.precision.ply / .recall.ply (hot_r colours of min(d, 3 tau) / 3 tau),
    <scene>.precision.txt / .recall.txt (the cumulative histograms) and <scene>.prf_tau_plotstr.txt."""
    os.makedirs(out_dir, exist_ok=True)
    ply_io.save_point_cloud_ply(f"{out_dir}/{scene}.precision.ply", r.source, distance_colors(r.dist_source, 3 * tau))
    ply_io.save_point_cloud_ply(f"{out_dir}/{scene}.recall.ply", r.target, distance_colors(r.dist_target, 3 * tau))
    np.savetxt(f"{out_dir}/{scene}.recall.txt", r.cum_target)
    np.savetxt(f"{out_dir}/{scene}.precision.txt", r.cum_source)
    np.savetxt(f"{out_dir}/{scene}.prf_tau_plotstr.txt", np.array([r.precision, r.recall, r.fscore, tau, PLOT_STRETCH]))


def main(argv=None) -> dict:
    parser = argparse.ArgumentParser(description="Tanks and Temples evaluation on the GPU (eval_tnt/run.py)")
    parser.add_argument("--dataset-dir", type=str, required=True, help="scene directory holding <scene>.json, <scene>.ply, ...")
    parser.add_argument("--traj-path", type=str, required=True, help="estimated trajectory (.log or .npy)")
    parser.add_argument("--ply-path", type=str, required=True, help="reconstruction mesh (PLY)")
    parser.add_argument("--out-dir", type=str, default="", help="default: <ply dir>/evaluation")
    parser.add_argument("--view-crop", type=int, default=0, help="accepted for compatibility; no viewer is opened")
    parser.add_argument("--seed", type=int, default=0, help="seed of the trajectory alignment's RANSAC (the reference's is unseeded)")
    args = parser.parse_args(argv)
    if args.out_dir.strip() == "":
        args.out_dir = os.path.join(os.path.dirname(args.ply_path), "evaluation")

    sc = load_scene(args.dataset_dir)
    scene, tau = sc.pop("scene"), sc["tau"]
    print("")
    print("===========================")
    print("Evaluating %s" % scene)
    print("===========================")
    print(args.ply_path)
    vertices, faces = ply_io.load_triangle_mesh_ply(args.ply_path)
    traj = load_trajectory(args.traj_path)
    r = evaluate(mesh_points(vertices, faces), traj=traj, seed=args.seed, verbose=True, **sc)
    write_outputs(r, args.out_dir, scene, tau)
    print("==============================")
    print("evaluation result : %s" % scene)
    print("==============================")
    print("distance tau : %.3f" % tau)
    print("precision : %.4f" % r.precision)
    print("recall : %.4f" % r.recall)
    print("f-score : %.4f" % r.fscore)
    print("==============================")
    return {"precision": r.precision, "recall": r.recall, "fscore": r.fscore, "transformation": r.transformation.tolist()}


if __name__ == "__main__":
    main()
