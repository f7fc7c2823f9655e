"""simple_knn drop-in on the GPU: distCUDA2 (rgs_knn.cu) bit-exact against the numpy fp32 brute-force oracle on hard cloud
families, against cKDTree (fp64) at the reference's sizes, deterministic, and free of quadratic cases."""
import time

import numpy as np
import pytest
import torch

from bench_knn import surface_cloud
from test_knn_host import kdtree_mean_dist2, knn_oracle

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _dist(points):
    from simple_knn._C import distCUDA2
    out = distCUDA2(torch.as_tensor(points).to(DEV))
    return out.cpu().numpy()


def cloud(family, P, seed=0):
    rng = np.random.default_rng([P, seed, sum(map(ord, family))])
    if family == "uniform":
        pts = rng.uniform(-1.3, 1.3, (P, 3))
    elif family == "clustered":            # Gaussian mixture plus 1 % far outliers, like a COLMAP sparse cloud
        centers = rng.uniform(-2, 2, (8, 3))
        pts = centers[rng.integers(0, 8, P)] + rng.normal(scale=0.03, size=(P, 3))
        out = rng.random(P) < 0.01
        pts[out] = rng.uniform(-60, 60, (out.sum(), 3))
    elif family == "surfaces":
        pts = surface_cloud(P, rng)
    elif family == "lattice":              # almost every distance is tied
        m = int(np.ceil(P ** (1 / 3)))
        g = np.stack(np.meshgrid(np.arange(m), np.arange(m), np.arange(m), indexing="ij"), -1).reshape(-1, 3)[:P]
        pts = rng.permutation(g) * 0.5
    elif family == "replacement":          # draws with replacement: exact duplicates
        base = rng.uniform(-1, 1, (max(1, P // 4), 3))
        pts = base[rng.integers(0, len(base), P)]
    elif family == "identical":
        pts = np.tile([[0.3, -0.7, 1.1]], (P, 1))
    elif family == "collinear":
        t = rng.uniform(-1, 1, (P, 1))
        pts = np.array([[0.1, 0.2, 0.3]]) + t * np.array([[1.0, 2.0, -0.5]])
    elif family == "translated":           # 1e-3 spacing far from the origin: fp32 precision at the last bits
        pts = 1e3 + rng.random((P, 3)) * (1e-3 * np.cbrt(P))
    else:
        raise ValueError(family)
    return np.ascontiguousarray(pts, dtype=np.float32)


FAMILIES = ["uniform", "clustered", "surfaces", "lattice", "replacement", "identical", "collinear", "translated"]
SIZES = [1, 2, 3, 4, 5, 31, 32, 33, 1000, 20000]


@pytest.mark.parametrize("P", SIZES)
@pytest.mark.parametrize("family", FAMILIES)
def test_bit_exact_against_oracle(family, P):
    pts = cloud(family, P)
    ours = _dist(pts)
    ref = knn_oracle(pts)
    assert ours.dtype == np.float32 and ours.shape == (P,)
    bad = np.flatnonzero(ours.view(np.uint32) != ref.view(np.uint32))
    assert bad.size == 0, f"{bad.size} rows differ, first {bad[:5]}: ours {ours[bad[:5]]} oracle {ref[bad[:5]]}"


def test_empty_cloud():
    from simple_knn._C import distCUDA2
    out = distCUDA2(torch.empty(0, 3, device=DEV))
    assert out.shape == (0,) and out.dtype == torch.float32 and out.is_cuda


@pytest.mark.parametrize("family,P", [("uniform", 1_000_000), ("clustered", 1_000_000), ("trimesh_fallback", 1_200_000)])
def test_against_kdtree_at_scale(family, P):
    """A wrong neighbour moves a value by far more than 2e-6 relative; a near-tie that fp32 resolves differently, by less."""
    if family == "trimesh_fallback":       # dataset_readers.py:233: 1.2 M draws with replacement from the mesh vertices
        rng = np.random.default_rng(12)
        verts = surface_cloud(300_000, rng).astype(np.float32)
        pts = verts[rng.integers(0, len(verts), P)]
    else:
        pts = cloud(family, P)
    ours = _dist(pts)
    ref = kdtree_mean_dist2(pts)
    err = np.abs(ours.astype(np.float64) - ref)
    assert np.all(err <= 2e-6 * ref), f"worst relative error {np.max(err / np.maximum(ref, 1e-300)):.3g}"
    assert np.all(ours[ref == 0.0] == 0.0)


def test_deterministic_and_permutation_invariant():
    pts = cloud("clustered", 200_000, seed=5)
    a, b = _dist(pts), _dist(pts)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    perm = np.random.default_rng(6).permutation(len(pts))
    c = _dist(pts[perm])
    assert np.array_equal(c.view(np.uint32), a[perm].view(np.uint32))


def test_non_finite_rows():
    pts = cloud("uniform", 5000, seed=7)
    rng = np.random.default_rng(8)
    bad = rng.choice(len(pts), 60, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    pts[bad, rng.integers(0, 3, len(bad))] = vals[rng.integers(0, 3, len(bad))]
    out = _dist(pts)
    assert np.isnan(out[bad]).all()
    keep = np.setdiff1d(np.arange(len(pts)), bad)
    alone = _dist(pts[keep])
    assert np.array_equal(out[keep].view(np.uint32), alone.view(np.uint32))
    assert np.array_equal(alone.view(np.uint32), knn_oracle(pts[keep]).view(np.uint32))
    # fewer than 4 finite points left, and none at all
    few = np.array([[0, 0, 0], [np.nan, 0, 0], [2, 0, 0], [0, np.inf, 0], [0, 3, 0]], np.float32)
    assert np.array_equal(_dist(few), knn_oracle(few), equal_nan=True)
    assert np.isnan(_dist(np.full((70, 3), np.nan, np.float32))).all()


@pytest.mark.parametrize("family", ["identical", "lattice"])
def test_no_quadratic_case_at_10m(family):
    """10 M identical points or a 10 M lattice: every box ties with the third-best distance.  A pruned search is expected far
    below the coarse 10 s bound, a quadratic one far above."""
    from simple_knn._C import distCUDA2
    distCUDA2(torch.rand(4096, 3, device=DEV))  # module load and allocator warm-up outside the timed call
    s = 0.25
    if family == "identical":
        x = torch.full((10_000_000, 3), 0.5, device=DEV)
    else:
        m = 216                                  # 216^3 = 10 077 696 points, spacing 0.25 (every distance exact in fp32)
        r = torch.arange(m, device=DEV, dtype=torch.float32) * s
        x = torch.stack(torch.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
        x = x[torch.randperm(len(x), device=DEV, generator=torch.Generator(DEV).manual_seed(9))]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = distCUDA2(x)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert dt < 10.0, f"{family}: {dt:.2f} s"
    want = 0.0 if family == "identical" else s * s  # corners have exactly three neighbours at the spacing, every other point more
    assert bool((out == want).all()), out.unique()[:8]


def test_reference_call_expression():
    """scene/gaussian_model.py:315: torch.clamp_min(distCUDA2(fused_point_cloud.detach().clone().float().cuda()), 0.0000001), where
    fused_point_cloud = torch.tensor(np.asarray(pcd.points)).float().cuda() (:304) from a float64 numpy cloud."""
    from simple_knn._C import distCUDA2
    np_points = np.random.default_rng(10).uniform(-1.3, 1.3, (3000, 3))  # float64, as pcd.points
    d = torch.clamp_min(distCUDA2(torch.tensor(np_points).float().cuda().detach().clone().float().cuda()), 1e-7)
    assert d.dtype == torch.float32 and d.shape == (3000,) and d.is_cuda
    base = torch.randn(4000, 4, device=DEV)
    col = base[:, :3]
    assert not col.is_contiguous()
    assert torch.equal(distCUDA2(col).view(torch.int32), distCUDA2(col.contiguous()).view(torch.int32))
