"""simple_knn drop-in (distCUDA2) without a GPU: the C ABI's host-side rejections, the Python surface, and the numpy fp32
brute-force oracle that tests/test_gpu_knn.py compares the kernels against bit for bit."""
import ctypes
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from conftest import ROOT

LIB = os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so")


def knn_oracle(points):
    """The rgs_knn_mean_dist2 contract, brute force in numpy float32.  numpy's float32 element-wise operations are rounded one
    by one, so (dx*dx + dy*dy) + dz*dz and ((d0 + d1) + d2) / 3 give exactly the contract's bits."""
    pts = np.asarray(points, np.float32)
    P = len(pts)
    out = np.full(P, np.nan, np.float32)
    fin = np.isfinite(pts).all(axis=1)
    q = pts[fin]
    F = len(q)
    if F == 0:
        return out
    if F == 1:
        out[fin] = np.float32(1.0)
        return out
    n = min(F - 1, 3)
    res = np.empty(F, np.float32)
    chunk = max(1, (1 << 24) // F)
    for s in range(0, F, chunk):
        e = min(F, s + chunk)
        dx = q[s:e, None, 0] - q[None, :, 0]
        d = dx * dx
        dy = q[s:e, None, 1] - q[None, :, 1]
        d += dy * dy
        dz = q[s:e, None, 2] - q[None, :, 2]
        d += dz * dz
        d[np.arange(e - s), np.arange(s, e)] = np.inf   # "other" is decided by index: only the point itself is excluded
        k = np.sort(np.partition(d, n - 1, axis=1)[:, :n], axis=1)
        acc = k[:, 0]
        for i in range(1, n):
            acc = acc + k[:, i]
        res[s:e] = acc / np.float32(n)
    out[fin] = res
    return out


def kdtree_mean_dist2(points):
    """fp64 reference: mean squared distance to the 3 nearest other points (k = 4 includes the point itself or a duplicate
    at distance 0; dropping the first zero is the same either way)."""
    p = np.asarray(points, np.float64)
    d, _ = cKDTree(p).query(p, k=4, workers=-1)
    return (d[:, 1:] ** 2).mean(axis=1)


def test_abi_host_rejections():
    lib = ctypes.CDLL(LIB)
    lib.rgs_last_error.restype = ctypes.c_char_p
    f = lib.rgs_knn_mean_dist2
    f.restype = ctypes.c_int32
    f.argtypes = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    assert f(-1, None, None, None, None, None) == -1
    assert b"negative" in lib.rgs_last_error()
    assert f(0, None, None, None, None, None) == 0          # P = 0: nothing to do, no CUDA call
    fake = ctypes.c_void_p(0x1000)                            # never dereferenced: rejected before any CUDA call
    assert f(5, None, fake, fake, None, None) == -1
    assert b"null" in lib.rgs_last_error()
    assert f(5, fake, fake, None, None, None) == -1           # no scratch callback
    assert b"null" in lib.rgs_last_error()


def test_simple_knn_resolves_to_this_package():
    import diff_gaussian_rasterization as dgr
    import simple_knn._C
    from simple_knn._C import distCUDA2
    assert os.path.realpath(simple_knn._C.__file__) == os.path.realpath(os.path.join(ROOT, "rade-gs_b200", "simple_knn", "_C.py"))
    assert distCUDA2 is dgr._C.knn_mean_dist2


def test_distcuda2_rejects_bad_input():
    from simple_knn._C import distCUDA2
    with pytest.raises(RuntimeError, match="no CPU path"):
        distCUDA2(torch.zeros(8, 3))
    with pytest.raises(RuntimeError, match=r"num_points, 3"):
        distCUDA2(torch.zeros(8, 2))
    with pytest.raises(RuntimeError, match="float32"):
        distCUDA2(torch.zeros(8, 3, dtype=torch.float64))


@pytest.mark.parametrize("P", [4, 5, 33, 500])
def test_oracle_agrees_with_kdtree(P):
    rng = np.random.default_rng(P)
    pts = rng.uniform(-1.3, 1.3, (P, 3)).astype(np.float32)
    pts[1] = pts[0]                                            # a duplicate is a neighbour at distance 0
    ours, ref = knn_oracle(pts), kdtree_mean_dist2(pts)
    assert ours.dtype == np.float32 and ours.shape == (P,)
    assert np.all(np.abs(ours - ref) <= 2e-6 * ref)
    assert np.array_equal(ours == 0.0, ref == 0.0)


def test_oracle_small_clouds():
    assert knn_oracle(np.zeros((0, 3))).shape == (0,)
    assert knn_oracle([[1.0, 2.0, 3.0]]).tolist() == [1.0]
    two = knn_oracle([[0, 0, 0], [1, 2, 2]])
    assert two.tolist() == [9.0, 9.0]
    three = knn_oracle([[0, 0, 0], [1, 0, 0], [0, 3, 0]])      # mean over the P - 1 = 2 others
    assert three.tolist() == [5.0, 5.5, 9.5]


def test_oracle_non_finite_rows():
    rng = np.random.default_rng(3)
    pts = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    bad = [2, 7, 30]
    pts[2, 0] = np.nan
    pts[7, 1] = np.inf
    pts[30, 2] = -np.inf
    out = knn_oracle(pts)
    assert np.isnan(out[bad]).all()
    keep = np.setdiff1d(np.arange(40), bad)
    assert np.array_equal(out[keep], knn_oracle(pts[keep]))
    # fewer than 4 finite points left: the small-cloud rule applies to them
    few = np.array([[0, 0, 0], [np.nan, 0, 0], [2, 0, 0], [0, np.inf, 0]], np.float32)
    assert np.array_equal(knn_oracle(few), np.array([4.0, np.nan, 4.0, np.nan], np.float32), equal_nan=True)
    assert np.isnan(knn_oracle(np.full((3, 3), np.nan))).all()
