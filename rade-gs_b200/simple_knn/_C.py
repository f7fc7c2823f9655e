"""``distCUDA2(points)``: points [P, 3] float32 on a CUDA device -> [P] float32, the mean squared distance from each point
to its 3 nearest other points (exact in fp32; the contract is documented at ``rgs_knn_mean_dist2`` in include/rgs_b200.h).
A plain module named ``_C`` is enough for the reference's import; the kernels live in ``diff_gaussian_rasterization._C``."""
from diff_gaussian_rasterization._C import knn_mean_dist2 as distCUDA2

__all__ = ["distCUDA2"]
