"""The fp64 3D-filter model (tests/filter3d_f64.py) validated without a GPU: on every point without an ambiguous decision it
equals the reference's loop in fp64, and torch's own fp32 loop lands inside every point's interval."""
import pytest
import torch

import filter3d_f64 as ff
from test_gpu_activation_exact import filter_scene
from test_gpu_fused import _ref_compute_3D_filter


def _loop64(xyz, cameras):
    """scene/gaussian_model.py:179-232 in fp64 (R and T as the fp32 values the kernel reads)."""
    import math
    dist = torch.full((xyz.shape[0],), 100000.0, dtype=torch.float64)
    seen = torch.zeros(xyz.shape[0], dtype=torch.bool)
    focal = 0.0
    for c in cameras:
        W, H = c.image_width, c.image_height
        fx, fy = W / (2 * math.tan(c.FoVx / 2.)), H / (2 * math.tan(c.FoVy / 2.))
        p = xyz @ torch.tensor(c.R, dtype=torch.float32).double() + torch.tensor(c.T, dtype=torch.float32).double()
        z = p[:, 2].clamp(min=0.001)
        x, y = p[:, 0] / z * fx + W / 2.0, p[:, 1] / z * fy + H / 2.0
        ok = (p[:, 2] > 0.2) & (x >= -0.15 * W) & (x <= W * 1.15) & (y >= -0.15 * H) & (y <= 1.15 * H)
        dist[ok] = torch.minimum(dist[ok], z[ok])
        seen |= ok
        focal = max(focal, fx)
    dist[~seen] = dist[seen].max()
    return dist / focal * 0.2 ** 0.5


@pytest.mark.parametrize("n_cams,P", [(1, 500), (7, 700), (257, 300)])
def test_model_and_torch_fp32_loop(n_cams, P):
    xyz, cams = filter_scene(n_cams, P, seed=n_cams)
    lo, hi, d = ff.filter_intervals(xyz, cams)
    ref64 = _loop64(torch.from_numpy(xyz).double(), cams)
    ref32 = _ref_compute_3D_filter(torch.from_numpy(xyz), cams)[0][:, 0].double()
    clear = ~d["ambiguous"] & d["surely_seen"]
    assert clear.sum() > 100
    mid = (lo + hi) / 2
    # the model's interval is centred on the fp64 minimum; the fp64 loop uses the Python focal and sqrt(0.2), not their fp32 forms
    assert ((mid[clear] - ref64[clear]).abs() <= 1e-6 * ref64[clear]).all()
    assert (((hi - lo) / mid)[clear] < 1e-5).all()
    bad = torch.nonzero(~((ref32 >= lo) & (ref32 <= hi)))
    assert bad.numel() == 0, [(i, ref32[i].item(), lo[i].item(), hi[i].item()) for i in bad[:5, 0].tolist()]
