"""The widened rows (SURVEY.md 8f-1, 8f-2, 8f-4) against fixtures produced by the REFERENCE'S OWN Python functions
(tools/gen_golden_fused.py imports utils/loss_utils.py, utils/graphics_utils.py and scene/gaussian_model.py from the reference checkout
and writes tests/golden/fused_*.npz).  GPU tests compare the fused kernels with those outputs; the CPU tests pin the PLY writer /
reader to the bytes the reference's save_ply produced.

Tolerances: each fixture also carries the same reference function evaluated in float64; a kernel passes when it is as close to
the float64 answer as the reference's own float32 evaluation is (factor 4 head-room), and within a small absolute bar of the
float32 fixture itself."""
import os

import numpy as np
import pytest
import torch
from types import SimpleNamespace

from conftest import GOLDEN_DIR

DEV = "cuda"


def _load(name):
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    if not os.path.exists(path):
        pytest.skip(path + " missing")
    return dict(np.load(path))


def _t(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _close(ours, ref32, ref64, name, abs_bar, factor=4.0):
    """|ours - f64| <= factor * |ref32 - f64| + abs_bar (L2 over the tensor, relative to |f64|), i.e. not worse than the reference's
    own fp32 evaluation; plus a max-norm check against the fp32 fixture."""
    o, r32, r64 = np.asarray(ours, np.float64), np.asarray(ref32, np.float64), np.asarray(ref64, np.float64)
    scale = np.linalg.norm(r64) + 1e-30
    e_ours, e_ref = np.linalg.norm(o - r64) / scale, np.linalg.norm(r32 - r64) / scale
    assert e_ours <= factor * e_ref + abs_bar, f"{name}: ours vs f64 {e_ours:.3e}, reference fp32 vs f64 {e_ref:.3e}"
    m = np.abs(r64).max() + 1e-30
    assert np.abs(o - r32).max() <= (factor * np.abs(r32 - r64).max() + abs_bar * m) * 2 + 1e-12, f"{name}: max |ours - ref32| {np.abs(o - r32).max():.3e} (scale {m:.3e})"


# ---- 8f-2: image-side losses --------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("which", ["l1", "ssim", "train163"])
def test_losses_match_the_reference_functions(which):
    from rade_gs_b200 import losses
    d = _load("fused_losses")
    img, gt = _t(d["img"], True), _t(d["gt"])
    v = {"l1": lambda: losses.l1_loss(img, gt), "ssim": lambda: losses.ssim(img, gt), "train163": lambda: losses.l1_ssim_loss(img, gt, 0.2)}[which]()
    v.backward()
    _close(v.item(), d[which], d[which + "_f64"], which, 2e-6)
    _close(img.grad.cpu().numpy(), d["d_" + which], d["d_" + which + "_f64"], "d_" + which, 2e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["depth", "point"])
def test_normal_consistency_matches_the_reference_functions(kind):
    from rade_gs_b200 import losses
    d = _load("fused_normals")
    nrm = _t(d["normal"], True)
    if kind == "depth":
        a, b = _t(d["depth1"], True), _t(d["depth2"], True)
        view = SimpleNamespace(FoVx=float(d["FoVx"]), FoVy=float(d["FoVy"]))
        v = losses.depth_normal_consistency_loss(view, nrm, a, b)
    else:
        a, b = _t(d["point1"], True), _t(d["point2"], True)
        v = losses.point_normal_consistency_loss(nrm, a, b)
    v.backward()
    _close(v.item(), d[kind + "_loss"], d[kind + "_loss_f64"], kind + " loss", 2e-6)
    _close(nrm.grad.cpu().numpy(), d[kind + "_d_normal"], d[kind + "_d_normal_f64"], kind + " d_normal", 2e-6)
    _close(a.grad.cpu().numpy(), d[kind + "_d1"], d[kind + "_d1_f64"], kind + " d_map1", 5e-6)
    _close(b.grad.cpu().numpy(), d[kind + "_d2"], d[kind + "_d2_f64"], kind + " d_map2", 5e-6)


# ---- 8f-1: activations, densification statistics; 8f-4: 3D filter -----------------------------------------------------------------

@pytest.mark.gpu
def test_activations_match_the_reference_properties():
    from rade_gs_b200 import fused
    d = _load("fused_model")
    s, o, r, f = _t(d["raw_scaling"], True), _t(d["raw_opacity"], True), _t(d["raw_rotation"], True), _t(d["filter_3D"])
    scales, opacity, rot = fused.activate_gaussians(s, o, r, f)
    for name, got in (("scales", scales), ("opacity", opacity), ("rotations", rot)):
        ref = d[name]
        err = np.abs(got.detach().cpu().numpy() - ref) / (np.abs(ref) + 1e-12)
        assert err.max() < 4e-6, (name, err.max())          # a few ulp: exp / sqrt / division orderings
    ((scales * _t(d["g_scales"])).sum() + (opacity * _t(d["g_opacity"])).sum() + (rot * _t(d["g_rotations"])).sum()).backward()
    for name, got in (("d_raw_scaling", s.grad), ("d_raw_opacity", o.grad), ("d_raw_rotation", r.grad)):
        ref = d[name]
        row = np.abs(ref).max(axis=1, keepdims=True) + 1e-6 * np.abs(ref).max()
        assert (np.abs(got.cpu().numpy() - ref) / row).max() < 2e-4, name    # fp32 autograd of the reference vs the closed form


@pytest.mark.gpu
def test_densification_stats_match_the_reference_method():
    from rade_gs_b200 import fused
    d = _load("fused_model")
    acc, ab, mx, den, mr = (_t(d["stats_in_" + k].copy()) for k in ("accum", "abs", "absmax", "denom", "maxradii"))
    fused.add_densification_stats_(_t(d["stats_grad"]), _t(d["stats_radii"]), acc, ab, mx, den, mr)
    for got, key, tol in ((acc, "accum", 1e-6), (ab, "abs", 1e-6), (mx, "absmax", 1e-6), (den, "denom", 0.0), (mr, "maxradii", 0.0)):
        ref = d["stats_out_" + key]
        assert np.abs(got.cpu().numpy() - ref).max() <= tol * (1 + np.abs(ref).max()), key


@pytest.mark.gpu
def test_compute_3d_filter_matches_the_reference_method():
    from rade_gs_b200 import fused
    d = _load("fused_model")
    cams = [SimpleNamespace(R=row[:9].reshape(3, 3), T=row[9:12], FoVx=float(row[12]), FoVy=float(row[13]), image_width=int(row[14]), image_height=int(row[15]))
            for row in d["filter_cams"]]
    got = fused.compute_3D_filter(_t(d["filter_xyz"]), cams).cpu().numpy()
    ref = d["filter_out"]
    rel = np.abs(got - ref) / np.abs(ref)
    # a point within an ulp of a frustum test can fall on the other side (different expression order): allow a handful
    assert (rel > 1e-5).sum() <= 3 and np.median(rel) < 1e-6, (int((rel > 1e-5).sum()), float(rel.max()))


# ---- 8f-4: PLY bytes (CPU) ------------------------------------------------------------------------------------------------------

def test_ply_writer_reproduces_the_bytes_of_the_reference_save_ply(tmp_path):
    from rade_gs_b200 import ply_io
    d = _load("fused_ply")
    path = str(tmp_path / "x" / "point_cloud.ply")
    ply_io.save_gaussian_ply(path, d["xyz"], d["features_dc"], d["features_rest"], d["opacity"], d["scaling"], d["rotation"], d["filter_3D"])
    assert open(path, "rb").read() == d["file_bytes"].tobytes()


def test_ply_reader_returns_what_the_reference_load_ply_returns(tmp_path):
    from rade_gs_b200 import ply_io
    d = _load("fused_ply")
    path = str(tmp_path / "ref.ply")
    open(path, "wb").write(d["file_bytes"].tobytes())
    m = ply_io.load_gaussian_ply(path, max_sh_degree=int(d["sh_degree"]))
    for k in ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation", "filter_3D"):
        assert np.array_equal(m[k], d["loaded_" + k]), k
