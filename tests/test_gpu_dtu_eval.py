"""DTU evaluation on the GPU, held bit for bit to the fp64 model (tests/dtu_eval_f64.py) and to fixtures made by the
reference's own eval.py / cull_mesh (tools/gen_golden_dtu_eval.py)."""
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import pytest
import torch

import dtu_eval_f64 as model
from conftest import ROOT
from test_dtu_eval_host import SCANS, cull_cameras, load, reference_keep

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _de():
    from rade_gs_b200 import dtu_eval
    return dtu_eval


def np_(t):
    return t.detach().cpu().numpy()


# ---- sampling ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [s for s in SCANS if s.startswith("mesh")])
def test_samples_equal_reference(name):
    d = load(name)
    out = _de().sample_mesh_points(d["vertices"], d["faces"], float(d["density"]))
    assert np.array_equal(np_(out), d["original"])


def _degenerate_mesh(rng):
    v = rng.normal(500, 3, (60, 3))
    f = rng.integers(0, 60, (150, 3))
    v = np.concatenate([v, [[500, 500, 500], [500, 500, 500], [501, 500, 500], [502, 500, 500], [490, 490, 490], [490 + 1e-10, 490, 490],
                            [520, 490, 490], [450, 450, 450], [470, 450, 450], [450, 471, 450]]])
    f = np.concatenate([f, [[60, 61, 62], [60, 62, 63], [61, 61, 62], [64, 65, 66], [67, 68, 69], [0, 0, 0]]])
    return v, f


@pytest.mark.parametrize("case", ["degenerate", "one_triangle", "no_faces", "large_only"])
def test_samples_equal_model(case):
    rng = np.random.default_rng(5)
    if case == "degenerate":
        v, f = _degenerate_mesh(rng)
    elif case == "one_triangle":
        v, f = np.array([[500.0, 500, 500], [503.7, 500.2, 500.1], [500.3, 502.9, 501.0]]), np.array([[0, 1, 2]])
    elif case == "no_faces":
        v, f = rng.normal(500, 1, (17, 3)), np.zeros((0, 3), np.int64)
    else:   # 10^5-sample triangle among small ones: the emit stays one thread per point
        v = np.concatenate([[[0.0, 0, 0], [90.0, 0, 0], [0, 90.0, 0]], rng.normal(0, 1, (30, 3))])
        f = np.concatenate([[[0, 1, 2]], rng.integers(3, 33, (40, 3))])
    for density in (0.2, 0.37):
        got = np_(_de().sample_mesh_points(v, f, density))
        assert np.array_equal(got, model.sample(v, f, density)), (case, density)
        if case == "large_only" and density == 0.2:
            assert len(got) > 100_000


def test_sample_count_over_2_31_rejected_before_allocation():
    v = np.array([[0.0, 0, 0], [30000.0, 0, 0], [0, 30000.0, 0]])   # about 1.1e10 samples at 0.2
    f = np.array([[0, 1, 2]])
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with pytest.raises(RuntimeError, match="2\\^31"):
        _de().sample_mesh_points(v, f, 0.2)
    assert torch.cuda.max_memory_allocated() - before < 1 << 20


# ---- downsample -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SCANS)
def test_kept_mask_equals_reference(name):
    d = load(name)
    r = _de().radius_downsample(d["original"], float(d["density"]), perm=d["perm"])
    assert np.array_equal(np_(r.kept), d["kept"])
    assert np.array_equal(np_(r.points), d["original"][d["perm"]][d["kept"]])


def _clouds():
    rng = np.random.default_rng(9)
    lat = np.stack(np.meshgrid(*[np.arange(12) * 0.25] * 3, indexing="ij"), -1).reshape(-1, 3) + 500.0
    yield "uniform", rng.uniform(490, 510, (40000, 3)), 0.2, None
    yield "dense", rng.uniform(499, 501, (30000, 3)), 0.2, None
    yield "lattice_at_r", lat, 0.25, None   # neighbours at exactly r (representable): d <= r includes them
    yield "clusters", np.concatenate([rng.normal(c, 0.3, (3000, 3)) for c in rng.uniform(480, 520, (5, 3))]), 0.2, None
    line = np.stack([np.arange(600) * 0.05, np.zeros(600), np.zeros(600)], 1) + 500.0
    yield "sorted_line", line, 0.2, np.arange(600)   # rank increases along the line: the most rounds


@pytest.mark.parametrize("case", ["uniform", "dense", "lattice_at_r", "clusters", "sorted_line"])
def test_kept_mask_equals_greedy_model(case):
    name, pts, r, perm = next(c for c in _clouds() if c[0] == case)
    if perm is None:
        perm = np.random.default_rng(1).permutation(len(pts))
    got = _de().radius_downsample(pts, r, perm=perm)
    assert np.array_equal(np_(got.kept), model.greedy_downsample(pts[perm], r))
    if case == "sorted_line":
        assert got.rounds > 10


def test_identical_points_are_linear():
    pts = torch.full((1_000_000, 3), 500.125, dtype=torch.float64, device=DEV)
    _de().radius_downsample(pts[:1000], 0.2, seed=0)
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = _de().radius_downsample(pts, 0.2, seed=3)
    torch.cuda.synchronize()
    assert time.perf_counter() - t < 5.0
    kept = np_(r.kept)
    assert kept.sum() == 1 and kept[0] and r.rounds <= 3


# ---- nearest ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", SCANS)
def test_evaluate_equals_reference(name):
    d = load(name)
    data = (d["vertices"], d["faces"]) if str(d["mode"]) == "mesh" else d["points"]
    r = _de().evaluate(data, d["stl"], d["obs_mask"], d["bb"], d["res"], d["plane"], mode=str(d["mode"]), downsample_density=float(d["density"]),
                       patch_size=float(d["patch"]), max_dist=float(d["max_dist"]), visualize_threshold=float(d["vis"]), perm=d["perm"])
    assert np.array_equal(np_(r.in_obs), d["in_obs"])
    assert np.array_equal(np_(r.dist_d2s), d["dist_d2s"]) and np.array_equal(np_(r.dist_s2d), d["dist_s2d"])
    np.testing.assert_allclose([r.mean_d2s, r.mean_s2d, r.overall], d["means"], rtol=1e-12, atol=0)
    assert np.array_equal(np_(r.data_color), d["data_color"]) and np.array_equal(np_(r.stl_color), d["stl_color"])


def _nn_cases():
    rng = np.random.default_rng(17)
    ref = np.concatenate([rng.normal(c, 0.5, (4000, 3)) for c in rng.uniform(0, 100, (6, 3))])
    yield "clustered", ref, rng.uniform(-10, 110, (20000, 3))
    dup = np.repeat(rng.uniform(0, 5, (300, 3)), 20, axis=0)
    yield "duplicates", dup, np.concatenate([dup[::7], rng.uniform(0, 5, (3000, 3))])
    yield "translated_1e3", ref + 1e3, rng.uniform(-10, 110, (5000, 3)) + 1e3
    yield "query_is_reference", ref, ref.copy()
    yield "tiny_reference", ref[:3], rng.uniform(0, 100, (100, 3))


@pytest.mark.parametrize("case", ["clustered", "duplicates", "translated_1e3", "query_is_reference", "tiny_reference"])
def test_nearest_equals_brute_force(case):
    _, ref, q = next(c for c in _nn_cases() if c[0] == case)
    dist, idx = _de().nearest_distances(ref, q)
    want = model.nearest(ref, q)
    assert np.array_equal(np_(dist), want)
    i = np_(idx)
    assert np.array_equal(np.sqrt(model.dist2(ref[i], q)), want)
    if case == "query_is_reference":
        assert not want.any()


def test_run_to_run_identity():
    d = load("mesh_a")
    outs = [_de().evaluate((d["vertices"], d["faces"]), d["stl"], d["obs_mask"], d["bb"], d["res"], d["plane"], seed=4, patch_size=3.0)
            for _ in range(2)]
    a, b = outs
    assert torch.equal(a.perm, b.perm) and torch.equal(a.kept, b.kept) and torch.equal(a.dist_d2s, b.dist_d2s) and torch.equal(a.dist_s2d, b.dist_s2d)
    assert a.mean_d2s == b.mean_d2s and a.mean_s2d == b.mean_s2d


def test_input_validation():
    de = _de()
    p = np.random.default_rng(0).normal(0, 1, (100, 3))
    bad = p.copy()
    bad[7, 1] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        de.nearest_distances(bad, p)
    with pytest.raises(ValueError, match="NaN"):
        de.radius_downsample(bad, 0.2, seed=0)
    with pytest.raises(ValueError, match="empty"):
        de.nearest_distances(np.zeros((0, 3)), p)
    from diff_gaussian_rasterization import _C   # the C ABI checks too, below the Python layer
    t = torch.as_tensor(bad, device=DEV)
    with pytest.raises(RuntimeError, match="NaN"):
        _C.dtu_nearest(t, t)
    with pytest.raises(RuntimeError, match="empty"):
        _C.dtu_nearest(t[:0], t)
    with pytest.raises(RuntimeError, match="radius"):
        _C.dtu_radius_downsample(t, 0.0)
    with pytest.raises(RuntimeError, match="face index"):
        _C.dtu_sample_mesh(torch.as_tensor(p, device=DEV), torch.tensor([[0, 1, 100]], dtype=torch.int32, device=DEV), 0.2)


# ---- culling ----------------------------------------------------------------------------------------------------------

def test_cull_equals_model_and_reference():
    de = _de()
    d = load("cull")
    cams = cull_cameras(d)
    v, f, keep = de.cull_mesh(cams, d["vertices"], d["faces"])
    dil = np.stack([model.dilate(m[0]) for m in d["masks"]])
    want = model.cull_keep(d["vertices"], de.cull_projections(cams), dil)
    assert np.array_equal(np_(keep), want)
    assert np.array_equal(np_(de._C.dtu_dilate_masks(de.cull_masks(cams))), dil.astype(np.uint8))
    new = np.cumsum(want) - 1
    assert np.array_equal(np_(v), d["vertices"][want]) and np.array_equal(np_(f), new[d["faces"][want[d["faces"]].all(1)]])
    W, H = (int(x) for x in d["size"])
    near = model.cull_near_boundary(d["vertices"], de.cull_projections(cams), W, H)
    assert np.array_equal(want[~near], reference_keep(d)[~near])


# ---- end to end -------------------------------------------------------------------------------------------------------

def test_tsdf_cull_evaluate_sphere_end_to_end():
    """Analytic depth of a sphere -> VoxelBlockGrid -> mesh -> cull_mesh -> evaluate, against points sampled on the exact
    sphere (mm).  Bound, stated before the run: the fused surface lies within test_tsdf_host's sphere bound
    2 (dist + r) / f + vs^2 / (8 r) + trunc / 2 of the sphere (pixel footprint, voxel interpolation, grazing-view bias in
    the truncation band, 4 voxels as there), a point of a triangle adds at most the sagitta of a voxel diagonal
    3 vs^2 / (8 r), and each nearest-neighbour distance adds at most the spacing of the cloud it searches (the 2 mm
    downsample radius; the STL's mean spacing is below 2 mm at 400 000 points).  Every mean stays below the sum."""
    import tsdf_scenes as ts
    from rade_gs_b200.tsdf import VoxelBlockGrid
    de = _de()
    r_m, dist, vs = 0.3, 1.2, 0.02
    sc = ts.sphere_scene(n_views=30, W=96, H=80, vs=vs, r=r_m, dist=dist)
    sc.trunc_mult = 4.0
    vbg = VoxelBlockGrid(sc.vs, 16, 64)
    for vw in sc.views:
        dep, col = torch.as_tensor(vw.depth, device=DEV), torch.as_tensor(vw.color, device=DEV)
        coords = vbg.compute_unique_block_coordinates(dep, vw.K, vw.E, 1.0, sc.depth_max, sc.trunc_mult)
        vbg.integrate(coords, dep, col, vw.K, vw.E, 1.0, sc.depth_max, sc.trunc_mult)
    mesh = vbg.extract_triangle_mesh()
    cams = []
    for vw in sc.views:
        H, W = vw.depth.shape
        cams.append(types.SimpleNamespace(world_view_transform=torch.tensor(vw.E.T), FoVx=2 * np.arctan(W / (2 * vw.K[0, 0])),
                                          FoVy=2 * np.arctan(H / (2 * vw.K[1, 1])), image_width=W, image_height=H,
                                          gt_mask=torch.tensor((vw.depth > 0)[None].astype(np.float32))))
    v, f, keep = de.cull_mesh(cams, mesh.vertices.double(), mesh.triangles)
    assert keep.float().mean() > 0.99
    rng = np.random.default_rng(0)
    u = rng.normal(size=(400000, 3))
    stl = 300.0 * u / np.linalg.norm(u, axis=1, keepdims=True) + 500.0
    bb = np.array([[180.0, 180.0, 180.0], [820.0, 820.0, 820.0]])
    r = de.evaluate((v * 1000.0 + 500.0, f), stl, np.ones((33, 33, 33), np.uint8), bb, np.array([[20.0]]), np.array([0.0, 0.0, 1.0, 0.0]),
                    downsample_density=2.0, seed=0)
    print(f"sphere: mean_d2s {r.mean_d2s:.3f} mm, mean_s2d {r.mean_s2d:.3f} mm, overall {r.overall:.3f} mm")
    f_px = sc.views[0].K[0, 0]
    bound = 1000.0 * (2 * (dist + r_m) / f_px + vs * vs / (8 * r_m) + sc.trunc_mult * vs / 2 + 3 * vs * vs / (8 * r_m)) + 2.0 + 2.0
    print(f"sphere: bound {bound:.3f} mm")
    assert r.overall < bound and r.mean_d2s < bound and r.mean_s2d < bound


def test_cli_writes_results_without_open3d_trimesh_skimage_or_sklearn(tmp_path):
    import scipy.io
    from rade_gs_b200 import ply_io
    d = load("mesh_a")
    ds = tmp_path / "dtu"
    (ds / "ObsMask").mkdir(parents=True)
    (ds / "Points" / "stl").mkdir(parents=True)
    scipy.io.savemat(str(ds / "ObsMask" / "ObsMask1_10.mat"), {"ObsMask": d["obs_mask"], "BB": d["bb"], "Res": d["res"]})
    scipy.io.savemat(str(ds / "ObsMask" / "Plane1.mat"), {"P": d["plane"]})
    ply_io.save_point_cloud_ply(str(ds / "Points" / "stl" / "stl001_total.ply"), d["stl"])
    mesh = tmp_path / "mesh.ply"
    ply_io.save_triangle_mesh_ply(str(mesh), d["vertices"].astype(np.float32), d["faces"])
    out = tmp_path / "vis"
    code = ("import sys; sys.path.insert(0, %r); import runpy; sys.argv = ['dtu_eval'] + sys.argv[1:]; "
            "runpy.run_module('rade_gs_b200.dtu_eval', run_name='__main__'); "
            "print('BAD', sorted(m for m in sys.modules if m.split('.')[0] in ('open3d', 'trimesh', 'skimage', 'sklearn')))") % os.path.join(ROOT, "rade-gs_b200")
    res = subprocess.run([sys.executable, "-c", code, "--data", str(mesh), "--scan", "1", "--dataset_dir", str(ds), "--vis_out_dir", str(out),
                          "--patch_size", "3", "--seed", "0"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    assert "BAD []" in res.stdout
    j = json.load(open(out / "results.json"))
    assert set(j) == {"mean_d2s", "mean_s2d", "overall"} and abs(j["overall"] - (j["mean_d2s"] + j["mean_s2d"]) / 2) < 1e-12
    assert np.isfinite(j["overall"])
    assert (out / "vis_001_d2s.ply").exists() and (out / "vis_001_s2d.ply").exists()
    assert len(ply_io.load_point_cloud_ply(str(out / "vis_001_s2d.ply"))) == len(d["stl"])
