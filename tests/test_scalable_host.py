"""CPU checks of the bounded TSDF (Open3D's legacy ScalableTSDFVolume) and the image export: the byte rule against numpy's
own cast, the numpy model (tests/scalable_f32.py) and the Python layer against the fixture made by the reference's code
(tools/gen_golden_bounded.py), the model's TSDF against an fp64 ray distance, the argument checks, the CPU refusals of
`_C._scalable_tsdf` and the GPU file's case list."""
from __future__ import annotations

import os
import types
import warnings

import numpy as np
import pytest
import torch

import scalable_f32 as M
import tsdf_f32 as T
import tsdf_scenes as ts

F = np.float32


def fixture() -> dict:
    return dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "bounded", "bounded.npz")))


def fixture_cameras(f, device="cpu"):
    W, H = (int(x) for x in f["size"])
    return [types.SimpleNamespace(image_width=W, image_height=H, FoVx=float(f["fovx"][i]), FoVy=float(f["fovy"][i]),
                                  world_view_transform=torch.from_numpy(f["world_view"][i]).to(device),
                                  gt_mask=torch.from_numpy(f["mask"][i]).to(device), original_image=torch.from_numpy(f["gt"][i]).to(device))
            for i in range(len(f["rgb"]))]


def test_byte_rule_is_numpys_cast():
    """The contract's B(x) against np.asarray(x, dtype=np.uint8) over wrap, negatives, NaN, +-inf and |x| >= 2^31."""
    g = np.random.default_rng(0)
    edges = np.array([0, 0.5, 0.99, 1, 254.9, 255, 255.5, 256, 257.55, 300, 76500, -0.5, -1, -2.55, -255, -256, -257, np.nan, np.inf, -np.inf,
                      2.0 ** 31, -2.0 ** 31, np.nextafter(F(2.0 ** 31), F(0)), np.nextafter(F(-2.0 ** 31), F(0)), 2.0 ** 32, 1e10, -1e10, 3e38,
                      -3e38, 2.0 ** 24 + 3, -(2.0 ** 24) - 5], F)
    x = np.concatenate([edges, g.uniform(-600, 600, 20000).astype(F), (g.standard_normal(20000) * 1e9).astype(F),
                        g.uniform(-1, 2, 20000).astype(F) * F(255)])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = np.asarray(x, dtype=np.uint8)
    assert np.array_equal(M.numpy_u8(x), want)
    assert M.numpy_u8(F(1.01) * F(255)) == 1 and M.numpy_u8(F(-0.01) * F(255)) == 254 and M.numpy_u8(F(300)) == 44


def test_model_and_glue_against_the_fixture():
    """The reference's recorded Open3D inputs: colour bytes, masked depth, intrinsic, extrinsic and the volume's arguments;
    the export's arrays.  The model reproduces every byte and float, and the Python layer builds the same camera."""
    from rade_gs_b200 import unbounded as ub
    f = fixture()
    assert float(f["voxel_length"]) == 0.004 and float(f["sdf_trunc"]) == 0.02
    assert (f["rec_depth_scale"] == 1).all() and not f["rec_intensity"].any() and (f["rec_depth_trunc"] == 3).all()
    assert np.isnan(f["rgb"]).any() and (f["rgb"] > 1).any() and (f["rgb"] < 0).any()
    for i, cam in enumerate(fixture_cameras(f)):
        color, depth = M.rgbd(f["rgb"][i], f["depth"][i], 3, f["mask"][i])
        assert np.array_equal(color, f["rec_color"][i])
        rec = f["rec_depth"][i][..., 0]
        want = np.where(rec >= 3, F(0), rec)
        assert np.array_equal(depth.view(np.uint32), want.view(np.uint32))
        K, E = ub.open3d_camera(cam)
        Wd, Hd, fx, fy, cx, cy = f["rec_intrinsic"][i]
        assert np.array_equal(K, [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]) and (Wd, Hd) == (cam.image_width, cam.image_height)
        assert np.array_equal(E, f["rec_extrinsic"][i])
        assert np.array_equal(M.image_u8(f["gt"][i]), f[f"file:gt/{i:05d}.png"])
        assert np.array_equal(M.image_u8(f["rgb"][i]), f[f"file:renders/{i:05d}.png"])
        assert np.array_equal(M.image_u8(f["normals"][i], 0.5, 0.5), f[f"file:vis/normal_{i:05d}.png"])
        assert np.array_equal(np.nan_to_num(f["depth"][i][0]), f[f"file:vis/depth_{i:05d}.tiff"])
    assert (f["rec_depth"][2] >= 3).any() and (f["mask"] < 0.5).any()


def _f64_sdf(cam, units, depth, model_grid):
    """fp64 restatement of the ray distance at every voxel the model updated in one view, with the model's own pixel (so
    both take the same discrete decisions), and the fp32 error bound of each value."""
    keys = np.unique(T.pack(units))
    g = T.grid_points(T.unpack(keys)).astype(np.float64)
    p = (g + 0.5) * float(cam.vs)
    R, t = cam.R.astype(np.float64), cam.t.astype(np.float64)
    pc = p @ R.T + t
    u = np.floor(((pc[..., 0] / pc[..., 2]).astype(F) * cam.fx + cam.cx) + F(0.5))   # the model's pixel (fp32 rule)
    v = np.floor(((pc[..., 1] / pc[..., 2]).astype(F) * cam.fy + cam.cy) + F(0.5))
    xn, yn = (u - np.float64(cam.cx)) / np.float64(cam.fx), (v - np.float64(cam.cy)) / np.float64(cam.fy)
    m = np.sqrt(1 + xn * xn + yn * yn)
    wt = np.stack([model_grid[int(k)][1] for k in keys])
    ts_ = np.stack([model_grid[int(k)][0] for k in keys])
    upd = wt == 1
    ui, vi = np.clip(u, 0, cam.W - 1).astype(np.int64), np.clip(v, 0, cam.H - 1).astype(np.int64)
    d = np.asarray(depth, np.float64)[vi, ui]
    sdf = (d - pc[..., 2]) * m
    want = np.minimum(1.0, sdf / float(cam.trunc))
    # fp32: p carries 2^-24 |p|; each of the 3 products and 3 sums of z_c one rounding of its magnitude; d - z_c, the
    # multiplier (2 products, 2 sums, sqrt: 3 roundings of m), the product and the division one rounding each
    eps = 2.0 ** -24
    mag = np.abs(p) @ np.abs(R[2]) + abs(t[2])
    ez = eps * (2 * (np.abs(p) @ np.abs(R[2])) + 3 * mag)
    bound = (ez * m + (np.abs(d - pc[..., 2]) * m) * 6 * eps) / float(cam.trunc) + 2 * eps * np.maximum(np.abs(want), 1)
    return ts_[upd].astype(np.float64), want[upd], bound[upd]


@pytest.mark.parametrize("family", ["fronto", "tilted", "sphere"])
def test_model_tsdf_within_the_fp32_error_of_the_ray_distance(family):
    sc = ts.make(family)
    v = sc.views[0]
    cam = M.Camera(v.K, v.E, *v.depth.shape, sc.vs, 5 * sc.vs)
    units = M.touch(cam, v.depth)
    color, depth = M.rgbd(np.transpose(v.color, (2, 0, 1)), v.depth, sc.depth_max)
    grid = {}
    M.integrate(grid, cam, units, depth, color)
    got, want, bound = _f64_sdf(cam, units, depth, grid)
    assert len(got) > 1000
    err = np.abs(got - want)
    assert (err <= bound).all(), (err.max(), bound[np.argmax(err - bound)])
    assert (got < 0).any() and (got > 0).any() and (got == 1).any()


def test_model_mesh_of_a_fronto_plane_lies_on_the_plane():
    """Depth d everywhere: the SDF changes sign at z = d on every ray.  Along a z edge the two voxel centres may project to
    neighbouring pixels, whose ray multipliers m differ by at most dm; that moves the vertex by at most vs dm / m."""
    vs, d, W, H = 0.01, F(1.2345), 64, 48
    K = ts.intrinsic(W, H)
    cam = M.Camera(K, np.eye(4), H, W, vs, 4 * vs)
    depth = np.full((H, W), d, F)
    color = np.zeros((H, W, 3), np.uint8)
    grid = {}
    for _ in range(2):
        M.integrate(grid, cam, M.touch(cam, depth), depth, color)
    verts, cols, tris = M.extract(grid, vs)
    assert len(tris) > 1000
    vv, uu = np.mgrid[-1:H + 1, -1:W + 1].astype(np.float64)
    m = np.sqrt(1 + ((uu - W / 2) / K[0, 0]) ** 2 + ((vv - H / 2) / K[1, 1]) ** 2)
    dm = max(np.abs(np.diff(m, axis=0)).max() + np.abs(np.diff(m, axis=1)).max(), 0)
    bound = vs * dm / m.min() + 2.0 ** -20
    err = np.abs(verts[:, 2].astype(np.float64) - float(d))
    assert err.max() <= bound, (err.max(), bound)
    assert (cols == 0).all()


def test_arguments_are_checked_before_the_device():
    from rade_gs_b200 import tsdf
    from rade_gs_b200 import unbounded as ub
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="sdf_trunc"):
            tsdf.ScalableTSDFVolume(0.004, bad)
        with pytest.raises(ValueError, match="voxel_length"):
            tsdf.ScalableTSDFVolume(bad, 0.02)
    with pytest.raises(ValueError, match="block_count"):
        tsdf.ScalableTSDFVolume(0.004, 0.02, block_count=0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        tsdf.ScalableTSDFVolume(0.004, 0.02, device="cpu")
    with pytest.raises(ValueError, match="CUDA"):
        tsdf.rgbd_from_color_and_depth(torch.zeros(3, 4, 4), torch.zeros(1, 4, 4), 3.0)
    ex = ub.GaussianExtractor.__new__(ub.GaussianExtractor)
    ex.clean()
    with pytest.raises(ValueError, match="reconstruction"):
        ex.extract_mesh_bounded()
    with pytest.raises(ValueError, match="reconstruction"):
        ex.export_image("/nonexistent")
    ex.viewpoint_stack = [object()]                  # a render() without "normal" maps: the mesh works, the export cannot
    with pytest.raises(ValueError, match="normal"):
        ex.export_image("/nonexistent")


def test_every_entry_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    S = _C._scalable_tsdf
    f = torch.zeros
    vol = types.SimpleNamespace(voxel_size=0.01, hash_keys=f(4, dtype=torch.int64), hash_values=f(4, dtype=torch.int32), tsdf=f(4096),
                                weight=f(4096), color=f(3 * 4096), stamps=f(1, dtype=torch.int32), frame_keys=f(4, dtype=torch.int64),
                                frame_list=f(2, dtype=torch.int64), counters=f(4, dtype=torch.int32))
    K, E = torch.eye(3, dtype=torch.float64), torch.eye(4, dtype=torch.float64)
    calls = {
        "rgbd": lambda: S.rgbd(f(3, 4, 5), f(1, 4, 5), 3.0),
        "image_u8": lambda: S.image_u8(f(3, 4, 5)),
        "touch": lambda: S.touch(vol, f(4, 5), K, E, 0.02),
        "integrate": lambda: S.integrate(vol, f(1, 3, dtype=torch.int32), f(4, 5), f(4, 5, 3, dtype=torch.uint8), K, E, 0.02, 1),
    }
    assert set(calls) == {n for n in dir(S) if not n.startswith("_")}
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="CUDA"):
            call()


def test_gpu_case_list_names_every_entry():
    import ast
    from diff_gaussian_rasterization import _C
    src = open(os.path.join(os.path.dirname(__file__), "test_gpu_scalable.py")).read()
    tree = ast.parse(src)
    cases = next(ast.literal_eval(n.value) for n in tree.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "CASES")
    tests = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
    assert set(cases) == {n for n in dir(_C._scalable_tsdf) if not n.startswith("_")}
    assert all(t in tests for ts_ in cases.values() for t in ts_)
