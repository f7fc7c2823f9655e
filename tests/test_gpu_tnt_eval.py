"""Tanks and Temples evaluation on the GPU, held bit for bit to the fp64 model (tests/tnt_eval_f64.py) wherever the
contract fixes the bits, within 1e-12 where it fixes only the summation tree, and to fixtures made by the reference's own
run.py (tools/gen_golden_tnt_eval.py)."""
import io
import json
import os

import numpy as np
import pytest
import torch

import tnt_eval_f64 as model
from test_tnt_eval_host import SCENES, golden_inputs, load

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _te():
    from rade_gs_b200 import tnt_eval
    return tnt_eval


def np_(t):
    return t.detach().cpu().numpy()


POLY = np.array([[-1.0, -1.0], [1.0, -1.0], [1.0, 1.0], [0.0, 0.25], [-1.0, 1.0], [-1.0, 0.2], [-0.5, 0.2], [-0.5, -0.3], [-1.0, -0.3]])


def _crop_points(rng):
    """Random points plus points exactly on the polygon's vertices, on its edges (horizontal ones included) and exactly
    on axis_min / axis_max."""
    p = rng.uniform(-1.3, 1.3, (20000, 3))
    on = []
    for k in range(len(POLY)):
        a, b = POLY[k], POLY[(k + 1) % len(POLY)]
        for t in (0.0, 0.25, 0.5, 1.0 / 3.0):
            u, v = a + t * (b - a)
            on.append([u, v, rng.uniform(-0.4, 0.4)])
    on = np.array(on)
    ends = rng.uniform(-1, 1, (200, 3))
    ends[:100, 2], ends[100:, 2] = -0.5, 0.5
    return np.concatenate([p, on, ends])


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("with_transform", [False, True])
def test_crop_mask_equals_model(axis, with_transform):
    rng = np.random.default_rng(10 + axis)
    p = _crop_points(rng)
    perm = [a for a in range(3) if a != axis]
    q = np.empty_like(p)   # put the polygon's (u, v) on the two remaining axes and the range on `axis`
    q[:, perm[0]], q[:, perm[1]], q[:, axis] = p[:, 0], p[:, 1], p[:, 2]
    T = None
    if with_transform:
        T = np.eye(4)
        T[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) * 1.25
        T[:3, 3] = [0.125, -0.25, 0.0625]
        q = model.transform(np.linalg.inv(T), q)
    vol = _te().CropVolume(axis, -0.5, 0.5, POLY)
    got, kept = _te().crop(q, vol, T)
    want, wkept = model.crop(q, (axis, -0.5, 0.5, POLY), T)
    assert np.array_equal(np_(kept), wkept)
    assert np.array_equal(np_(got), want)
    assert 0 < wkept.sum() < len(q)
    if not with_transform:
        assert wkept[-200:].any()   # both ends of the axis range are inside
    got2, _ = _te().crop(q, vol, T)
    assert torch.equal(got, got2)


def test_crop_without_volume_and_empty():
    rng = np.random.default_rng(3)
    p = rng.normal(size=(1000, 3))
    T = np.eye(4)
    T[:3, 3] = [1.0, 2.0, 3.0]
    got, kept = _te().crop(p, None, T)
    assert bool(kept.all()) and np.array_equal(np_(got), model.transform(T, p))
    got, kept = _te().crop(np.zeros((0, 3)), _te().CropVolume(2, 0, 1, POLY))
    assert got.shape == (0, 3) and kept.shape == (0,)
    bad = T.copy()
    bad[3, 0] = 1e-3
    with pytest.raises(ValueError):
        _te().crop(p, None, bad)
    p[5, 1] = np.nan
    with pytest.raises(ValueError):
        _te().crop(p, None)


def test_transform_in_place_equals_model():
    from diff_gaussian_rasterization import _C
    rng = np.random.default_rng(4)
    p = rng.normal(size=(5000, 3))
    T = np.eye(4)
    T[:3, :3] = rng.normal(size=(3, 3))
    T[:3, 3] = rng.normal(size=3)
    t = torch.as_tensor(p, device=DEV).contiguous()
    _C.tnt_transform(t, torch.as_tensor(T))
    assert np.array_equal(np_(t), model.transform(T, p))


@pytest.mark.parametrize("case", ["random", "faces", "negative", "big_voxel", "single", "empty"])
def test_voxel_equals_model(case):
    rng = np.random.default_rng(20)
    voxel = 0.05
    if case == "random":
        p = rng.uniform(0, 3, (50000, 3))
    elif case == "faces":   # coordinates exactly on voxel faces (origin = min - voxel / 2)
        p = np.round(rng.uniform(0, 1, (20000, 3)) / voxel) * voxel + voxel * 0.5
        p = np.concatenate([p, [[0.0, 0.0, 0.0]]])
    elif case == "negative":
        p = rng.uniform(-7.5, -2.0, (30000, 3))
    elif case == "big_voxel":   # one voxel of 10^5 points among small ones
        p = np.concatenate([rng.uniform(0.5, 0.5 + voxel / 4, (100000, 3)), rng.uniform(0, 3, (5000, 3))])
        p = p[rng.permutation(len(p))]
    elif case == "single":
        p = np.array([[-0.0, 1.5, -2.25]])
    else:
        p = np.zeros((0, 3))
    means, counts = _te().voxel_down_sample(p, voxel)
    wm, wc = model.voxel_down_sample(p, voxel)
    assert np.array_equal(np_(means), wm) and np.array_equal(np_(counts), wc)
    if case == "big_voxel":
        assert wc.max() >= 100000
    m2, c2 = _te().voxel_down_sample(p, voxel)
    assert torch.equal(means, m2) and torch.equal(counts, c2)


def test_voxel_more_than_2_21_cells_rejected_before_allocation():
    p = np.array([[0.0, 0.0, 0.0], [3000.0, 1.0, 1.0]])
    t = torch.as_tensor(p, device=DEV)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with pytest.raises(ValueError, match="2\\^21"):
        _te().voxel_down_sample(t, 1e-3)
    assert torch.cuda.max_memory_allocated() - before < 1 << 20
    means, _ = _te().voxel_down_sample(t, 3000.0 / 2097150)   # just below the limit
    assert means.shape[0] == 2


def test_distances_and_histogram_equal_model():
    rng = np.random.default_rng(30)
    a = rng.normal(0, 0.3, (30000, 3))
    b = a[:20000] + rng.normal(0, 0.004, (20000, 3))
    d1, i1 = _te().nearest_distances(a, b)
    want = model.nearest(a, b)[0]
    assert np.array_equal(np_(d1), want)
    edges = _te().histogram_edges(0.005)
    assert np.array_equal(_te().cumulative_histogram(d1, edges), np.cumsum(np.histogram(want, edges)[0]).astype(float) / len(want))


def _icp_scene(seed, n=20000):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-1, 1, (n, 2))
    tgt = np.column_stack([xy, 0.1 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1])])
    T = np.eye(4)
    c, s = np.cos(0.03), np.sin(0.03)
    T[:3, :3] = 1.02 * np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    T[:3, 3] = [0.01, -0.02, 0.015]
    src = model.transform(np.linalg.inv(T), tgt[rng.permutation(n)[: n // 2]] + rng.normal(0, 0.002, (n // 2, 3)))
    return src, tgt


def test_moments_within_1e12_and_repeatable():
    from diff_gaussian_rasterization import _C
    src, tgt = _icp_scene(40)
    s, t = torch.as_tensor(src, device=DEV), torch.as_tensor(tgt, device=DEV)
    d, idx = _te().nearest_distances(t, s)
    for thr in (0.02, 0.05, 1.0):
        got = _te().icp_moments(s, t, d, idx, thr)
        want = model.moments(src, tgt, np_(d), np_(idx), thr)
        assert got[0] == want[0]
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
        again = _C.tnt_icp_moments(s, t, d, idx, thr).numpy()
        assert np.array_equal(got, again)
    assert np.array_equal(_te().icp_moments(s, t, d, idx, 0.0), np.zeros(18))
    assert np.array_equal(_te().umeyama(np.zeros(18)), np.eye(4))


@pytest.mark.parametrize("thr", [0.01, 0.05])
def test_icp_iterations_equal_model(thr):
    src, tgt = _icp_scene(41)
    T, fit, rmse, it, hist, counts = model.icp(src, tgt, thr, max_iteration=30)
    # no distance within 1e-9 of the threshold at any evaluation, so both sides see the same correspondences
    for H in [np.eye(4)] + hist:
        d = model.nearest(tgt, model.transform(H, src))[0]
        assert np.abs(d - thr).min() > 1e-9
    r = _te().icp(src, tgt, thr, max_iteration=30)
    assert r.iterations == it and len(r.history) == len(hist) and it >= 2
    for a, b in zip(r.history, hist):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
    assert abs(r.fitness - fit) == 0.0
    np.testing.assert_allclose(r.inlier_rmse, rmse, rtol=1e-12)


def _write_mesh_ply(path, v, f):
    with open(path, "wb") as fp:
        fp.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty double x\nproperty double y\nproperty double z\n"
                  "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), len(f))).encode())
        fp.write(np.ascontiguousarray(v, "<f8").tobytes())
        rec = np.zeros(len(f), dtype=[("n", "u1"), ("i", "<i4", 3)])
        rec["n"], rec["i"] = 3, f
        fp.write(rec.tobytes())


@pytest.mark.parametrize("name", SCENES)
def test_mesh_points_equal_trimesh_centroids(name):
    d = load(name)
    source, _, _ = golden_inputs(d)
    assert np.array_equal(np_(_te().mesh_points(d["vertices"], d["faces"])), source)


@pytest.mark.parametrize("name", SCENES)
def test_cli_end_to_end_equals_reference(name, tmp_path, capsys):
    from gen_golden_tnt_eval import write_log
    from rade_gs_b200 import ply_io
    d = load(name)
    scene = str(d["scene"])
    ds = tmp_path / scene
    ds.mkdir()
    ply_io.save_point_cloud_ply(str(ds / (scene + ".ply")), d["gt"])
    (ds / (scene + ".json")).write_text(str(d["crop_json"]))
    np.savetxt(ds / (scene + "_trans.txt"), d["gt_trans"])
    write_log(ds / (scene + "_COLMAP_SfM.log"), d["gt_traj"])
    ext = str(d["traj_format"])
    traj = tmp_path / ("traj" + ext)
    if ext == ".npy":
        np.save(traj, d["traj"])
    else:
        write_log(traj, d["traj"])
    _write_mesh_ply(tmp_path / "recon.ply", d["vertices"], d["faces"])
    out = tmp_path / "out"
    r = _te().main(["--dataset-dir", str(ds), "--traj-path", str(traj), "--ply-path", str(tmp_path / "recon.ply"), "--out-dir", str(out),
                    "--seed", str(int(d["seed"]))])
    printed = capsys.readouterr().out
    assert [r["precision"], r["recall"], r["fscore"]] == list(d["prf"][:3])
    np.testing.assert_allclose(np.array(r["transformation"]), d["stage_T"][-1], rtol=1e-9, atol=1e-10)
    assert sorted(os.listdir(out)) == list(d["files"])
    for k, txt in zip(d["txt_names"], d["txt_contents"]):
        got = (out / str(k)).read_text()
        assert np.loadtxt(io.StringIO(got)).shape == np.loadtxt(io.StringIO(str(txt))).shape
        assert got == str(txt), k
    assert len(ply_io.load_point_cloud_ply(str(out / (scene + ".precision.ply")))) == d["ply_sizes"][0]
    assert "f-score : %.4f" % d["prf"][2] in printed

    # the same through evaluate(): every stage within tolerance, iteration counts equal
    sc = _te().load_scene(str(ds))
    sc.pop("scene")
    res = _te().evaluate(_te().mesh_points(d["vertices"], d["faces"]), traj=d["traj"], seed=int(d["seed"]), **sc)
    np.testing.assert_allclose(res.alignment, d["alignment"], rtol=1e-12, atol=1e-12)
    for k, st in enumerate(res.stages):
        np.testing.assert_allclose(st.transformation, d["stage_T"][k], rtol=1e-9, atol=1e-10)
        assert st.iterations == d["stage_iterations"][k]
        assert [st.source_points, st.target_points] == list(d["stage_sizes"][k])
    np.testing.assert_allclose([st.fitness for st in res.stages], d["stage_fitness"], rtol=1e-12)
    source, vol, _ = golden_inputs(d)
    s = model.voxel_down_sample(model.crop(source, vol, res.transformation)[0], float(d["tau"]) / 2)[0]
    assert np.array_equal(np_(res.source), s)
    t = model.voxel_down_sample(model.crop(d["gt"], vol)[0], float(d["tau"]) / 2)[0]
    assert np.array_equal(np_(res.target), t)
    assert np.array_equal(np_(res.dist_source), model.nearest(t, s)[0]) and np.array_equal(np_(res.dist_target), model.nearest(s, t)[0])
    json.dumps(r)
