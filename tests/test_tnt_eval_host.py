"""Tanks and Temples evaluation without a GPU: the fp64 model (tests/tnt_eval_f64.py) against fixtures made by the
reference's own run.py (tools/gen_golden_tnt_eval.py), the seeded RANSAC, the readers and the package's imports."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tnt_eval_f64 as model
from conftest import GOLDEN_DIR, ROOT

TNT_DIR = os.path.join(GOLDEN_DIR, "tnt_eval")
SCENES = ["barn", "caterpillar"]


def load(name):
    return dict(np.load(os.path.join(TNT_DIR, name + ".npz")))


def golden_inputs(d):
    """(source cloud as run.py builds it, crop volume tuple for the model, crop dict)."""
    v, f = d["vertices"], d["faces"].astype(np.int64)
    source = np.concatenate([v, v[f].mean(axis=1)])
    crop = json.loads(str(d["crop_json"]))
    axis = "XYZ".index(crop["orthogonal_axis"])
    poly = np.asarray(crop["bounding_polygon"])[:, [a for a in range(3) if a != axis]]
    return source, (axis, crop["axis_min"], crop["axis_max"], poly), crop


@pytest.mark.parametrize("name", SCENES)
def test_model_equals_reference_run(name):
    d = load(name)
    source, vol, _ = golden_inputs(d)
    r = model.evaluate(source, d["gt"], vol, d["gt_trans"], d["traj"], d["gt_traj"], float(d["tau"]), int(d["seed"]))
    np.testing.assert_allclose(r["alignment"], d["alignment"], rtol=1e-12, atol=1e-12)
    for k, st in enumerate(r["stages"]):
        np.testing.assert_allclose(st["T"], d["stage_T"][k], rtol=1e-12, atol=1e-12)
        assert st["iterations"] == d["stage_iterations"][k]
    assert [r["precision"], r["recall"], r["fscore"]] == list(d["prf"][:3])
    assert d["prf"][3] == float(d["tau"]) and d["prf"][4] == 5
    assert np.array_equal(r["edges"], d["edges_source"]) and np.array_equal(r["edges"], d["edges_target"])
    assert np.array_equal(r["cum_source"], d["cum_source"]) and np.array_equal(r["cum_target"], d["cum_target"])
    assert list(d["ply_sizes"]) == [len(r["source"]), len(r["target"])]
    assert list(d["stage_threshold"]) == [80 * float(d["tau"]), 20 * float(d["tau"]), 2 * float(d["tau"])]
    # the text files, as np.savetxt writes them
    texts = dict(zip(d["txt_names"], d["txt_contents"]))
    scene = str(d["scene"])
    for suffix, arr in ((".precision.txt", r["cum_source"]), (".recall.txt", r["cum_target"]),
                        (".prf_tau_plotstr.txt", np.array([r["precision"], r["recall"], r["fscore"], float(d["tau"]), 5]))):
        buf = io.StringIO()
        np.savetxt(buf, arr)
        assert buf.getvalue() == texts[scene + suffix]
    assert 0.5 < r["precision"] < 1 and 0.5 < r["recall"] < 1   # the scenes are neither trivial nor broken
    np.testing.assert_allclose(r["T"], d["planted"], atol=5e-3)  # the pipeline recovers the planted similarity


def _planted(seed, n=60, scale=2.3, outliers=6):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = scale * q, rng.normal(0, 2, 3)
    src = rng.normal(0, 3, (n, 3))
    dst = model.transform(T, src)
    bad = rng.choice(n, outliers, replace=False)
    dst[bad] += rng.normal(0, 5, (outliers, 3))
    return src, dst, T, bad


def test_model_ransac_recovers_planted_similarity_and_is_seeded():
    src, dst, T, bad = _planted(3)
    R1, n_in, rmse, _ = model.ransac(src, dst, seed=7, iterations=2000)
    assert n_in == len(src) - len(bad)
    np.testing.assert_allclose(R1, T, rtol=0, atol=1e-9)
    R2 = model.ransac(src, dst, seed=7, iterations=2000)[0]
    assert np.array_equal(R1, R2)
    hyp = model.ransac_hypotheses(len(src), 5000, 6, 11)
    assert all(len(set(h)) == 6 for h in hyp.tolist())
    assert not np.array_equal(hyp, model.ransac_hypotheses(len(src), 5000, 6, 12))


def test_package_alignment_equals_model():
    from rade_gs_b200 import tnt_eval
    src, dst, T, _ = _planted(4)
    traj = np.tile(np.eye(4), (len(src), 1, 1))
    traj[:, :3, 3] = src
    G = np.eye(4)
    G[:3, 3] = [0.5, -0.25, 1.0]
    gt_traj = np.tile(np.eye(4), (len(src), 1, 1))
    gt_traj[:, :3, 3] = dst - G[:3, 3]
    got = tnt_eval.trajectory_alignment(traj, gt_traj, G, seed=5, max_iteration=3000)
    want = model.ransac(src, model.transform(G, gt_traj[:, :3, 3]), 5, 3000)[0]
    assert np.array_equal(got, want)
    np.testing.assert_allclose(got, T, atol=1e-9)
    with pytest.raises(ValueError):
        tnt_eval.trajectory_alignment(traj[:10], gt_traj, G)


def test_read_trajectory_and_crop_volume(tmp_path):
    from rade_gs_b200 import tnt_eval
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from gen_golden_tnt_eval import write_log
    d = load("barn")
    write_log(tmp_path / "t.log", d["gt_traj"])
    got = tnt_eval.read_trajectory(str(tmp_path / "t.log"))
    np.testing.assert_allclose(got, d["gt_traj"], rtol=0, atol=1e-12)   # the .log keeps 12 decimals
    (tmp_path / "tab.log").write_text("0 0 1\n1\t0 0 0.5\n0 1 0 0\n0 0 1 0\n0 0 0 1\n")
    assert tnt_eval.read_trajectory(str(tmp_path / "tab.log"))[0, 0, 3] == 0.5
    np.save(tmp_path / "t.npy", d["traj"])
    assert np.array_equal(tnt_eval.load_trajectory(str(tmp_path / "t.npy")), d["traj"])
    with pytest.raises(ValueError):
        tnt_eval.load_trajectory(str(tmp_path / "t.json"))
    (tmp_path / "bad.log").write_text("0 0 1\n1 0 0\n")
    with pytest.raises(ValueError):
        tnt_eval.read_trajectory(str(tmp_path / "bad.log"))
    (tmp_path / "c.json").write_text(str(d["crop_json"]))
    v = tnt_eval.load_crop_volume(str(tmp_path / "c.json"))
    _, vol, crop = golden_inputs(d)
    assert v.orthogonal_axis == 2 and (v.axis_min, v.axis_max) == (crop["axis_min"], crop["axis_max"])
    assert np.array_equal(v.polygon, vol[3])
    (tmp_path / "y.json").write_text(json.dumps(dict(crop, orthogonal_axis="y")))
    assert np.array_equal(tnt_eval.load_crop_volume(str(tmp_path / "y.json")).polygon, np.asarray(crop["bounding_polygon"])[:, [0, 2]])
    (tmp_path / "n.json").write_text(json.dumps({"axis_min": 0}))
    with pytest.raises(ValueError):
        tnt_eval.load_crop_volume(str(tmp_path / "n.json"))


def test_uniform_down_sample_rule():
    from rade_gs_b200 import tnt_eval
    for n, rate in ((4_000_000, 1), (4_000_001, 1), (6_000_001, 2), (9_000_001, 2), (10_000_001, 3)):
        p = np.broadcast_to(np.zeros(3), (n, 3))
        got = tnt_eval.uniform_for_registration(p)
        assert len(got) == len(range(0, n, rate)) == len(model.uniform_for_registration(p)), n
    t = torch.arange(30.0).reshape(10, 3)
    assert torch.equal(tnt_eval.uniform_down_sample(t, 3), t[[0, 3, 6, 9]])


def test_histogram_and_fscore_rules():
    from rade_gs_b200 import tnt_eval
    tau = 0.005
    edges = tnt_eval.histogram_edges(tau)
    assert np.array_equal(edges, np.arange(0, tau * 5, tau / 100))
    rng = np.random.default_rng(1)
    d = np.concatenate([rng.uniform(0, 6 * tau, 3000), edges[:40], [edges[-1], 0.0, tau, 7 * tau]])
    want = np.cumsum(np.histogram(d, edges)[0]).astype(float) / len(d)
    assert np.array_equal(tnt_eval.cumulative_histogram(torch.as_tensor(d), edges), want)
    d2 = rng.uniform(0, 2 * tau, 500)
    p, r, f = tnt_eval.f_score(torch.as_tensor(d), torch.as_tensor(d2), tau)
    assert (p, r, f) == model.f_score_histo(d, d2, tau)[:3]
    assert tnt_eval.f_score(torch.full((3,), 1.0), torch.full((2,), 1.0), tau) == (0.0, 0.0, 0.0)


def test_hot_r_table():
    from rade_gs_b200 import tnt_eval
    lut = tnt_eval._hot_r_table()
    assert lut.shape == (256, 3)
    assert np.array_equal(lut[0], [1.0, 1.0, 1.0])              # hot(1) is white
    np.testing.assert_allclose(lut[-1], [0.0416, 0.0, 0.0])     # hot(0)
    assert (np.diff(lut, axis=0) <= 1e-15).all()                # every channel falls along hot_r


def test_module_imports_no_open3d_trimesh_or_matplotlib():
    code = ("import sys; sys.path.insert(0, %r); import rade_gs_b200.tnt_eval; "
            "print(sorted(m for m in ('open3d', 'trimesh', 'matplotlib') if m in sys.modules))") % os.path.join(ROOT, "rade-gs_b200")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.strip()
    assert out == "[]"
