"""Host checks of the tetrahedra extraction: the numpy model (tests/tetra_model.py) reproduces, bit for bit, every stage the
reference's own code recorded in tests/golden/tetra/*.npz (tools/gen_golden_tetra.py), and the Python entry points reject
malformed input before anything reaches the GPU."""
import glob
import os

import numpy as np
import pytest
import torch

import tetra_model as model
import tetra_scenes as scenes

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "tetra", "*.npz")))
CASES = [os.path.basename(p)[:-4] for p in GOLDEN]


def load(name):
    return dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "tetra", name + ".npz")))


def model_sdf(views):
    def evaluate(points):
        final = np.ones(len(points), np.float32)
        weight = np.zeros(len(points), np.int32)
        for v in views:
            ret = scenes.integrate(torch.from_numpy(np.ascontiguousarray(points)), v)
            model.cull_add(final, weight, ret["alpha_integrated"].numpy(), ret["point_coordinate"].numpy(), ret["render"][7].numpy(), v.gt_mask)
        return model.cull_finish(final, weight)
    return evaluate


def test_fixtures_present():
    assert set(CASES) >= {"sphere_gt", "sphere_nogt", "empty"}


@pytest.mark.parametrize("case", CASES)
def test_model_reproduces_reference(case):
    d = load(case)
    evaluate = model_sdf(scenes.views_of(d))
    sdf = evaluate(d["points"])
    assert np.array_equal(sdf, d["sdf"])
    out = model.marching(d["points"], sdf, d["scales"], d["cells"])
    for got, key in zip(out, ("ends", "end_sdf", "end_scales", "faces", "interp_v")):
        assert got.dtype == d[key].dtype and np.array_equal(got, d[key]), key
    steps = []
    verts, faces = model.extract_mesh(d["points"], d["scales"], d["cells"], evaluate, int(d["n_steps"].item()), record=steps)
    if len(d["ends"]):
        assert len(steps) == int(d["n_steps"].item()) == 8
        for k, (mid, msdf) in enumerate(steps):
            assert np.array_equal(mid, d[f"mid_{k}"]), k
            assert np.array_equal(msdf, d[f"mid_sdf_{k}"]), k
    assert np.array_equal(verts, d["vertices"]) and np.array_equal(faces, d["out_faces"])


def test_fixtures_cover_cases():
    """Every valid occupancy code, never-seen points, gt_mask on and off, an empty surface, at least two views."""
    codes, seen_never, gt_on, gt_off, empty = set(), False, False, False, False
    for case in CASES:
        d = load(case)
        occ = d["sdf"] > 0
        c = (occ[d["cells"].astype(np.int64)] * (1 << np.arange(4))).sum(-1)
        codes |= set(np.unique(c).tolist())
        seen_never |= bool((d["sdf"] == -100).any())
        views = scenes.views_of(d)
        assert len(views) >= 2
        gt_on |= any(v.gt_mask is not None for v in views)
        gt_off |= any(v.gt_mask is None for v in views)
        empty |= len(d["ends"]) == 0
    assert set(range(1, 15)) <= codes
    assert seen_never and gt_on and gt_off and empty


def test_model_rejects_out_of_range():
    pts = np.zeros((4, 3), np.float32)
    with pytest.raises(ValueError):
        model.marching(pts, np.ones(4, np.float32), np.ones(4, np.float32), np.array([[0, 1, 2, 4]]))


def test_entry_points_validate_input():
    from rade_gs_b200 import tetra
    cpu = torch.zeros((2, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        tetra.tetra_points(cpu, cpu, torch.zeros((2, 4)))
    with pytest.raises(RuntimeError, match="CUDA"):
        tetra.CullSDF(3, "cpu")
    with pytest.raises(ValueError):
        tetra.CullSDF(-1, "cuda")
    with pytest.raises(ValueError):
        tetra._tets(np.zeros((3, 3), np.int64), "cpu")
    with pytest.raises(TypeError):
        tetra._tets(np.zeros((3, 4), np.float32), "cpu")
    with pytest.raises(ValueError):
        tetra.extract_mesh(cpu, cpu, np.zeros((0, 4)), lambda p: p, n_binary_steps=-1)


def test_triangulate_fallback():
    from rade_gs_b200 import tetra
    pts = np.random.default_rng(1).normal(size=(50, 3)).astype(np.float32)
    cells = tetra.triangulate(torch.from_numpy(pts))
    assert cells.dtype == torch.int32 and cells.shape[1] == 4 and cells.shape[0] > 0
    assert int(cells.min()) >= 0 and int(cells.max()) < 50
