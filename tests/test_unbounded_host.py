"""CPU checks of the unbounded-scene mesh: the numpy model (tests/unbounded_f32.py) against the reference's expressions
restated in torch at fp64, the normalisation on cameras with a known focus, the merge and cluster models against
independent restatements, the argument checks of the public functions and of `_C._unbounded`, and the GPU file's case
list."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import unbounded_f32 as M
import unbounded_scenes as S


def test_model_sdf_within_four_times_the_references_fp32_error():
    """|model - fp64| <= 4 max |reference fp32 - fp64| + 2^-22 over samples whose discrete decisions (in view, kept) agree
    between the fp32 and the fp64 run; the samples dropped for that are counted and few."""
    d, c, wv, fp = S.views(6, W=40, H=30, seed=1)
    g = np.random.default_rng(1)
    axes = [np.sort(g.uniform(-1.9, 1.9, 14)).astype(np.float32) for _ in range(3)]
    center, radius, vs = np.array([0.1, -0.05, 0.2]), 1.4, 1.4 * 2 / 64
    trunc = float(np.float32(5 * vs))
    model = M.sdf(*axes, fp.numpy(), d.numpy(), center.astype(np.float32), radius, trunc).reshape(-1)
    s = torch.from_numpy(np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3))
    t32, w32 = S.torch_tsdf(s, center.astype(np.float32), radius, vs, d, fp, torch.float32)
    t64, w64 = S.torch_tsdf(s, center.astype(np.float32), radius, vs, d, fp, torch.float64)
    same = (w32.double() == w64).numpy()
    assert same.mean() > 0.98
    ref_err = (t32.double() - t64).abs().numpy()[same].max()
    err = np.abs(model.astype(np.float64) - t64.numpy())[same]
    assert err.max() <= 4 * ref_err + 2.0 ** -22, (err.max(), ref_err)
    assert (w64.numpy() > 1).mean() > 0.05            # the scene fuses views


def test_normalization_finds_the_focus():
    from rade_gs_b200 import unbounded as ub
    target = (0.3, -0.2, 0.1)
    eyes = [(target[0] + 2.5 * math.cos(a), target[1] + 2.5 * math.sin(a), target[2] + 0.4) for a in np.linspace(0, 2 * np.pi, 9)[:-1]]
    wv = [S.camera(e, target)[0] for e in eyes]
    center, radius = ub.normalization(wv)
    assert np.allclose(center, target, atol=1e-5)
    assert abs(radius - math.hypot(2.5, 0.4)) < 1e-5
    with pytest.raises(ValueError, match="4x4"):
        ub.normalization([])


def test_model_mcubes_is_closed_and_oriented():
    n = 21
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    f = (np.sqrt(X ** 2 + Y ** 2 + (1.2 * Z) ** 2) - 0.6).astype(np.float32)
    v, t = M.mcubes(f, (-1.0,) * 3, (2.0 / (n - 1),) * 3)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert (cnt == 2).all()
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    assert ((np.cross(b - a, c - a) * (a + b + c)).sum(1) > 0).all()
    assert np.allclose(np.linalg.norm(v * [1, 1, 1.2], axis=1), 0.6, atol=0.02)


def test_model_merge_against_a_dictionary():
    g = np.random.default_rng(0)
    base = g.uniform(-1.5, 1.5, (300, 3))
    v = np.concatenate([base, base + g.uniform(-3e-7, 3e-7, base.shape), base[g.permutation(300)]])
    t = g.integers(0, len(v), (500, 3)).astype(np.int32)
    mv, mt = M.merge(v, t)
    first, order = {}, []
    for i, p in enumerate(v):
        k = tuple(np.rint(p * 1e6).astype(np.int64))
        if k not in first:
            first[k] = i
            order.append(i)
    newid = {o: j for j, o in enumerate(order)}
    rep = [newid[first[tuple(np.rint(p * 1e6).astype(np.int64))]] for p in v]
    assert np.array_equal(mv, v[order].astype(np.float32))
    assert np.array_equal(mt, np.array(rep)[t])


def _bfs_clusters(tris):
    edges = {}
    for i, tr in enumerate(tris.tolist()):
        for a, b in ((tr[0], tr[1]), (tr[1], tr[2]), (tr[2], tr[0])):
            edges.setdefault((min(a, b), max(a, b)), []).append(i)
    lab = [-1] * len(tris)
    sizes = []
    for s in range(len(tris)):
        if lab[s] >= 0:
            continue
        lab[s] = len(sizes)
        stack, n = [s], 0
        while stack:
            t = stack.pop()
            n += 1
            tr = tris[t].tolist()
            for a, b in ((tr[0], tr[1]), (tr[1], tr[2]), (tr[2], tr[0])):
                for u in edges[(min(a, b), max(a, b))]:
                    if lab[u] < 0:
                        lab[u] = lab[s]
                        stack.append(u)
        sizes.append(n)
    return np.array(lab), np.array(sizes)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_model_clusters_against_a_search(seed):
    g = np.random.default_rng(seed)
    V = 400
    tris = np.concatenate([g.integers(0, V, (600, 3)), [[5, 5, 6], [7, 7, 7]]]).astype(np.int32)
    lab, sizes = _bfs_clusters(tris)
    for k in (0, 1, 3, len(sizes), len(sizes) + 1):
        vi, tt, msizes = M.clusters(V, tris, k)
        assert np.array_equal(np.sort(msizes), np.sort(sizes))
        srt = np.sort(sizes)
        thr = max(srt[0] if k == 0 else (srt[-k] if k <= len(sizes) else 0), 50)
        kept = tris[sizes[lab] >= thr]
        used = np.unique(kept)
        remap = {int(o): j for j, o in enumerate(used)}
        nd = kept[(kept[:, 0] != kept[:, 1]) & (kept[:, 1] != kept[:, 2]) & (kept[:, 0] != kept[:, 2])]
        assert np.array_equal(vi, used)
        assert np.array_equal(tt, np.vectorize(remap.get)(nd).reshape(-1, 3) if len(nd) else np.zeros((0, 3), np.int32))


def test_functional_form_rejects_bad_arguments_before_the_device():
    from rade_gs_b200 import unbounded as ub
    d, c, wv, fp = S.views(2, W=8, H=6)
    xyz = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="multiple"):
        ub.extract_mesh_unbounded_maps(d, c, list(wv), fp, xyz, resolution=100, crop=32)
    with pytest.raises(ValueError, match="CUDA"):
        ub.extract_mesh_unbounded_maps(d, c, list(wv), fp, xyz, resolution=64, crop=32)
    with pytest.raises(ValueError, match="crop"):
        ub.extract_mesh_unbounded_maps(d, c, list(wv), fp, xyz, resolution=64, crop=1)
    with pytest.raises(ValueError, match="CUDA"):
        ub.contract(torch.zeros(3, 3))
    with pytest.raises(ValueError, match=">= 0"):
        from rade_gs_b200 import tsdf
        ub.post_process_mesh(tsdf.TriangleMesh(torch.zeros(0, 3), torch.zeros((0, 3), dtype=torch.int32), torch.zeros(0, 3)), -1)


def test_extractor_checks_resolution_and_views():
    from rade_gs_b200 import unbounded as ub
    ex = ub.GaussianExtractor.__new__(ub.GaussianExtractor)
    ex.clean()
    with pytest.raises(ValueError, match="multiple of 512"):
        ex.extract_mesh_unbounded(resolution=1000)
    with pytest.raises(ValueError, match="reconstruction"):
        ex.extract_mesh_unbounded(resolution=512)
    ex._render = lambda *a: None
    with pytest.raises(ValueError, match="at least one view"):
        ex.reconstruction([])


def test_every_entry_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    U = _C._unbounded
    f = torch.zeros
    calls = {
        "contract": lambda: U.contract(f(4, 3), [0.0, 0.0, 0.0], 1.0, False, math.inf),
        "sdf": lambda: U.sdf(f(4), f(4), f(4), f(2, 4, 4), f(2, 3, 5), [0.0, 0.0, 0.0], 1.0, 0.1),
        "colors": lambda: U.colors(f(4, 3), f(2, 4, 4), f(2, 3, 5), f(2, 3, 3, 5), 0.1),
        "mcubes": lambda: U.mcubes(f(4, 4, 4), [0.0] * 3, [1.0] * 3),
        "merge": lambda: U.merge(f(4, 3, dtype=torch.float64), f(1, 3, dtype=torch.int32)),
        "clusters": lambda: U.clusters(4, f(1, 3, dtype=torch.int32), 1),
    }
    assert set(calls) == {n for n in dir(U) if not n.startswith("_")}
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="CUDA"):
            call()


def test_gpu_case_list_names_every_entry():
    import ast
    import os
    from diff_gaussian_rasterization import _C
    src = open(os.path.join(os.path.dirname(__file__), "test_gpu_unbounded.py")).read()
    tree = ast.parse(src)
    cases = next(ast.literal_eval(n.value) for n in tree.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", "") == "CASES")
    tests = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
    assert set(cases) == {n for n in dir(_C._unbounded) if not n.startswith("_")}
    assert all(t in tests for ts in cases.values() for t in ts)


# ---- against the fixture made by the reference's own code (tools/gen_golden_unbounded.py) ----------------------------

def fixture() -> dict:
    """tests/golden/unbounded/unbounded.npz with the voxels of the three planes (x = 128, y = 300, z = 411) rebuilt, the fp64
    SDF restored from its stored difference and the decision marks unpacked (`*_keep`: away from every decision)."""
    import os
    f = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "unbounded", "unbounded.npz")))
    ax = np.arange(512)
    planes = [np.stack(np.meshgrid(*[[c] if k == a else ax for k in range(3)], indexing="ij"), -1).reshape(-1, 3)
              for a, c in ((0, 128), (1, 300), (2, 411))]
    f["voxels"] = np.concatenate(planes + [f["voxels"]]).astype(np.int64)
    f["sdf64"] = f["sdf"].astype(np.float64) + f.pop("sdf64_minus_sdf").astype(np.float64)
    f["sdf_keep"] = np.unpackbits(f.pop("sdf_decided"))[:len(f["sdf"])].astype(bool)
    f["vertex_keep"], f["color_keep"] = f.pop("vertex_decided"), f.pop("color_decided")
    return f


_fixture = fixture



def _R(f):
    """The fixture's R in the dtype the reference's numpy gave it."""
    return np.asarray(f["R"], dtype=str(f["R_dtype"]))[()]


def test_normalization_and_bound_against_the_fixture():
    from rade_gs_b200 import unbounded as ub
    f = _fixture()
    center, radius = ub.normalization(list(f["world_view"]))
    assert np.allclose(center, f["center"], rtol=0, atol=1e-12) and abs(radius - float(f["radius"])) <= 1e-12
    assert np.array_equal(np.float32(center), f["center32"])
    assert radius * 2 / 512 == float(f["voxel_size"])
    # R through the model's norms and numpy's expressions: the same dtype as the reference's, within one fp32 step
    norms = M.norm3(M.contract(f["xyz"], center, radius))
    R = min(np.quantile(norms, q=0.95) + 0.01, 1.9)
    assert np.asarray(R).dtype == np.asarray(_R(f)).dtype
    assert abs(float(R) - float(f["R"])) <= 2.0 ** -22


def _fixture_samples(f):
    xs = np.linspace(-_R(f), _R(f), 512).astype(np.float32)
    v = f["voxels"]
    return np.stack([xs[v[:, 0]], xs[v[:, 1]], xs[v[:, 2]]], -1)


def test_model_sdf_against_the_fixture():
    """|model - fp64| <= 4 max |reference fp32 - fp64| over the fixture's voxels away from a discrete decision."""
    f = _fixture()
    keep = f["sdf_keep"]
    assert keep.mean() > 0.95, keep.mean()
    model = M.sdf_points(_fixture_samples(f), f["full_proj"], f["depth"], f["center"], float(f["radius"]), np.float32(5 * float(f["voxel_size"])))
    ref_err = np.abs(f["sdf"].astype(np.float64) - f["sdf64"])[keep].max()
    err = np.abs(model.astype(np.float64) - f["sdf64"])[keep].max()
    assert err <= 4 * ref_err + 2.0 ** -24, (err, ref_err)
    assert (f["sdf"][keep] < 1).mean() > 0.02                 # views were fused at these voxels


def test_model_vertices_and_colors_against_the_fixture():
    f = _fixture()
    from rade_gs_b200 import unbounded as ub
    (lo, sp, _), = ub.crop_axes(_R(f), 512, 512)                  # origin and spacing as the Python layer passes them
    pos = f["planted"] * np.asarray(sp, np.float64) + np.asarray(lo, np.float64)   # the vertex rule of rgs_unbounded_mcubes
    world = M.inv_contraction(pos.astype(np.float32), f["center"], float(f["radius"]), 32.0)
    kv = f["vertex_keep"]
    ref_err = np.abs(f["vertices"].astype(np.float64) - f["vertices64"])[kv].max()
    err = np.abs(world.astype(np.float64) - f["vertices64"])[kv].max()
    assert err <= 4 * ref_err, (err, ref_err)
    kc = f["color_keep"]
    assert kc.mean() > 0.9
    col = M.colors(f["vertices"], f["full_proj"], f["depth"], f["rgb"], np.float32(5 * float(f["voxel_size"])))
    ref_err = np.abs(f["colors"].astype(np.float64) - f["colors64"])[kc].max()
    err = np.abs(col.astype(np.float64) - f["colors64"])[kc].max()
    assert err <= 4 * ref_err + 2.0 ** -24, (err, ref_err)
    # the reference's colour average starts from 0 with weight 1: a vertex seen by k views keeps k / (k + 1) of its colour
    assert (f["colors"][kc].max(1) < 1).all()
