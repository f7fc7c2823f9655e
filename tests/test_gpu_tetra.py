"""Tetrahedra mesh extraction on the GPU (rade_gs_b200.tetra, csrc/rgs_tetra.cu) against the fixtures the reference's own code
made (tests/golden/tetra, tools/gen_golden_tetra.py) and against the numpy model of the contract (tests/tetra_model.py)."""
import math

import numpy as np
import pytest
import torch

import tetra_model as model
import tetra_scenes as scenes
from test_tetra_host import CASES, load

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gpu_sdf(views):
    from rade_gs_b200 import tetra

    def evaluate(points):
        cull = tetra.CullSDF(points.shape[0], points.device)
        for v in views:
            ret = scenes.integrate(points, v)
            gt = None if v.gt_mask is None else torch.from_numpy(v.gt_mask).to(points.device)
            cull.add(ret["alpha_integrated"], ret["point_coordinate"], ret["render"][7], gt)
        return cull.sdf()
    return evaluate


def np_(t):
    return t.cpu().numpy()


@pytest.mark.parametrize("case", CASES)
def test_stages_match_fixture(case):
    from rade_gs_b200 import tetra
    d = load(case)
    evaluate = gpu_sdf(scenes.views_of(d))
    pts = torch.from_numpy(d["points"]).to(DEV)
    sdf = evaluate(pts)
    assert np.array_equal(np_(sdf), d["sdf"])
    (ends, esdf), escl, faces, interp = [x[0] for x in tetra.marching_tetrahedra(pts[None], torch.from_numpy(d["cells"]), sdf[None],
                                                                                  torch.from_numpy(d["scales"]).to(DEV)[None])]
    for got, key in zip((ends, esdf, escl, faces, interp), ("ends", "end_sdf", "end_scales", "faces", "interp_v")):
        assert np.array_equal(np_(got), d[key]) and np_(got).dtype == d[key].dtype, key
    steps = []

    def recording(p):
        s = evaluate(p)
        steps.append((np_(p), np_(s)))
        return s
    verts, fout = tetra.extract_mesh(pts, torch.from_numpy(d["scales"]).to(DEV), d["cells"], recording)
    if len(d["ends"]):
        assert len(steps) == 9
        for k, (p, s) in enumerate(steps[1:]):
            assert np.array_equal(p, d[f"mid_{k}"]) and np.array_equal(s, d[f"mid_sdf_{k}"]), k
    else:
        assert len(steps) == 1        # an empty surface returns without evaluating midpoints
    assert np.array_equal(np_(verts), d["vertices"]) and np.array_equal(np_(fout), d["out_faces"])


@pytest.mark.parametrize("case", CASES)
def test_tetra_points_within_reference_error(case):
    from rade_gs_b200 import tetra
    d = load(case)
    t = lambda k: torch.from_numpy(d[k]).to(DEV)  # noqa: E731
    pts, scl = tetra.tetra_points(t("xyz"), t("scaling"), t("rotation"))
    assert np.array_equal(np_(scl), d["scales"])
    ref_err = np.abs(d["points"].astype(np.float64) - d["points_f64"]).max()
    our_err = np.abs(np_(pts).astype(np.float64) - d["points_f64"]).max()
    assert our_err <= 4 * ref_err, (our_err, ref_err)


def kuhn_lattice(n, device):
    """(n+1)^3 lattice points and the 6 n^3 tets of the Kuhn subdivision of its cubes (int64 [T, 4])."""
    idx = lambda i, j, k: (i * (n + 1) + j) * (n + 1) + k  # noqa: E731
    c = torch.arange(n, device=device)
    i, j, k = torch.meshgrid(c, c, c, indexing="ij")
    i, j, k = i.reshape(-1), j.reshape(-1), k.reshape(-1)
    tets = []
    for a, b, cc in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        v = [torch.stack([i, j, k])]
        for ax in (a, b):
            step = v[-1].clone()
            step[ax] += 1
            v.append(step)
        v.append(torch.stack([i + 1, j + 1, k + 1]))
        tets.append(torch.stack([idx(*p) for p in v], dim=1))
    tets = torch.stack(tets, dim=1).reshape(-1, 4)
    g = torch.arange(n + 1, device=device, dtype=torch.float32)
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    return torch.stack([X, Y, Z], -1).reshape(-1, 3), tets


def test_marching_large_lattice_chunk_order(monkeypatch):
    from rade_gs_b200 import tetra
    n = 180
    pts, tets = kuhn_lattice(n, DEV)
    assert tets.shape[0] > 2 ** 25
    c = n * 0.5 + 0.37
    o = pts - torch.tensor([c, c - 0.21, c + 0.13], device=DEV)
    sdf = (o * o).sum(-1) - (n * 0.4) ** 2
    scales = torch.rand(pts.shape[0], device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    (ends, esdf), escl, faces, interp = [x[0] for x in tetra.marching_tetrahedra(pts[None], tets, sdf[None], scales[None])]
    ref = model.marching(np_(pts), np_(sdf), np_(scales), np_(tets))
    for got, want, key in zip((ends, esdf, escl, faces, interp), ref, ("ends", "end_sdf", "end_scales", "faces", "interp")):
        assert np.array_equal(np_(got), want), key
    # the surface spans both chunks, so the chunked face order is not the one-pass order
    monkeypatch.setattr(model, "CHUNK", 1 << 40)
    one_pass = model.marching(np_(pts), np_(sdf), np_(scales), np_(tets))[3]
    assert not np.array_equal(one_pass, ref[3]) and np.array_equal(np.sort(one_pass, axis=0), np.sort(ref[3], axis=0))


def test_random_fields_on_delaunay_cells():
    from scipy.spatial import Delaunay
    from rade_gs_b200 import tetra
    from diff_gaussian_rasterization import _C
    rng = np.random.default_rng(5)
    P = rng.normal(size=(20000, 3)).astype(np.float32)
    cells = Delaunay(P.astype(np.float64)).simplices.astype(np.int32)
    sdf = rng.normal(size=len(P)).astype(np.float32)
    sdf[rng.integers(0, len(P), 500)] = 0.0
    sdf[rng.integers(0, len(P), 500)] = -100.0
    scl = rng.uniform(0.01, 0.5, len(P)).astype(np.float32)
    tp, ts, tsc = (torch.from_numpy(x).to(DEV) for x in (P, sdf, scl))
    (ends, esdf), escl, faces, interp = [x[0] for x in tetra.marching_tetrahedra(tp[None], torch.from_numpy(cells), ts[None], tsc[None])]
    ref = model.marching(P, sdf, scl, cells)
    for got, want in zip((ends, esdf, escl, faces, interp), ref):
        assert np.array_equal(np_(got), want)
    # bisection with zeros and NaN among the midpoint values, then the filter
    M = ends.shape[0]
    left, right = ends[:, 0].contiguous(), ends[:, 1].contiguous()
    ls, rs = esdf[:, 0, 0].contiguous(), esdf[:, 1, 0].contiguous()
    mid = torch.empty_like(left)
    _C.tetra_bisect(left.new_empty((0,)), left, right, ls, rs, mid)
    L, R, LS, RS = ref[0][:, 0].copy(), ref[0][:, 1].copy(), ref[1][:, 0, 0].copy(), ref[1][:, 1, 0].copy()
    assert np.array_equal(np_(mid), model.midpoints(L, R))
    for step in range(4):
        ms = rng.normal(size=M).astype(np.float32)
        ms[rng.integers(0, M, 50)] = 0.0
        ms[rng.integers(0, M, 20)] = np.nan
        _C.tetra_bisect(torch.from_numpy(ms).to(DEV), left, right, ls, rs, mid)
        want = model.bisect(ms, L, R, LS, RS)
        bits = lambda a: np.ascontiguousarray(a).view(np.uint32)  # noqa: E731  (the NaN midpoint values go right, bit for bit)
        assert all(np.array_equal(bits(np_(a)), bits(b)) for a, b in ((mid, want), (left, L), (right, R), (ls, LS), (rs, RS))), step
    v, f = _C.tetra_filter(mid, ends, escl, faces)
    wv, wf = model.filter_mesh(np_(mid), ref[0], ref[2], ref[3])
    assert 0 < len(wv) < M and 0 < len(wf) < len(ref[3])
    assert np.array_equal(np_(v), wv) and np.array_equal(np_(f), wf)


def test_out_of_range_indices_are_rejected():
    from rade_gs_b200 import tetra
    from diff_gaussian_rasterization import _C
    pts = torch.zeros((5, 3), device=DEV)
    sdf = torch.tensor([1.0, -1, -1, -1, 1], device=DEV)
    for bad in ([0, 1, 2, 5], [0, -1, 2, 3], [0, 1, 2, 1 << 40]):
        with pytest.raises(RuntimeError, match="outside"):
            tetra.marching_tetrahedra(pts[None], torch.tensor([[0, 1, 2, 3], bad]), sdf[None], sdf[None])
    ends = torch.zeros((2, 2, 3), device=DEV)
    with pytest.raises(RuntimeError, match="outside"):
        _C.tetra_filter(torch.zeros((2, 3), device=DEV), ends, torch.ones((2, 2), device=DEV), torch.tensor([[0, 1, 2]], device=DEV))
    torch.cuda.synchronize()


def test_run_to_run_identity():
    from rade_gs_b200 import tetra
    d = load("sphere_gt")
    evaluate = gpu_sdf(scenes.views_of(d))
    pts, scl = torch.from_numpy(d["points"]).to(DEV), torch.from_numpy(d["scales"]).to(DEV)
    a = tetra.extract_mesh(pts, scl, d["cells"], evaluate)
    b = tetra.extract_mesh(pts, scl, d["cells"], evaluate)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- end to end through the real integrate ----------------------------------------------------------------------------------

def _disc_sphere(P, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.randn(P, 3, generator=g)
    n = n / n.norm(dim=1, keepdim=True)
    # quaternion turning +z onto the normal: (1 + z, -y, x, 0) normalised (w, x, y, z) = rotation about z x n
    q = torch.stack([1 + n[:, 2], -n[:, 1], n[:, 0], torch.zeros(P)], 1)
    q = q / q.norm(dim=1, keepdim=True)
    scales = torch.tensor([0.06, 0.06, 0.003]).repeat(P, 1)
    return n.contiguous(), scales, q


def _camera(eye, W, H, fov):
    from rade_gs_b200 import scenes as sc
    V = sc.look_at_view(eye, (0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0) if abs(eye[2]) < 0.9 * math.dist(eye, (0, 0, 0)) else (0.0, 1.0, 0.0))
    Pm = sc.projection_matrix(0.01, 100.0, fov, fov)
    view = V.t().contiguous()
    proj = (V.t() @ Pm.t()).contiguous()
    campos = torch.linalg.inv(V)[:3, 3].contiguous()
    return view, proj, campos


def test_end_to_end_through_integrate():
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import tetra
    P, W, H, fov = 6000, 160, 160, math.radians(50)
    xyz, scales, rot = _disc_sphere(P, 7)
    xyz, scales, rot = xyz.to(DEV), scales.to(DEV), rot.to(DEV)
    opac = torch.full((P, 1), 0.95, device=DEV)
    shs = torch.zeros((P, 1, 3), device=DEV)
    rng = np.random.default_rng(8)
    eyes = []
    for k in range(20):
        d = rng.normal(size=3)
        eyes.append(tuple(3.5 * d / np.linalg.norm(d)))
    rasts = []
    for e in eyes:
        view, proj, campos = _camera(e, W, H, fov)
        s = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=math.tan(fov / 2), tanfovy=math.tan(fov / 2), kernel_size=0.0,
                                              bg=torch.zeros(3, device=DEV), scale_modifier=1.0, viewmatrix=view.to(DEV), projmatrix=proj.to(DEV),
                                              sh_degree=0, campos=campos.to(DEV), prefiltered=False, require_depth=True, require_coord=True, debug=False)
        rasts.append(dgr.GaussianRasterizer(s))

    compared, ambiguous = [0], [0]

    def evaluate(points):
        cull = tetra.CullSDF(points.shape[0], points.device)
        final = torch.ones(points.shape[0], device=DEV)
        weight = torch.zeros(points.shape[0], dtype=torch.int32, device=DEV)
        amb = torch.zeros(points.shape[0], dtype=torch.bool, device=DEV)
        for r in rasts:
            color, alpha, _, coord, _, _ = r.integrate(points3D=points, means3D=xyz, means2D=None, opacities=opac, shs=shs, scales=scales, rotations=rot)
            cull.add(alpha, coord, color[7])
            # mesh_extract_tetrahedra.py's eager expressions on the same outputs
            pc = coord.clone()
            pc[:, 0] = (pc[:, 0] * 2 + 1) / (W - 1) - 1
            pc[:, 1] = (pc[:, 1] * 2 + 1) / (H - 1) - 1
            prob = torch.nn.functional.grid_sample(color[7][None][None], pc[None, None], padding_mode="zeros", align_corners=False)[0, 0, 0]
            valid = prob > 0.5
            final = torch.where(valid, torch.min(alpha, final), final)
            weight = torch.where(valid, weight + 1, weight)
            p64 = torch.nn.functional.grid_sample(color[7][None][None].double(), pc[None, None].double(), padding_mode="zeros", align_corners=False)
            amb |= (p64[0, 0, 0] - 0.5).abs() < 1e-5
        ours = cull.sdf()
        ref = torch.where(weight > 0, 0.5 - final, -100)
        ok = ~amb
        compared[0] += int(ok.sum())
        ambiguous[0] += int(amb.sum())
        assert torch.equal(ours[ok], ref[ok])
        return ours

    pts, pscl = tetra.tetra_points(xyz, scales, rot)
    cells = tetra.triangulate(pts)
    verts, faces = tetra.extract_mesh(pts, pscl, cells, evaluate)
    r = verts.double().norm(dim=1).cpu().numpy()
    print(f"compared {compared[0]} points ({ambiguous[0]} ambiguous), {len(r)} vertices, {faces.shape[0]} faces, "
          f"|r - 1|: median {np.median(np.abs(r - 1)):.4g}, p99 {np.quantile(np.abs(r - 1), 0.99):.4g}, max {np.abs(r - 1).max():.4g}")
    assert compared[0] > 0.99 * (compared[0] + ambiguous[0])
    assert len(r) > 1000 and faces.shape[0] > 1000
    # the discs are 0.003 thick and 0.06 wide: the extracted surface lies within 0.05 of the unit sphere
    assert np.quantile(np.abs(r - 1), 0.99) < 0.05
