"""GPU checks of rgs_delaunay: the device predicates against the exact model, the cells against scipy in general
position and against the exact checker on degenerate families, and the invariances of the output."""
import itertools

import numpy as np
import pytest
import torch

import delaunay_exact as dx

pytestmark = pytest.mark.gpu


def _dt(p, **kw):
    from rade_gs_b200 import tetra
    x = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p, dtype=np.float32)).cuda()
    return tetra.delaunay(x, **kw)


def _signs(p, tuples):
    from diff_gaussian_rasterization import _C
    return _C._delaunay.predicates(torch.as_tensor(p, dtype=torch.float32).cuda(), torch.as_tensor(tuples, dtype=torch.int32).cuda()).cpu().numpy()


def _model_signs(p, tuples):
    return np.array([(dx.orient3d(*p[t[:4]]), dx.insphere(*p[t]), dx.insphere_perturbed(*p[t])) for t in tuples], dtype=np.int8)


def _tetra_points(P, seed, axis_aligned=False, zero_scale=0, identical=0):
    g = np.random.default_rng(seed)
    xyz = g.normal(size=(P, 3)) * 2
    s = np.exp(g.normal(-4.0, 0.6, size=(P, 3))) * 3
    s[:zero_scale] = 0
    if axis_aligned:
        q = np.tile([1.0, 0, 0, 0], (P, 1))
    else:
        q = g.normal(size=(P, 4))
    if identical:
        xyz[1:identical] = xyz[0]
        s[1:identical] = s[0]
        q[1:identical] = q[0]
    from rade_gs_b200 import tetra
    pts, _ = tetra.tetra_points(torch.tensor(xyz, dtype=torch.float32).cuda(), torch.tensor(s, dtype=torch.float32).cuda(),
                                torch.tensor(q, dtype=torch.float32).cuda())
    return pts.cpu().numpy()


def test_predicates_match_the_exact_model():
    g = np.random.default_rng(0)
    pts = [g.normal(size=(400, 3))]
    sphere = np.array([p for p in itertools.product(range(-25, 26), repeat=3) if p[0] ** 2 + p[1] ** 2 + p[2] ** 2 == 625], dtype=np.float32)
    pts.append(sphere)
    base = g.normal(size=(100, 3)).astype(np.float32)
    flat = base.copy()
    flat[:, 2] = np.nextafter(np.float32(0), np.float32(1)) * g.integers(-2, 3, size=100)   # just off the plane z = 0
    pts.append(flat)
    pts.append(base * np.float32(2.0 ** 118))                                               # ghost-scale magnitudes
    pts.append(np.array(list(itertools.product((0, 1), repeat=3)), dtype=np.float32))
    off_sphere = (sphere / np.float32(25)).astype(np.float32)                                  # fp32 points one ulp off a sphere
    k = g.integers(0, 3, size=len(off_sphere))
    idx = np.arange(len(off_sphere))
    off_sphere[idx, k] = np.nextafter(off_sphere[idx, k], np.float32(2) * np.sign(g.integers(0, 2, len(idx)) - 0.5).astype(np.float32))
    pts.append(off_sphere)
    offsets = np.cumsum([0] + [len(x) for x in pts])
    P = np.concatenate(pts).astype(np.float32)
    tuples = []
    for k in range(len(pts)):
        lo, hi = offsets[k], offsets[k + 1]
        tuples.append(g.integers(lo, hi, size=(6000 if k else 70000, 5)))
    cube = offsets[4]
    tuples.append(np.array([[cube + i for i in perm] for five in itertools.combinations(range(8), 5) for perm in itertools.permutations(five)]))
    T = np.concatenate(tuples).astype(np.int32)
    T = T[np.array([len(set(t)) == 5 for t in T])]
    got = _signs(P, T)
    want = _model_signs(P, T)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, (T[bad[:5]].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
    assert (want[:, 1] == 0).sum() > 1000 and ((want[:, 0] != 0) & (want[:, 2] == 0)).sum() == 0


@pytest.mark.parametrize("n", [5, 100, 10_000, 200_000])
@pytest.mark.parametrize("kind", ["uniform", "gaussian", "clustered"])
def test_against_scipy_in_general_position(n, kind):
    from scipy.spatial import Delaunay
    g = np.random.default_rng(n)
    if kind == "uniform":
        p = g.random((n, 3))
    elif kind == "gaussian":
        p = g.normal(size=(n, 3))
    else:
        p = g.normal(size=(max(n // 50, 1), 3))[g.integers(0, max(n // 50, 1), n)] + g.normal(size=(n, 3)) * 1e-3
    p = p.astype(np.float32)
    ours = _dt(p).cpu().numpy()
    ref = Delaunay(p.astype(np.float64)).simplices
    A = {frozenset(t) for t in ours.tolist()}
    B = {frozenset(t) for t in ref.tolist()}
    assert A <= B
    # the one stated difference from Del(P): a missing cell has a ghost strictly inside its circumsphere
    G = dx.ghosts(p)
    for t in dx.reorient(p, np.array([sorted(c) for c in B - A], dtype=np.int64).reshape(-1, 4)):
        assert any(dx.insphere(*p[t], gh) > 0 for gh in G), t
    if n <= 100:
        dx.check(p, ours)


def _lattice(n):
    return np.array(list(itertools.product(range(n), repeat=3)), dtype=np.float32)


@pytest.mark.parametrize("case", ["lattice3", "lattice5", "tetra_aligned", "tetra_rotated", "duplicates", "one_repeated", "sphere", "skew_lines"])
def test_degenerate_families_pass_the_exact_checker(case):
    g = np.random.default_rng(7)
    lattice = False
    if case.startswith("lattice"):
        p, lattice = _lattice(int(case[-1])), True
    elif case == "tetra_aligned":
        p = _tetra_points(40, 1, axis_aligned=True, zero_scale=3, identical=4)
    elif case == "tetra_rotated":
        p = _tetra_points(40, 2, zero_scale=3, identical=4)
    elif case == "duplicates":
        b = g.normal(size=(300, 3)).astype(np.float32)
        p = np.concatenate([b, b[g.integers(0, 300, 30)]])
        p[g.integers(0, 330, 5)] *= -0.0
    elif case == "one_repeated":
        b = g.normal(size=(200, 3)).astype(np.float32)
        p = np.concatenate([b, np.repeat(b[:1], 10_000, axis=0)])
    elif case == "sphere":
        p = np.array([q for q in itertools.product(range(-25, 26), repeat=3) if q[0] ** 2 + q[1] ** 2 + q[2] ** 2 == 625], dtype=np.float32)
    else:
        t = np.linspace(-1, 1, 300)
        p = np.concatenate([np.stack([t, np.zeros_like(t), np.zeros_like(t) - 1], 1), np.stack([np.zeros_like(t), t, np.ones_like(t)], 1)]).astype(np.float32)
    cells, st = _dt(p, return_stats=True)
    cells = cells.cpu().numpy()
    assert len(cells) > 0
    dx.check(p, cells, lattice=lattice)
    print(case, "points", len(p), "cells", len(cells), st)
    if case == "skew_lines":
        assert st["mesh_growths"] > 0


@pytest.mark.parametrize("case", ["coplanar", "collinear", "three", "empty", "one"])
def test_flat_and_tiny_inputs_give_no_cells(case):
    g = np.random.default_rng(3)
    p = {"coplanar": np.c_[g.normal(size=(50, 2)), np.zeros(50)], "collinear": np.outer(g.normal(size=40), [1, 2, 3]),
         "three": g.normal(size=(3, 3)), "empty": np.zeros((0, 3)), "one": np.zeros((5, 3))}[case]
    assert _dt(p).shape == (0, 4)


def test_shuffle_repeat_poison_and_side_stream_give_the_same_cells():
    from diff_gaussian_rasterization import _C
    g = np.random.default_rng(11)
    p = np.concatenate([_tetra_points(300, 5, zero_scale=2), _lattice(4)])
    p = np.concatenate([p, p[g.integers(0, len(p), 50)]])
    ref = _dt(p).cpu().numpy()
    assert np.array_equal(ref, _dt(p).cpu().numpy())
    perm = g.permutation(len(p))
    got = _dt(p[perm]).cpu().numpy()
    # map back: shuffled index -> original index -> its duplicate class's representative
    rep = {}
    for i, q in enumerate(p.tolist()):
        rep.setdefault(tuple(v + 0.0 for v in q), i)
    to_rep = np.array([rep[tuple(v + 0.0 for v in q)] for q in p.tolist()])
    mapped = to_rep[perm][got]
    assert {frozenset(t) for t in mapped.tolist()} == {frozenset(t) for t in ref.tolist()}
    _C.set_poison(0x7f)
    try:
        s = torch.cuda.Stream()
        x = torch.as_tensor(p).cuda()
        torch.cuda._sleep(20_000_000)
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(s):
            s.wait_event(ev)
            late = _dt(x).cpu().numpy()
        s.synchronize()
    finally:
        _C.set_poison(-1)
    assert np.array_equal(late, ref)


def test_cells_are_canonical_and_sorted():
    p = np.random.default_rng(2).normal(size=(2000, 3)).astype(np.float32)
    c = _dt(p).cpu().numpy()
    assert (c[:, 0] == c.min(axis=1)).all() and (c[:, 1] == c[:, 1:].min(axis=1)).all()
    assert np.all(np.diff(c.astype(np.int64) @ np.array([1 << 45, 1 << 30, 1 << 15, 1])) > 0)
    v = p.astype(np.float64)[c]
    assert (np.linalg.det(v[:, 1:] - v[:, :1]) > 0).all()


def test_growth_on_poisoned_memory_and_a_late_stream_gives_the_same_cells():
    # two skew lines: the mesh outgrows its first capacity several times, and 601 points make it no multiple of 256
    from diff_gaussian_rasterization import _C
    t = np.linspace(-1, 1, 301)
    z = np.zeros_like(t)
    p = np.concatenate([np.stack([t, z, z - 1], 1), np.stack([z, t, z + 1], 1)]).astype(np.float32)
    ref, st = _dt(p, return_stats=True)
    assert st["mesh_growths"] > 0 and (8 * len(p) + 64) % 256 != 0
    ref = ref.cpu().numpy()
    _C.set_poison(0x7f)
    try:
        s = torch.cuda.Stream()
        x = torch.as_tensor(p).cuda()
        torch.cuda._sleep(20_000_000)
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(s):
            s.wait_event(ev)
            late = _dt(x).cpu().numpy()
        s.synchronize()
    finally:
        _C.set_poison(-1)
    assert np.array_equal(late, ref)
    dx.check(p, ref)


def _disc_sphere(P, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.randn(P, 3, generator=g)
    n = n / n.norm(dim=1, keepdim=True)
    q = torch.stack([1 + n[:, 2], -n[:, 1], n[:, 0], torch.zeros(P)], 1)   # turns +z onto the normal
    q = q / q.norm(dim=1, keepdim=True)
    return n.contiguous(), torch.tensor([0.06, 0.06, 0.003]).repeat(P, 1), q


def _camera(eye, W, H, fov):
    import math
    from rade_gs_b200 import scenes as sc
    V = sc.look_at_view(eye, (0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0) if abs(eye[2]) < 0.9 * math.dist(eye, (0, 0, 0)) else (0.0, 1.0, 0.0))
    Pm = sc.projection_matrix(0.01, 100.0, fov, fov)
    return V.t().contiguous(), (V.t() @ Pm.t()).contiguous(), torch.linalg.inv(V)[:3, 3].contiguous()


def _winding(faces):
    """(edges in more than two faces, edges in two faces, those two faces traversing the edge in opposite directions)"""
    f = faces.cpu().numpy()
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und = np.sort(directed, axis=1)
    keys, inv, counts = np.unique(und, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    two = np.nonzero(counts == 2)[0]
    fwd = np.zeros(len(keys), dtype=np.int64)
    np.add.at(fwd, inv, (directed[:, 0] < directed[:, 1]).astype(np.int64))
    return int((counts > 2).sum()), len(two), int((fwd[two] == 1).sum())


def test_end_to_end_through_integrate_on_delaunay_cells():
    """The disc-sphere scene of the tetra tests, meshed on tetra.delaunay cells."""
    import math
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import tetra
    dev = "cuda:0"
    P, W, H, fov = 6000, 160, 160, math.radians(50)
    xyz, scales, rot = (t.to(dev) for t in _disc_sphere(P, 7))
    opac = torch.full((P, 1), 0.95, device=dev)
    shs = torch.zeros((P, 1, 3), device=dev)
    rng = np.random.default_rng(8)
    rasts = []
    for _ in range(20):
        d = rng.normal(size=3)
        view, proj, campos = _camera(tuple(3.5 * d / np.linalg.norm(d)), W, H, fov)
        s = dgr.GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=math.tan(fov / 2), tanfovy=math.tan(fov / 2), kernel_size=0.0,
                                              bg=torch.zeros(3, device=dev), scale_modifier=1.0, viewmatrix=view.to(dev), projmatrix=proj.to(dev),
                                              sh_degree=0, campos=campos.to(dev), prefiltered=False, require_depth=True, require_coord=True, debug=False)
        rasts.append(dgr.GaussianRasterizer(s))

    def evaluate(points):
        cull = tetra.CullSDF(points.shape[0], points.device)
        for r in rasts:
            color, alpha, _, coord, _, _ = r.integrate(points3D=points, means3D=xyz, means2D=None, opacities=opac, shs=shs, scales=scales, rotations=rot)
            cull.add(alpha, coord, color[7])
        return cull.sdf()

    pts, pscl = tetra.tetra_points(xyz, scales, rot)
    cells = tetra.delaunay(pts)
    verts, faces = tetra.extract_mesh(pts, pscl, cells, evaluate)
    r = verts.double().norm(dim=1).cpu().numpy()
    over, two, opposite = _winding(faces)
    scipy_cells = tetra.triangulate(pts)
    _, sfaces = tetra.extract_mesh(pts, pscl, scipy_cells, evaluate)
    s_over, s_two, s_opposite = _winding(sfaces)
    print(f"delaunay: {len(cells)} cells, {len(r)} vertices, {faces.shape[0]} faces, |r - 1| p99 {np.quantile(np.abs(r - 1), 0.99):.4g}; "
          f"edges shared by two faces traversed oppositely (consistent winding): {opposite}/{two}; scipy cells: {s_opposite}/{s_two}")
    assert len(r) > 1000 and faces.shape[0] > 1000
    assert np.quantile(np.abs(r - 1), 0.99) < 0.05
    assert over == 0                       # every mesh edge lies in at most two faces


def test_one_million_tetra_points_pass_the_gpu_checker():
    """About 1 M tetra points (110 k Gaussians): the checker at scale (fp64 on the GPU, the exact model where it cannot decide)."""
    g = np.random.default_rng(21)
    P = 110_000
    from rade_gs_b200 import tetra
    t = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda")  # noqa: E731
    pts, _ = tetra.tetra_points(t(g.normal(size=(P, 3)) * 2), t(np.exp(g.normal(-4.0, 0.6, size=(P, 3))) * 3), t(g.normal(size=(P, 4))))
    cells, st = tetra.delaunay(pts, return_stats=True)
    res = dx.check_gpu(pts, cells)
    print(f"{pts.shape[0]} points, {cells.shape[0]} cells ({cells.shape[0] / pts.shape[0]:.3f} per point), {st}, {res}")
    assert res["negative_cells"] == 0 and res["non_delaunay_faces"] == 0 and not res["faces_in_three_cells"]
    assert set(torch.unique(cells).tolist()) == set(range(pts.shape[0]))   # random Gaussians: no duplicates, all vertices
