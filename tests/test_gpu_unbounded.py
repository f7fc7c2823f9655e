"""GPU checks of the unbounded-scene mesh (rgs_unbounded_*): every stage bit for bit against the numpy model
(tests/unbounded_f32.py), the whole pipeline across crop seams, the cluster cleanup on its corner cases, an end-to-end run
through this repository's rasterizer, and identical bits on repeat calls, poisoned memory and a late-ready side stream."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import unbounded_f32 as M
import unbounded_scenes as S

pytestmark = pytest.mark.gpu
DEV = "cuda"

# every `_C._unbounded` entry and the tests below that call it (test_unbounded_host checks the list is complete)
CASES = {
    "contract": ["test_contract_both_ways"],
    "sdf": ["test_sdf_every_voxel", "test_sdf_behind_and_on_the_border", "test_against_the_reference_fixture"],
    "colors": ["test_pipeline_across_crop_seams", "test_against_the_reference_fixture"],
    "mcubes": ["test_mcubes_planted_fields", "test_mcubes_closed_surface"],
    "merge": ["test_pipeline_across_crop_seams", "test_merge_keeps_the_first_vertex"],
    "clusters": ["test_clusters"],
}


def _U():
    from diff_gaussian_rasterization import _C
    return _C._unbounded


def _np(t):
    return t.detach().cpu().numpy()


def _eq(a, b):
    """Bit equality; a NaN matches a NaN of any payload (the device and numpy write different quiet NaNs)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(np.where(na, 0, a).view(np.uint8), np.where(nb, 0, b).view(np.uint8))


# ---- contraction ------------------------------------------------------------------------------------------------------

def test_contract_both_ways():
    g = np.random.default_rng(3)
    p = np.concatenate([g.normal(size=(20000, 3)) * s for s in (0.3, 1.0, 5.0, 100.0)]).astype(np.float32)
    p[:4] = [[0, 0, 0], [1, 0, 0], [0, -1, 0], [1e-30, 0, 0]]
    c, r = (0.25, -0.5, 1.0), 2.5
    out, norms = _U().contract(torch.from_numpy(p).to(DEV), list(c), r, False, math.inf)
    ref = M.contract(p, c, r)
    assert _eq(_np(out), ref) and _eq(_np(norms), M.norm3(ref))
    y = (g.uniform(-1.9, 1.9, size=(50000, 3))).astype(np.float32)
    y[:3] = [[2, 0, 0], [0, 1.5, 0], [0.5, 0.5, 0.5]]
    back, _ = _U().contract(torch.from_numpy(y).to(DEV), list(c), r, True, 32.0)
    assert _eq(_np(back), M.inv_contraction(y, c, r, 32.0))
    from rade_gs_b200 import unbounded as ub
    yt = torch.from_numpy(y).to(DEV)
    assert _eq(_np(ub.uncontract(yt)), M.uncontract(y)) and _eq(_np(ub.contract(yt)), M.contract(y))


# ---- SDF --------------------------------------------------------------------------------------------------------------

def _sdf_case(n_views, n, W=40, H=30, seed=0, lo=-1.9, hi=1.9):
    d, c, wv, fp = S.views(n_views, W=W, H=H, seed=seed)
    center, radius = (0.1, -0.05, 0.2), 1.4
    g = np.random.default_rng(seed)
    axes = [np.sort(g.uniform(lo, hi, n)).astype(np.float32) for _ in range(3)]
    return d, fp, center, radius, axes


@pytest.mark.parametrize("n_views,n", [(1, 24), (7, 31), (300, 20)])
def test_sdf_every_voxel(n_views, n):
    d, fp, center, radius, axes = _sdf_case(n_views, n, seed=n_views)
    trunc = float(np.float32(5 * radius * 2 / 64))
    got = _np(_U().sdf(*(torch.from_numpy(a).to(DEV) for a in axes), fp.to(DEV), d.to(DEV), list(center), radius, trunc))
    ref = M.sdf(*axes, fp.numpy(), d.numpy(), center, radius, trunc)
    assert _eq(got, ref)
    assert np.isfinite(got).all() and (got < 1).mean() > 0.01     # some views were fused, nothing became NaN


def test_sdf_behind_and_on_the_border():
    """A projection with h = (x, y, 0, z): u = x / z and v = y / z exactly.  With radius 2 and |samples| < 1 the world
    point is 2 s exactly, so the grid puts samples on u = +-1 and v = +-1 (outside), on the w = 0 plane, behind the camera
    (w < 0), on pixel centres and pixel borders (W - 1 = 16, H - 1 = 8), and at |p| > 1 (the widened truncation)."""
    W, H = 17, 9
    proj = np.zeros((3, 4, 4), np.float32)
    proj[:, 0, 0] = proj[:, 1, 1] = proj[:, 2, 3] = 1.0
    proj[1, 3, 0] = 0.0625                              # a second view shifted by one pixel width / 2
    proj[2, 3, 3] = -0.125                              # a third with the w = 0 plane moved
    g = np.random.default_rng(13)
    depth = g.uniform(0.0, 1.2, (3, H, W)).astype(np.float32)
    k = np.arange(-4, 5, dtype=np.float32) / 8          # multiples of 1/8 in [-0.5, 0.5]
    axes = [np.concatenate([k, np.float32([-0.55, 0.55])]), np.concatenate([k, np.float32([0.03125])]),
            np.float32([-0.25, -0.0625, 0.0, 0.0625, 0.125, 0.25, 0.5, 0.55])]
    n = max(len(a) for a in axes)
    axes = [np.sort(np.resize(a, n)) for a in axes]
    center, radius, trunc = (0.0, 0.0, 0.0), 2.0, float(np.float32(0.3))
    s = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    assert (M.norm3(s) < 1).all()
    got = _np(_U().sdf(*(torch.from_numpy(a).to(DEV) for a in axes), torch.from_numpy(proj).to(DEV), torch.from_numpy(depth).to(DEV),
                       list(center), radius, trunc))
    ref = M.sdf(*axes, proj, depth, center, radius, trunc)
    assert _eq(got, ref) and np.isfinite(got).all()
    with np.errstate(all="ignore"):
        u = s[:, 0] / s[:, 2]
    assert (np.abs(u) == 1).any() and (s[:, 2] == 0).any() and (s[:, 2] < 0).any() and (M.norm3(2 * s) > 1).any()
    assert (got != 1).any()


def test_against_the_reference_fixture():
    """The kernels on the inputs of the fixture made by the reference's own code (tools/gen_golden_unbounded.py): the
    normalisation and R from the device norms, the whole 512^3 volume, the planted vertices' world positions and the
    colours, each bit-equal to the model (which test_unbounded_host checks against the fixture) and within 4x the
    reference's fp32 error against fp64 at every sample away from a discrete decision."""
    from test_unbounded_host import fixture
    from rade_gs_b200 import unbounded as ub
    f = fixture()
    center, radius = ub.normalization(list(f["world_view"]))
    R = ub.scene_bound(torch.from_numpy(f["xyz"]).to(DEV), center, radius)
    Rf = np.asarray(f["R"], dtype=str(f["R_dtype"]))[()]
    assert np.asarray(R).dtype == np.asarray(Rf).dtype and abs(float(R) - float(Rf)) <= 2.0 ** -22
    xs = np.linspace(-Rf, Rf, 512).astype(np.float32)
    trunc = np.float32(5 * float(f["voxel_size"]))
    x = torch.from_numpy(xs).to(DEV)
    vol = _U().sdf(x, x, x, torch.from_numpy(f["full_proj"]).to(DEV), torch.from_numpy(f["depth"]).to(DEV), list(center), radius, float(trunc))
    vx = torch.from_numpy(f["voxels"]).to(DEV)
    got = _np(vol[vx[:, 0], vx[:, 1], vx[:, 2]])
    del vol
    s = np.stack([xs[f["voxels"][:, 0]], xs[f["voxels"][:, 1]], xs[f["voxels"][:, 2]]], -1)
    assert _eq(got, M.sdf_points(s, f["full_proj"], f["depth"], center, radius, trunc))
    keep = f["sdf_keep"]
    ref_err = np.abs(f["sdf"].astype(np.float64) - f["sdf64"])[keep].max()
    assert np.abs(got.astype(np.float64) - f["sdf64"])[keep].max() <= 4 * ref_err + 2.0 ** -24
    (lo, sp, _), = ub.crop_axes(Rf, 512, 512)
    pos = (f["planted"] * np.asarray(sp, np.float64) + np.asarray(lo, np.float64)).astype(np.float32)
    world, _ = _U().contract(torch.from_numpy(pos).to(DEV), list(center), radius, True, 32.0)
    world = _np(world)
    assert _eq(world, M.inv_contraction(pos, center, radius, 32.0))
    kv = f["vertex_keep"]
    assert np.abs(world.astype(np.float64) - f["vertices64"])[kv].max() <= 4 * np.abs(f["vertices"].astype(np.float64) - f["vertices64"])[kv].max()
    col = _np(_U().colors(torch.from_numpy(f["vertices"]).to(DEV), torch.from_numpy(f["full_proj"]).to(DEV), torch.from_numpy(f["depth"]).to(DEV),
                          torch.from_numpy(f["rgb"]).to(DEV), float(trunc)))
    assert _eq(col, M.colors(f["vertices"], f["full_proj"], f["depth"], f["rgb"], trunc))
    kc = f["color_keep"]
    assert np.abs(col.astype(np.float64) - f["colors64"])[kc].max() <= 4 * np.abs(f["colors"].astype(np.float64) - f["colors64"])[kc].max() + 2.0 ** -24


# ---- marching cubes ---------------------------------------------------------------------------------------------------

def _mc(f, lo=(-1.0, -0.5, 0.25), hi=(1.0, 0.7, 1.5)):
    sp = [(b - a) / (f.shape[0] - 1) for a, b in zip(lo, hi)]
    v, t = _U().mcubes(torch.from_numpy(f).to(DEV), list(lo), sp)
    rv, rt = M.mcubes(f, lo, sp)
    assert _eq(_np(v), rv) and _eq(_np(t), rt)
    return rv, rt


def test_mcubes_planted_fields():
    g = np.random.default_rng(11)
    n = 17
    f = g.choice([-1.0, 1.0], size=(n, n, n)).astype(np.float32) * g.uniform(0.1, 2, (n, n, n)).astype(np.float32)
    cs = np.zeros((n - 1,) * 3, np.int64)
    for c in range(8):
        cs |= (f[c & 1:n - 1 + (c & 1), c >> 1 & 1:n - 1 + (c >> 1 & 1), c >> 2 & 1:n - 1 + (c >> 2 & 1)] < 0).astype(np.int64) << c
    assert len(np.unique(cs)) == 256                    # every case
    _mc(f)
    z = f.copy()
    z[g.random(z.shape) < 0.3] = 0.0                   # exact zeros are outside
    z[g.random(z.shape) < 0.05] = -0.0
    _mc(z)
    _mc(np.ones((5, 5, 5), np.float32))                # no sign change: empty
    v, t = _U().mcubes(torch.full((4, 4, 4), -1.0, device=DEV), [0.0] * 3, [1.0] * 3)
    assert v.shape == (0, 3) and t.shape == (0, 3)


def test_mcubes_closed_surface():
    n = 33
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    f = (np.sqrt(X ** 2 + (1.3 * Y) ** 2 + Z ** 2) - 0.7).astype(np.float32)
    v, t = _mc(f, (-1.0,) * 3, (1.0,) * 3)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert (cnt == 2).all()                             # closed: every edge in exactly two faces
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    nrm = np.cross(b - a, c - a)
    out = ((nrm * ((a + b + c) / 3)).sum(1) > 0).mean()
    assert out > 0.999                                  # right-hand normals point to free space (f > 0, outside)


# ---- merge ------------------------------------------------------------------------------------------------------------

def test_merge_keeps_the_first_vertex():
    g = np.random.default_rng(4)
    base = g.uniform(-1.8, 1.8, (500, 3))
    v = np.concatenate([base, base + g.uniform(-4e-7, 4e-7, base.shape), base[::-1]])
    t = g.integers(0, len(v), (900, 3)).astype(np.int32)
    t[0] = [0, 500, 1000 - 1]                           # all three merge: a degenerate triangle that stays
    mv, mt = _U().merge(torch.from_numpy(v).to(DEV), torch.from_numpy(t).to(DEV))
    rv, rt = M.merge(v, t)
    assert _eq(_np(mv), rv) and _eq(_np(mt), rt)
    with pytest.raises(RuntimeError, match="out of range"):
        _U().merge(torch.from_numpy(v).to(DEV), torch.tensor([[0, 1, len(v)]], dtype=torch.int32, device=DEV))
    with pytest.raises(RuntimeError, match="not finite"):
        _U().merge(torch.tensor([[np.nan, 0, 0]], dtype=torch.float64, device=DEV), torch.zeros((0, 3), dtype=torch.int32, device=DEV))


# ---- the pipeline across crop seams -------------------------------------------------------------------------------------

def _model_pipeline(d, c, wv, fp, xyz, resolution, crop):
    from rade_gs_b200 import unbounded as ub
    center, radius = ub.normalization(list(wv))
    R = ub.scene_bound(xyz.to(DEV), center, radius)
    trunc = float(np.float32(5 * (radius * 2 / resolution)))
    verts, tris, base = [], [], 0
    for lo, sp, axes in ub.crop_axes(R, resolution, crop):
        f = M.sdf(*axes, fp.numpy(), d.numpy(), center, radius, trunc)
        v, t = M.mcubes(f, [float(x) for x in lo], [float(x) for x in sp])
        if len(t):
            verts.append(v)
            tris.append(t + base)
            base += len(v)
    mv, mt = M.merge(np.concatenate(verts), np.concatenate(tris))
    world = M.inv_contraction(mv, center, radius, 32.0)
    return world, mt, M.colors(world, fp.numpy(), d.numpy(), c.numpy(), trunc)


def _pipeline(d, c, wv, fp, xyz, resolution, crop):
    from rade_gs_b200 import unbounded as ub
    m = ub.extract_mesh_unbounded_maps(d.to(DEV), c.to(DEV), list(wv), fp, xyz.to(DEV), resolution=resolution, crop=crop)
    return _np(m.vertices), _np(m.triangles), _np(m.vertex_colors)


def test_pipeline_across_crop_seams():
    d, c, wv, fp = S.views(6, W=48, H=36, seed=2)
    xyz = S.sphere_xyz(3000)
    got = _pipeline(d, c, wv, fp, xyz, 48, 24)
    ref = _model_pipeline(d, c, wv, fp, xyz, 48, 24)
    for a, b in zip(got, ref):
        assert _eq(a, b)
    assert len(got[1]) > 500
    # seams are joined: no vertex of the merged mesh is within 1e-6 (contracted) of another
    from rade_gs_b200 import unbounded as ub
    center, radius = ub.normalization(list(wv))
    y = M.contract(got[0], center, radius)
    k = np.rint(y.astype(np.float64) * 1e6)
    assert len(np.unique(k, axis=0)) >= len(k) - 2      # two vertices may meet after the fp32 round trip


# ---- clusters ---------------------------------------------------------------------------------------------------------

def _strip(n, start, off=0):
    """n triangles in a strip (edge-connected), vertices from `start`."""
    return np.array([[start + i, start + i + 1, start + i + 2] for i in range(n)], np.int32) + off


def _cluster_case(name):
    if name == "ties":
        parts = [_strip(60, 0), _strip(60, 100), _strip(70, 200), _strip(55, 300)]
        return 400, np.concatenate(parts), 2
    if name == "exactly_50":
        return 300, np.concatenate([_strip(50, 0), _strip(49, 100), _strip(51, 200)]), 1000
    if name == "non_manifold":      # three triangles on one edge, plus a vertex-only contact
        t = np.concatenate([[[0, 1, 2], [0, 1, 3], [1, 0, 4]], _strip(60, 10), [[12, 40, 41]]]).astype(np.int32)
        return 100, t, 1
    if name == "degenerate":
        t = np.concatenate([_strip(60, 0), [[5, 5, 6], [70, 70, 70], [80, 81, 80]]]).astype(np.int32)
        return 90, t, 1
    if name == "vertex_contact":
        return 200, np.concatenate([_strip(60, 0), [[0, 100, 101]], _strip(55, 101)]), 1
    if name == "empty":
        return 10, np.zeros((0, 3), np.int32), 5
    if name == "few_clusters":
        g = np.random.default_rng(1)
        t = np.concatenate([_strip(int(k), 300 * i) for i, k in enumerate(g.integers(1, 120, 40))])
        return 12000, t[g.permutation(len(t))], 1000
    if name == "random":
        g = np.random.default_rng(2)
        return 5000, g.integers(0, 5000, (20000, 3)).astype(np.int32), 3
    if name == "keep_zero":
        return 400, np.concatenate([_strip(60, 0), _strip(80, 100)]), 0
    raise KeyError(name)


@pytest.mark.parametrize("name", ["ties", "exactly_50", "non_manifold", "degenerate", "vertex_contact", "empty", "few_clusters", "random", "keep_zero"])
def test_clusters(name):
    V, t, k = _cluster_case(name)
    t = t.astype(np.int32)
    vi, tt, st = _U().clusters(V, torch.from_numpy(t).to(DEV), k)
    rv, rt, sizes = M.clusters(V, t, k)
    assert _eq(_np(vi).astype(np.int64), rv) and _eq(_np(tt), rt)
    assert st["num_clusters"] == len(sizes)
    with pytest.raises(RuntimeError, match="out of range"):
        _U().clusters(3, torch.tensor([[0, 1, 3]], dtype=torch.int32, device=DEV), 1)


def test_post_process_mesh_carries_attributes():
    from rade_gs_b200 import tsdf, unbounded as ub
    V, t, k = _cluster_case("degenerate")
    g = np.random.default_rng(0)
    v = torch.from_numpy(g.normal(size=(V, 3)).astype(np.float32)).to(DEV)
    c = torch.from_numpy(g.random((V, 3)).astype(np.float32)).to(DEV)
    m = tsdf.TriangleMesh(v, torch.from_numpy(t).to(DEV), c)
    out = ub.post_process_mesh(m, 1)
    rv, rt, _ = M.clusters(V, t, 1)
    assert _eq(_np(out.vertices), _np(v)[rv]) and _eq(_np(out.vertex_colors), _np(c)[rv]) and _eq(_np(out.triangles), rt)


# ---- repeats, poisoned memory, a late side stream ---------------------------------------------------------------------

def test_repeat_poison_and_side_stream():
    from diff_gaussian_rasterization import _C
    d, c, wv, fp = S.views(4, W=40, H=30, seed=7)
    xyz = S.sphere_xyz(2000)
    ref = _pipeline(d, c, wv, fp, xyz, 40, 20)
    V, t, k = _cluster_case("random")
    cref = [_np(x) for x in _U().clusters(V, torch.from_numpy(t).to(DEV), k)[:2]]
    assert all(_eq(a, b) for a, b in zip(_pipeline(d, c, wv, fp, xyz, 40, 20), ref))
    _C.set_poison(0xff)
    try:
        assert all(_eq(a, b) for a, b in zip(_pipeline(d, c, wv, fp, xyz, 40, 20), ref))
        s = torch.cuda.Stream()
        dd, cc, tt = d.to(DEV), c.to(DEV), torch.from_numpy(t).to(DEV)
        torch.cuda._sleep(20_000_000)
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(s):
            s.wait_event(ev)
            from rade_gs_b200 import unbounded as ub
            m = ub.extract_mesh_unbounded_maps(dd, cc, list(wv), fp, xyz.to(DEV), resolution=40, crop=20)
            cl = _U().clusters(V, tt, k)
            late = (_np(m.vertices), _np(m.triangles), _np(m.vertex_colors))
            clate = [_np(x) for x in cl[:2]]
        s.synchronize()
    finally:
        _C.set_poison(-1)
    assert all(_eq(a, b) for a, b in zip(late, ref)) and all(_eq(a, b) for a, b in zip(clate, cref))


# ---- end to end through the rasterizer --------------------------------------------------------------------------------

class _Cam:
    def __init__(self, eye, W, H, fov):
        self.world_view_transform, self.full_proj_transform = (x.to(DEV) for x in S.camera(eye, W=W, H=H, fovx=fov))
        self.camera_center = torch.linalg.inv(self.world_view_transform)[3, :3]
        self.image_width, self.image_height = W, H
        self.FoVx = fov
        self.FoVy = 2 * math.atan(math.tan(fov / 2) * H / W)


class _Gaussians:
    def __init__(self, xyz, scales, rot):
        self.get_xyz, self.scales, self.rot = xyz, scales, rot


def _discs(points, normals, size):
    n = normals / normals.norm(dim=1, keepdim=True)
    q = torch.stack([1 + n[:, 2], -n[:, 1], n[:, 0], torch.zeros(len(n))], 1)
    bad = q.norm(dim=1) < 1e-6
    q[bad] = torch.tensor([0.0, 1.0, 0.0, 0.0])
    q = q / q.norm(dim=1, keepdim=True)
    return points, torch.tensor([size, size, size * 0.05]).repeat(len(points), 1), q


def _render(cam, pc, pipe, bg, kernel_size):
    import diff_gaussian_rasterization as dgr
    s = dgr.GaussianRasterizationSettings(image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx / 2),
                                          tanfovy=math.tan(cam.FoVy / 2), kernel_size=kernel_size, bg=bg, scale_modifier=1.0,
                                          viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, sh_degree=0,
                                          campos=cam.camera_center, prefiltered=False, require_depth=True, require_coord=True, debug=False)
    P = pc.get_xyz.shape[0]
    shs = torch.full((P, 1, 3), 1.0, device=DEV)
    out = dgr.GaussianRasterizer(s)(means3D=pc.get_xyz, means2D=torch.zeros_like(pc.get_xyz), shs=shs, opacities=torch.full((P, 1), 0.98, device=DEV),
                                    scales=pc.scales, rotations=pc.rot)
    color, radii, coord, mcoord, depth, mdepth, alpha, normal = out
    return {"render": color, "median_depth": mdepth}


def test_end_to_end_sphere_and_plane():
    from rade_gs_b200 import unbounded as ub
    g = torch.Generator().manual_seed(3)
    n = torch.randn(12000, 3, generator=g)
    n = n / n.norm(dim=1, keepdim=True)
    sph = _discs(n * 0.8, n, 0.03)
    xy = torch.rand(20000, 2, generator=g) * 6 - 3
    pl = _discs(torch.cat([xy, torch.full((len(xy), 1), -1.0)], 1), torch.tensor([[0.0, 0.0, 1.0]]).repeat(len(xy), 1), 0.04)
    xyz, sc, rot = (torch.cat([a, b]).to(DEV).contiguous() for a, b in zip(sph, pl))
    cams = [_Cam(e, 320, 240, math.radians(60)) for e in S.ring(24, dist=2.6, height=0.5, seed=4)]
    ex = ub.GaussianExtractor(_Gaussians(xyz, sc, rot), _render, pipe=None, kernel_size=0.0)
    ex.reconstruction(cams)
    mesh = ex.extract_mesh_unbounded(resolution=512)
    v = _np(mesh.vertices).astype(np.float64)
    t = _np(mesh.triangles)
    r = np.linalg.norm(v, axis=1)
    near_sphere = (np.abs(r - 0.8) < 0.1) & (v[:, 2] > -0.6)
    near_plane = (np.abs(v[:, 2] + 1.0) < 0.1) & (np.hypot(v[:, 0], v[:, 1]) < 1.6) & (r > 1.0)
    assert near_sphere.sum() > 1000 and near_plane.sum() > 1000
    es, ep = np.abs(r[near_sphere] - 0.8), np.abs(v[near_plane, 2] + 1.0)
    print(f"{len(v)} vertices, {len(t)} triangles; sphere |r - 0.8| median {np.median(es):.4g} p99 {np.quantile(es, .99):.4g}; "
          f"plane |z + 1| median {np.median(ep):.4g} p99 {np.quantile(ep, .99):.4g}")
    # grid_sample(align_corners=True) reads the maps half a pixel off the rasterizer's pixel centres (a quirk of the
    # reference kept here), which shifts surfaces seen at grazing angles, such as the plane, by about a voxel
    vox = 2 * 2.6 / 512
    assert np.median(es) < vox and np.median(ep) < 3 * vox
    # the tails: the window holds the inner shell about one truncation (5 voxels) behind each surface (below)
    q = lambda a, p: float(np.quantile(a, p)) / vox           # noqa: E731
    print(f"in voxels: sphere p90 {q(es, .9):.2f} p99 {q(es, .99):.2f}; plane p90 {q(ep, .9):.2f} p99 {q(ep, .99):.2f}")
    assert q(es, 0.99) < 6 and q(ep, 0.9) < 8
    # normals point outward (free space): on the sphere away from the centre, on the plane up.  Space behind a surface
    # that no view sees keeps the initial tsdf 1, so the reference's TSDF also has an inner shell about one truncation
    # (5 voxels) behind each surface, facing inward; the check takes the vertices within 2 (sphere) / 3 (plane) voxels.
    # Near each view's silhouette of the sphere, the background depth pushes points just inside it positive, which leaves
    # small inward-facing pockets close to the surface: 0.86 of the sphere's vertices were outward on an H100
    mesh.compute_vertex_normals()
    nv = _np(mesh.vertex_normals)
    outer = near_sphere & (np.abs(r - 0.8) < 2 * vox)
    top = near_plane & (np.abs(v[:, 2] + 1.0) < 3 * vox)
    fs, fp_ = ((nv[outer] * v[outer]).sum(1) > 0).mean(), (nv[top, 2] > 0).mean()
    print(f"outward normals: sphere {fs:.4f} of {outer.sum()}, plane {fp_:.4f} of {top.sum()}")
    so = near_sphere & ((nv * v).sum(1) > 0)
    po = near_plane & (nv[:, 2] > 0)
    print(f"outward-facing, in voxels: sphere p99 {q(np.abs(r[so] - 0.8), .99):.2f}, plane p99 {q(np.abs(v[po, 2] + 1), .99):.2f}")
    assert fs > 0.8 and fp_ > 0.95
    # outward-facing vertices are the surface itself: their tail stays within a few voxels (the plane's is wider: it is
    # seen at grazing angles through the half-pixel offset above)
    assert q(np.abs(r[so] - 0.8), 0.99) < 1.5 and q(np.abs(v[po, 2] + 1), 0.99) < 5     # observed 0.53 and 3.77 on an H100
    cleaned = ub.post_process_mesh(mesh, cluster_to_keep=1000)
    assert 0 < cleaned.triangles.shape[0] <= t.shape[0]
