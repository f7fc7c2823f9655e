"""TSDF fusion and marching cubes on the GPU (rgs_tsdf.cu through rade_gs_b200.tsdf) bit-exact against the numpy fp32 model
(tests/tsdf_f32.py): grid state, touched blocks, mesh and normals compared with np.array_equal, no tolerance."""
import math
import time

import numpy as np
import pytest
import torch

import tsdf_f32 as m
import tsdf_scenes as ts
from test_tsdf_host import manifold_report

pytestmark = pytest.mark.gpu

DEV = "cuda"


def VBG(*a, **kw):
    from rade_gs_b200.tsdf import VoxelBlockGrid
    return VoxelBlockGrid(*a, **kw)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8) if a.size else a, b.view(np.uint8) if b.size else b)


def gpu_fuse(sc, block_count=50000, check_touch=True, model=None):
    vbg = VBG(sc.vs, block_count=block_count)
    for v in sc.views:
        d = torch.from_numpy(v.depth).to(DEV)
        c = torch.from_numpy(v.color).to(DEV)
        coords = vbg.compute_unique_block_coordinates(d, v.K, v.E, sc.depth_scale, sc.depth_max, sc.trunc_mult)
        if check_touch:
            cam = m.Camera(v.K, v.E, *v.depth.shape, sc.vs, sc.depth_scale, sc.depth_max, sc.trunc_mult)
            want = m.touch(cam, v.depth)
            assert same(coords.cpu().numpy(), want), "touched blocks differ"
            if model is not None:
                m.integrate(model, cam, want, v.depth, v.color)
        vbg.integrate(coords, d, c, torch.from_numpy(v.K), v.E, sc.depth_scale, sc.depth_max, sc.trunc_mult)
    return vbg


def grid_state(vbg):
    keys, pool = vbg.active_blocks()
    keys, pool = keys.cpu().numpy(), pool.cpu().numpy().astype(np.int64)
    t = vbg.attribute("tsdf").cpu().numpy().reshape(vbg.capacity, -1)[pool]
    w = vbg.attribute("weight").cpu().numpy().reshape(vbg.capacity, -1)[pool]
    c = vbg.attribute("color").cpu().numpy().reshape(vbg.capacity, -1, 3)[pool]
    return keys, t, w, c


def check_mesh(vbg, model, vs, thr=3.0):
    mesh = vbg.extract_triangle_mesh(thr).compute_vertex_normals()
    v, c, t = m.extract(model, vs, thr)
    assert same(mesh.vertices.cpu().numpy(), v), "vertices differ"
    assert same(mesh.vertex_colors.cpu().numpy(), c), "vertex colours differ"
    assert same(mesh.triangles.cpu().numpy(), t), "triangles differ"
    assert same(mesh.vertex_normals.cpu().numpy(), m.vertex_normals(v, t)), "normals differ"
    return mesh


@pytest.mark.parametrize("family", ts.FAMILIES)
def test_bit_exact_against_model(family):
    sc = ts.make(family)
    model = {}
    vbg = gpu_fuse(sc, model=model)
    keys, t, w, c = grid_state(vbg)
    mk, mt, mw, mc = m.active(model)
    assert same(keys, mk) and same(t, mt) and same(w, mw) and same(c, mc), "grid state differs"
    mesh = check_mesh(vbg, model, sc.vs)
    if family == "few_views":
        assert mesh.triangles.shape[0] == 0 and w.max() < 3
    elif family not in ("1x1", "7x5"):
        assert mesh.triangles.shape[0] > 0
    if family == "on_grid":
        assert (t == 0).sum() > 100                      # exactly-zero tsdf occurs, and counts as outside


def test_planted_random_fields_hit_every_case():
    """Blocks allocated by an integrate that updates nothing (all-zero depth), then random fields written through
    attribute(): every one of the 256 cube cases occurs in a valid cell, and the mesh is bit-exact."""
    rng = np.random.default_rng(5)
    vs = 0.05
    vbg = VBG(vs, block_count=64)
    blocks = np.array([[x, y, z] for x in range(-2, 2) for y in range(-1, 2) for z in range(2)], np.int32)
    blocks = blocks[rng.permutation(len(blocks))]
    K, E = ts.intrinsic(8, 8), np.eye(4)
    zero = torch.zeros(8, 8, device=DEV)
    vbg.integrate(torch.from_numpy(blocks).to(DEV), zero, torch.zeros(8, 8, 3, device=DEV), K, E)
    keys, pool = vbg.active_blocks()
    n = len(keys)
    assert n == len(blocks) and same(keys.cpu().numpy(), np.sort(m.pack(blocks)))
    tsdf = rng.uniform(-1, 1, (n, m.BV)).astype(np.float32)
    tsdf[rng.random(tsdf.shape) < 0.02] = 0.0
    weight = np.where(rng.random((n, m.BV)) < 0.97, rng.integers(3, 9, (n, m.BV)), rng.integers(0, 3, (n, m.BV))).astype(np.float32)
    color = rng.random((n, m.BV, 3)).astype(np.float32)
    p = pool.long()
    vbg.attribute("tsdf").view(vbg.capacity, -1)[p] = torch.from_numpy(tsdf).to(DEV)
    vbg.attribute("weight").view(vbg.capacity, -1)[p] = torch.from_numpy(weight).to(DEV)
    vbg.attribute("color").view(vbg.capacity, -1, 3)[p] = torch.from_numpy(color).to(DEV)
    model = {int(k): (tsdf[i].copy(), weight[i].copy(), color[i].copy()) for i, k in enumerate(keys.cpu().numpy())}
    # which cases occur in valid cells (the model's own classification)
    cases = set()
    for i in range(n):
        ins = tsdf[i].reshape(16, 16, 16) < 0                     # [z, y, x]
        ok = weight[i].reshape(16, 16, 16) >= 3
        code = np.zeros((15, 15, 15), np.int64)
        allok = np.ones((15, 15, 15), bool)
        for cnr in range(8):
            cx, cy, cz = m.CORNERS[cnr]
            code |= ins[cz:cz + 15, cy:cy + 15, cx:cx + 15].astype(np.int64) << cnr
            allok &= ok[cz:cz + 15, cy:cy + 15, cx:cx + 15]
        cases.update(np.unique(code[allok]).tolist())
    assert len(cases) == 256
    check_mesh(vbg, model, vs)


def test_capacity_growth_and_determinism():
    sc = ts.make("occluders")
    a = gpu_fuse(sc, block_count=8, check_touch=False)
    b = gpu_fuse(sc, block_count=50000, check_touch=False)
    c = gpu_fuse(sc, block_count=50000, check_touch=False)
    assert a.capacity > 8
    sa, sb, sc_ = grid_state(a), grid_state(b), grid_state(c)
    for x, y, z in zip(sa, sb, sc_):
        assert same(x, y) and same(y, z)
    ma, mb, mc = (g.extract_triangle_mesh().compute_vertex_normals() for g in (a, b, c))
    for k in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
        assert same(getattr(ma, k).cpu().numpy(), getattr(mb, k).cpu().numpy())
        assert same(getattr(mb, k).cpu().numpy(), getattr(mc, k).cpu().numpy())


def test_duplicate_block_coordinates_update_once():
    sc = ts.make("fronto")
    v = sc.views[0]
    d, c = torch.from_numpy(v.depth).to(DEV), torch.from_numpy(v.color).to(DEV)
    g1, g2 = VBG(sc.vs), VBG(sc.vs)
    coords = g1.compute_unique_block_coordinates(d, v.K, v.E)
    g1.integrate(coords, d, c, v.K, v.E)
    g2.integrate(torch.cat([coords, coords.flip(0), coords]), d, c, v.K, v.E)
    for x, y in zip(grid_state(g1), grid_state(g2)):
        assert same(x, y)


def test_full_coverage_sphere_is_watertight():
    sc = ts.sphere_scene(30, 96, 80, vs=0.02, r=0.3, dist=1.2)
    sc.trunc_mult = 4.0
    mesh = gpu_fuse(sc, check_touch=False).extract_triangle_mesh()
    boundary, bad, chi, vol = manifold_report(mesh.vertices.cpu().numpy(), mesh.triangles.cpu().numpy().astype(np.int64))
    assert mesh.triangles.shape[0] > 500 and boundary == 0 and bad == 0 and chi == 2 and vol > 0


def test_input_validation():
    from rade_gs_b200.tsdf import VoxelBlockGrid
    K, E = ts.intrinsic(8, 6), np.eye(4)
    vbg = VoxelBlockGrid(0.01)
    d = torch.ones(6, 8, device=DEV)
    col = torch.ones(6, 8, 3, device=DEV)
    with pytest.raises(ValueError, match="block_resolution must be 16"):
        VoxelBlockGrid(0.01, block_resolution=8)
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="voxel_size"):
            VoxelBlockGrid(bad)
    with pytest.raises(RuntimeError, match="no CPU path"):
        vbg.compute_unique_block_coordinates(d.cpu(), K, E)
    with pytest.raises(RuntimeError, match="float32"):
        vbg.compute_unique_block_coordinates(d.double(), K, E)
    with pytest.raises(RuntimeError, match=r"\[H, W\]"):
        vbg.compute_unique_block_coordinates(d[None], K, E)
    with pytest.raises(RuntimeError, match="contiguous"):
        vbg.compute_unique_block_coordinates(torch.ones(8, 6, device=DEV).t(), K, E)
    with pytest.raises(ValueError, match="intrinsic"):
        vbg.compute_unique_block_coordinates(d, np.eye(4), E)
    coords = vbg.compute_unique_block_coordinates(d, K, E)
    with pytest.raises(RuntimeError, match="int32"):
        vbg.integrate(coords.long(), d, col, K, E)
    with pytest.raises(RuntimeError, match="contiguous"):
        vbg.integrate(coords.t().contiguous().t(), d, col, K, E)
    with pytest.raises(RuntimeError, match="no CPU path"):
        vbg.integrate(coords, d, col.cpu(), K, E)
    with pytest.raises(RuntimeError, match=r"\[H, W, 3\]"):
        vbg.integrate(coords, d, col[..., :2].contiguous(), K, E)
    far = np.eye(4)
    far[0, 3] = -0.16 * 2 ** 20                     # camera centre at x = 0.16 * 2^20: outside the block-key range
    with pytest.raises(RuntimeError, match="key range"):
        vbg.compute_unique_block_coordinates(d, K, far)
    with pytest.raises(RuntimeError, match="key range"):
        vbg.integrate(coords, d, col, K, far)
    bad = torch.tensor([[2 ** 20, 0, 0]], dtype=torch.int32, device=DEV)
    vbg.integrate(bad, d, col, K, E)                # found on the device, reported by the next call that reads the counters
    with pytest.raises(RuntimeError, match="outside"):
        vbg.extract_triangle_mesh()
    from rade_gs_b200.tsdf import TriangleMesh
    tm = TriangleMesh(torch.zeros(3, 3, device=DEV), torch.tensor([[0, 1, 3]], dtype=torch.int32, device=DEV), torch.zeros(3, 3, device=DEV))
    with pytest.raises(RuntimeError, match="out of"):
        tm.compute_vertex_normals()


def test_frame_hash_growth():
    """A view touching more blocks than the initial frame-local hash holds: the grid doubles it and the result is unchanged."""
    sc = ts.make("800x600")
    v = sc.views[0]
    d = torch.from_numpy(v.depth).to(DEV)
    small = VBG(sc.vs, block_count=1)
    got = small.compute_unique_block_coordinates(d, v.K, v.E)
    assert small.frame_keys.numel() > 4
    cam = m.Camera(v.K, v.E, *v.depth.shape, sc.vs, 1.0, sc.depth_max, 8.0)
    assert same(got.cpu().numpy(), m.touch(cam, v.depth))


def _quat_z_to(n):
    """(w, x, y, z) rotating +z onto the unit vectors n [P, 3]."""
    z = np.array([0.0, 0.0, 1.0])
    axis = np.cross(z, n)
    s = np.linalg.norm(axis, axis=1, keepdims=True)
    ang = np.arctan2(s[:, 0], n[:, 2])
    axis = np.where(s > 1e-12, axis / np.maximum(s, 1e-12), [1.0, 0.0, 0.0])
    return np.concatenate([np.cos(ang / 2)[:, None], np.sin(ang / 2)[:, None] * axis], 1)


def test_end_to_end_through_the_rasterizer():
    """Thin discs tangent to a sphere, rendered with GaussianRasterizer, fused from mesh_extract.py's median_depth (alpha < 0.5
    masked to 0, cx = W / 2) and extracted.  Bound, stated before the run: the median depth lies within the disc's
    thickness (3 sigma_n, doubled for oblique rays inside the band); the half-pixel offset between mesh_extract.py's
    cx = W / 2 and the pixel centres the rasterizer samples shifts a sample by half a footprint, at a slope <= 2 in the band;
    one more footprint for the pixel chosen by floor; plus vs^2 / (8 r) for interpolation and trunc / 2 for grazing views
    (as in the host sphere test)."""
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import scenes
    from rade_gs_b200.tsdf import VoxelBlockGrid
    r, dist, vs, W, H, fov = 0.3, 1.2, 0.01, 128, 128, math.radians(50)
    P = 6000
    ctr = ts.orbit(P, r)
    nrm = ctr / r
    spacing = math.sqrt(4 * math.pi * r * r / P)
    sig_t, sig_n = 0.9 * spacing, 0.0005
    dev = torch.device(DEV)
    means = torch.tensor(ctr, dtype=torch.float32, device=dev)
    scales = torch.tensor([[sig_t, sig_t, sig_n]] * P, dtype=torch.float32, device=dev)
    rots = torch.tensor(_quat_z_to(nrm), dtype=torch.float32, device=dev)
    opac = torch.full((P, 1), 0.98, device=dev)
    cols = torch.tensor(0.5 + 0.5 * nrm, dtype=torch.float32, device=dev)
    f = W / (2 * math.tan(fov / 2))
    trunc_mult = 4.0
    bound = 2 * 3 * sig_n + 2 * 0.5 * (dist + r) / f + 2 * (dist + r) / f + vs * vs / (8 * r) + trunc_mult * vs / 2
    vbg = VoxelBlockGrid(vs, block_count=2000)
    proj = scenes.projection_matrix(0.01, 100.0, fov, fov).t().to(dev)
    for eye in ts.orbit(30, dist, seed=0.3):
        V = scenes.look_at_view(tuple(eye), (0.0, 0.0, 0.0)).to(dev)
        view = V.t().contiguous()
        s = dgr.GaussianRasterizationSettings(H, W, math.tan(fov / 2), math.tan(fov / 2), 0.0, torch.ones(3, device=dev), 1.0, view,
                                              (view @ proj).contiguous(), 0, torch.tensor(eye, dtype=torch.float32, device=dev), False, True, False, False)
        out = dgr.GaussianRasterizer(s)(means, torch.zeros_like(means), opac, colors_precomp=cols, scales=scales, rotations=rots)
        color, mdepth, alpha = out[0], out[5], out[6]
        depth = mdepth.clone()
        depth[alpha < 0.5] = 0
        K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
        ext = view.t().cpu().numpy().astype(np.float64)
        img = torch.clamp(color, 0, 1).permute(1, 2, 0).contiguous()
        coords = vbg.compute_unique_block_coordinates(depth[0].contiguous(), K, ext, 1.0, 8.0, trunc_mult)
        vbg.integrate(coords, depth[0].contiguous(), img, K, ext, 1.0, 8.0, trunc_mult)
    mesh = vbg.extract_triangle_mesh().compute_vertex_normals()
    v = mesh.vertices.cpu().numpy().astype(np.float64)
    assert len(v) > 1000
    err = np.abs(np.linalg.norm(v, axis=1) - r)
    assert err.max() < bound, (err.max(), bound)
    n = mesh.vertex_normals.cpu().numpy()
    assert np.mean(np.sum(n * v / np.linalg.norm(v, axis=1, keepdims=True), 1) > 0.9) > 0.95   # normals point outward


def test_dtu_sized_run_under_a_coarse_bound():
    """49 views at 800x600, vs = 0.002, depth_max = 8 (mesh_extract.py's settings).  A probing or quadratic blow-up takes
    minutes; the expected time is well under a second."""
    sc = ts.sphere_scene(49, 800, 600, vs=0.002, r=0.3, dist=1.2, depth_max=8.0)
    views = [(torch.from_numpy(v.depth).to(DEV), torch.from_numpy(v.color).to(DEV), v.K, v.E) for v in sc.views]
    vbg = VBG(0.002)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for d, c, K, E in views:
        coords = vbg.compute_unique_block_coordinates(d, K, E, 1.0, 8.0)
        vbg.integrate(coords, d, c, K, E, 1.0, 8.0)
    mesh = vbg.extract_triangle_mesh().compute_vertex_normals()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert mesh.triangles.shape[0] > 10000
    assert dt < 30.0, f"{dt:.1f} s"
