"""The bounded TSDF on the GPU (rgs_scalable_* in rgs_tsdf.cu through rade_gs_b200.tsdf.ScalableTSDFVolume and the
extractor) bit-exact against the numpy fp32 model (tests/scalable_f32.py), against the fixture made by the reference's code,
end to end through the rasterizer, and on poisoned memory and a late-ready side stream."""
import math
import os

import numpy as np
import pytest
import torch

import scalable_f32 as M
import tsdf_f32 as T
import tsdf_scenes as ts
from test_gpu_tsdf import same
from test_gpu_unbounded import _Cam, _discs, _Gaussians
from test_scalable_host import fixture, fixture_cameras

pytestmark = pytest.mark.gpu

DEV = "cuda"
F = np.float32

CASES = {
    "rgbd": ["test_bit_exact_against_model", "test_against_the_reference_fixture"],
    "image_u8": ["test_against_the_reference_fixture", "test_image_u8_sweep"],
    "touch": ["test_bit_exact_against_model"],
    "integrate": ["test_bit_exact_against_model", "test_against_the_reference_fixture"],
}


def _np(t):
    return t.detach().cpu().numpy()


def _volume(vs, trunc, block_count=1):
    from rade_gs_b200.tsdf import ScalableTSDFVolume
    return ScalableTSDFVolume(vs, trunc, block_count=block_count)


def _state(vol):
    keys, pool = vol.active_blocks()
    keys, pool = _np(keys), _np(pool).astype(np.int64)
    return (keys, _np(vol.tsdf).reshape(vol.capacity, -1)[pool], _np(vol.weight).reshape(vol.capacity, -1)[pool],
            _np(vol.color).reshape(vol.capacity, -1, 3)[pool])


def _inputs(sc, k, v):
    """render()-like maps of a view: colour pushed outside [0, 1] (so bytes wrap), depth [1, H, W], a mask on every other view."""
    rgb = (np.transpose(v.color, (2, 0, 1)) * F(1.3) - F(0.1)).astype(np.float32)
    mask = None
    if k % 2 == 0:
        mask = (np.random.default_rng(k).random((1,) + v.depth.shape) > 0.1).astype(np.float32)
    return rgb, v.depth[None].copy(), mask


def _fuse(sc, trunc, model=None):
    from rade_gs_b200.tsdf import rgbd_from_color_and_depth
    vol = _volume(sc.vs, trunc)
    for k, v in enumerate(sc.views):
        rgb, depth, mask = _inputs(sc, k, v)
        color, d = rgbd_from_color_and_depth(torch.from_numpy(rgb).to(DEV), torch.from_numpy(depth).to(DEV), sc.depth_max,
                                             None if mask is None else torch.from_numpy(mask).to(DEV))
        units = vol.touch(d, v.K, v.E)
        if model is not None:
            mc, md = M.rgbd(rgb, depth, sc.depth_max, mask)
            assert same(_np(color), mc) and same(_np(d), md), "rgbd differs"
            cam = M.Camera(v.K, v.E, *v.depth.shape, sc.vs, trunc)
            want = M.touch(cam, md)
            assert same(_np(units), want), "touched units differ"
            M.integrate(model, cam, want, md, mc)
        vol.integrate(color, d, v.K, v.E)
    return vol


@pytest.mark.parametrize("family", ts.FAMILIES)
def test_bit_exact_against_model(family):
    sc = ts.make(family)
    trunc = 5 * sc.vs
    model = {}
    vol = _fuse(sc, trunc, model)
    assert vol.capacity > 1 or len(model) <= 1                     # grown from one unit
    keys, t, w, c = _state(vol)
    mk, mt, mw, mc = T.active(model)
    assert same(keys, mk) and same(t, mt) and same(w, mw) and same(c, mc), "volume state differs"
    mesh = vol.extract_triangle_mesh()
    v, col, tri = M.extract(model, sc.vs)
    assert same(_np(mesh.vertices), v) and same(_np(mesh.vertex_colors), col) and same(_np(mesh.triangles), tri), "mesh differs"
    if family not in ("1x1", "7x5"):
        assert tri.shape[0] > 0


def test_image_u8_sweep():
    from diff_gaussian_rasterization import _C
    g = np.random.default_rng(2)
    x = g.uniform(-0.5, 1.5, (3, 37, 53)).astype(np.float32)
    x.reshape(-1)[:8] = [np.nan, np.inf, -np.inf, 0, 1, np.nextafter(F(1), F(0)), -0.0, 3e38]
    for scale, offset in ((1.0, 0.0), (0.5, 0.5)):
        got = _C._scalable_tsdf.image_u8(torch.from_numpy(x).to(DEV), scale, offset)
        assert same(_np(got), M.image_u8(x, scale, offset))


def test_against_the_reference_fixture(tmp_path):
    """The extractor on the fixture's maps: the RGBD the reference handed Open3D, the export's files decoded, and the
    bounded mesh equal to the model fed with the reference's recorded colour, depth and cameras."""
    from PIL import Image

    from rade_gs_b200 import unbounded as ub
    from rade_gs_b200.tsdf import rgbd_from_color_and_depth
    f = fixture()
    cams = fixture_cameras(f, DEV)
    ex = ub.GaussianExtractor.__new__(ub.GaussianExtractor)
    ex.clean()
    ex.viewpoint_stack = cams
    ex.rgbmaps = torch.from_numpy(f["rgb"]).to(DEV)
    ex.depthmaps = torch.from_numpy(f["depth"]).to(DEV)
    ex.normals = torch.from_numpy(f["normals"]).to(DEV)
    ex.export_image(str(tmp_path))
    for name in (k[5:] for k in f if k.startswith("file:")):
        got = np.asarray(Image.open(os.path.join(tmp_path, name)))
        assert same(got, f["file:" + name]), name
    model = {}
    for i, cam in enumerate(cams):
        color, d = rgbd_from_color_and_depth(ex.rgbmaps[i], ex.depthmaps[i], 3, cam.gt_mask)
        rec = f["rec_depth"][i][..., 0]
        assert same(_np(color), f["rec_color"][i]) and same(_np(d), np.where(rec >= 3, F(0), rec))
        W, H, fx, fy, cx, cy = f["rec_intrinsic"][i]
        mcam = M.Camera([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], f["rec_extrinsic"][i], int(H), int(W), 0.004, 0.02)
        M.integrate(model, mcam, M.touch(mcam, _np(d)), _np(d), f["rec_color"][i])
    mesh = ex.extract_mesh_bounded()
    assert same(_np(ex.depthmaps), f["depth"])                     # the stored maps stay unmasked
    v, c, t = M.extract(model, 0.004)
    assert t.shape[0] > 0
    assert same(_np(mesh.vertices), v) and same(_np(mesh.vertex_colors), c) and same(_np(mesh.triangles), t)


def _render(cam, pc, pipe, bg, kernel_size):
    import diff_gaussian_rasterization as dgr
    s = dgr.GaussianRasterizationSettings(image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx / 2),
                                          tanfovy=math.tan(cam.FoVy / 2), kernel_size=kernel_size, bg=bg, scale_modifier=1.0,
                                          viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, sh_degree=0,
                                          campos=cam.camera_center, prefiltered=False, require_depth=True, require_coord=True, debug=False)
    P = pc.get_xyz.shape[0]
    out = dgr.GaussianRasterizer(s)(means3D=pc.get_xyz, means2D=torch.zeros_like(pc.get_xyz), shs=torch.full((P, 1, 3), 1.0, device=DEV),
                                    opacities=torch.full((P, 1), 0.98, device=DEV), scales=pc.scales, rotations=pc.rot)
    color, radii, coord, mcoord, depth, mdepth, alpha, normal = out
    return {"render": color, "median_depth": mdepth, "normal": normal}


def test_end_to_end_sphere(tmp_path):
    """Thin discs on a sphere of radius 0.8, 24 views at 320x240 from 2.6 away, fused at voxel 0.01 and sdf_trunc 0.04.
    Bound, stated before the run: the median vertex lies within one voxel of the sphere, and 99% lie within sdf_trunc
    (the half-pixel offset of the reference's cx = W / 2 and the discs' thickness are both below a voxel here; silhouettes
    against the empty background can pull a few vertices by up to the truncation)."""
    from rade_gs_b200 import unbounded as ub
    import unbounded_scenes as S
    g = torch.Generator().manual_seed(3)
    n = torch.randn(12000, 3, generator=g)
    n = n / n.norm(dim=1, keepdim=True)
    xyz, sc, rot = (x.to(DEV).contiguous() for x in _discs(n * 0.8, n, 0.03))
    cams = [_Cam(e, 320, 240, math.radians(60)) for e in S.ring(24, dist=2.6, height=0.5, seed=4)]
    ex = ub.GaussianExtractor(_Gaussians(xyz, sc, rot), _render, pipe=None, kernel_size=0.0)
    ex.reconstruction(cams)
    assert ex.normals.shape == ex.rgbmaps.shape
    mesh = ex.extract_mesh_bounded(voxel_size=0.01, sdf_trunc=0.04, depth_trunc=3.5, mask_backgrond=False)
    v = _np(mesh.vertices).astype(np.float64)
    e = np.abs(np.linalg.norm(v, axis=1) - 0.8)
    print(f"{len(v)} vertices, {mesh.triangles.shape[0]} triangles; |r - 0.8| median {np.median(e):.4g} p99 {np.quantile(e, .99):.4g} max {e.max():.4g}")
    assert len(v) > 10000
    assert np.median(e) < 0.01 and np.quantile(e, 0.99) < 0.04
    c = _np(mesh.vertex_colors)
    assert (c >= 0).all() and (c <= 1).all()
    for cam in cams:
        cam.original_image = torch.rand(3, 240, 320, device=DEV)
    ex.export_image(str(tmp_path))
    assert len(os.listdir(tmp_path / "vis")) == 2 * len(cams)


def _run(sc, trunc):
    vol = _fuse(sc, trunc)
    m = vol.extract_triangle_mesh()
    return _state(vol) + (_np(m.vertices), _np(m.vertex_colors), _np(m.triangles))


def test_repeat_poison_and_side_stream():
    from diff_gaussian_rasterization import _C
    sc = ts.make("occluders")
    trunc = 5 * sc.vs
    ref = _run(sc, trunc)
    assert all(same(a, b) for a, b in zip(_run(sc, trunc), ref))
    _C.set_poison(0xff)
    try:
        assert all(same(a, b) for a, b in zip(_run(sc, trunc), ref))
        s = torch.cuda.Stream()
        torch.cuda._sleep(20_000_000)
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(s):
            s.wait_event(ev)
            late = _run(sc, trunc)
        s.synchronize()
    finally:
        _C.set_poison(-1)
    assert all(same(a, b) for a, b in zip(late, ref))
