"""The Tanks and Temples cull kernels on the GPU: every depth map and every count bit for bit against the numpy model of
the header contracts (tests/tnt_cull_model.py), the reference script's fixtures end to end, a scene with a known answer,
and identical bits on repeat calls, poisoned memory and a late-ready side stream."""
import glob
import os

import numpy as np
import pytest
import torch

import tnt_cull_model as M
from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "tnt_cull")
FLIP = np.diag([1.0, -1.0, -1.0, 1.0])
H, W, FX, FY, CX, CY = 90, 160, 97.3, 98.1, 80.37, 44.62


def _C():
    from diff_gaussian_rasterization import _C
    return _C._tnt_cull


def look_at(eye, target):
    z = np.asarray(target, float) - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, [0.0, -1.0, 0.0])
    x /= np.linalg.norm(x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, np.cross(z, x), z, eye
    return T


def kernel_depth(v, f, m=M.w2c_rows(np.eye(4))[0], H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY, znear=0.01, zfar=20.0):
    vt = torch.as_tensor(np.asarray(v, np.float32).reshape(-1, 3), device="cuda")
    ft = torch.as_tensor(np.asarray(f, np.int32).reshape(-1, 3), device="cuda")
    return _C().mesh_depth(vt, ft, [float(x) for x in m], fx, fy, cx, cy, H, W, znear, zfar).cpu().numpy()


def same_depth(v, f, pose, **k):
    m = M.w2c_rows(pose)[0]
    d = kernel_depth(v, f, m, **k)
    ref = M.mesh_depth(v, f, m, k.get("fx", FX), k.get("fy", FY), k.get("cx", CX), k.get("cy", CY), k.get("H", H), k.get("W", W),
                       k.get("znear", 0.01), k.get("zfar", 20.0))
    assert np.array_equal(d.view(np.uint32), ref.view(np.uint32)), f"{(d != ref).sum()} pixels differ"
    return d


def grid(o, du, dv, n):
    s = np.linspace(0.0, 1.0, n + 1)
    a, b = np.meshgrid(s, s, indexing="ij")
    v = o + a.reshape(-1, 1) * du + b.reshape(-1, 1) * dv
    i = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    q = np.stack([i[:-1, :-1], i[1:, :-1], i[1:, 1:], i[:-1, 1:]], -1).reshape(-1, 4)
    return v, np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])


def merge(parts):
    vs, fs, off = [], [], 0
    for v, f in parts:
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs)


def box(lo, hi, n):
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    parts = []
    for ax in range(3):
        u, w = [k for k in range(3) if k != ax]
        for side in (lo[ax], hi[ax]):
            o = lo.copy()
            o[ax] = side
            du, dv = np.zeros(3), np.zeros(3)
            du[u], dv[w] = hi[u] - lo[u], hi[w] - lo[w]
            parts.append(grid(o, du, dv, n))
    return parts


def room():
    return merge(box([-3, -1.5, -3], [3, 1.5, 3], 24) + box([-0.5, -1.5, -0.5], [0.5, 0.3, 0.5], 6) + box([1.2, -1.5, 0.8], [2.0, -0.2, 2.4], 5))


ROOM_POSES = [look_at(np.array(e), np.array(t)) for e, t in [((0, 0, -2.9), (0, 0, 0)), ((2.95, 0.5, 2.9), (0, 0, 0)), ((-1, 1.4, 0), (1, -1, 1)),
                                                             ((0.3, 0.2, -0.52), (0, 0, 3)), ((-2.99, -1.0, -2.99), (3, 1, 3))]]


@pytest.mark.parametrize("k", range(len(ROOM_POSES)))
def test_room_with_occluders_and_cameras_at_the_walls(k):
    v, f = room()
    d = same_depth(v, f, ROOM_POSES[k])
    assert (d > 0).mean() > 0.5


def test_million_subpixel_triangles_and_each_side_of_the_split():
    rng = np.random.default_rng(5)
    n = 1_000_000
    p = rng.uniform([-3, -2, 3], [3, 2, 9], (n, 3))
    v = np.concatenate([p, p + rng.normal(0, 0.004, (n, 3)), p + rng.normal(0, 0.004, (n, 3))]).astype(np.float32)
    f = np.arange(3 * n).reshape(3, n).T
    big, bf = merge([grid(np.array([-2.0, -1.0, 6.0]), np.array([1.0, 0, 0]), np.array([0, 1.0, 0]), 4),    # medium boxes
                     grid(np.array([-20.0, -20.0, 9.5]), np.array([40.0, 0, 0]), np.array([0, 40.0, 0]), 1)])  # screen-sized
    v = np.concatenate([v, big])
    f = np.concatenate([f, bf + 3 * n])
    small, medium, large = M.split(v, f, M.w2c_rows(np.eye(4))[0], FX, FY, CX, CY, H, W)
    assert small > 0.9 * n and medium >= 8 and large >= 1
    same_depth(v, f, np.eye(4))


def test_one_screen_covering_triangle_and_triangles_on_one_pixel():
    v = np.array([[-100, -100, 5], [100, -100, 5.5], [0, 100, 4]], np.float32)
    d = same_depth(v, [[0, 1, 2]], np.eye(4))
    assert (d > 0).all()
    rng = np.random.default_rng(1)
    c = np.array([(10.5 - CX) / FX * 3, (7.5 - CY) / FY * 3, 3.0])
    tv = (c + rng.normal(0, 0.002, (3000, 3))).astype(np.float32)
    same_depth(tv, np.arange(3000).reshape(-1, 3), np.eye(4))


def test_duplicate_degenerate_far_cut_and_empty():
    v, f = room()
    f2 = np.concatenate([f, f[:500], f[:500, [0, 0, 1]], f[:500, [2, 2, 2]]])
    same_depth(v, f2, ROOM_POSES[0])
    same_depth(v, f, ROOM_POSES[1], zfar=3.0)
    same_depth(v, f, ROOM_POSES[2], znear=0.7)
    assert (kernel_depth(np.zeros((0, 3)), np.zeros((0, 3))) == 0).all()
    assert (kernel_depth(v, np.zeros((0, 3))) == 0).all()


def test_intrinsics_and_image_sizes():
    v, f = room()
    for H_, W_, fx, fy, cx, cy in [(1, 1, 1.0, 1.0, 0.5, 0.5), (37, 211, 150.0, 75.0, -20.3, 60.0), (1080, 1920, 1163.8678928442187, 1172.793101201448,
                                                                                                      962.3120628412543, 542.0667209577691)]:
        same_depth(v, f, ROOM_POSES[3], H=H_, W=W_, fx=fx, fy=fy, cx=cx, cy=cy)


def test_bad_index_and_arguments_are_rejected():
    v, f = room()
    with pytest.raises(RuntimeError, match="outside"):
        kernel_depth(v, np.array([[0, 1, len(v)]]))
    with pytest.raises(RuntimeError, match="znear"):
        kernel_depth(v, f, M.w2c_rows(np.eye(4))[0], znear=0.0)
    with pytest.raises(RuntimeError, match="znear"):
        kernel_depth(v, f, M.w2c_rows(np.eye(4))[0], znear=2.0, zfar=1.0)


def kernel_counts(p, depths, ms, fx=FX, fy=FY, cx=CX, cy=CY, eps=0.005):
    pt = torch.as_tensor(np.asarray(p, np.float32), device="cuda")
    counts = torch.zeros(len(pt), dtype=torch.int32, device="cuda")
    for D, m in zip(depths, ms):
        _C().visibility_count(pt, torch.as_tensor(np.asarray(D, np.float32), device="cuda"), [float(x) for x in m], fx, fy, cx, cy, eps, counts)
    return counts.cpu().numpy()


def test_counts_bit_exact_on_borders_behind_the_camera_and_occlusion():
    v, f = room()
    poses = ROOM_POSES
    ms = M.w2c_rows(np.stack(poses))
    depths = [M.mesh_depth(v, f, m, FX, FY, CX, CY, H, W) for m in ms]
    rng = np.random.default_rng(2)
    pts = [v, rng.uniform(-3.2, 3.2, (200000, 3)).astype(np.float32)]
    # points on the u = W - 1, u = 0, v = H - 1 borders and the z = 0 plane of the first camera
    c2w = poses[0]
    for u, w, z in [(W - 1, 40.0, 2.0), (0.0, 10.0, 1.0), (60.0, H - 1, 3.0), (30.0, 30.0, 0.0), (30.0, 30.0, -1.0)]:
        cam = np.array([(u - CX) / FX * z, (w - CY) / FY * z, z, 1.0]) if z else np.array([0.3, 0.1, 0.0, 1.0])
        pts.append((c2w @ cam)[None, :3].astype(np.float32))
    p = np.concatenate(pts)
    assert np.array_equal(kernel_counts(p, depths, ms), M.visibility_count(p, depths, ms, FX, FY, CX, CY))


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "small_*.npz"))), ids=os.path.basename)
def test_reference_fixtures_end_to_end_in_shipped_pose_mode(path):
    from rade_gs_b200 import tnt_cull
    g = np.load(path)
    Hh, Ww, fx, fy, cx, cy, far = g["camera"]
    Hh, Ww = int(Hh), int(Ww)
    d = tnt_cull.render_depth(g["vertices"], g["faces"], g["c2w"] @ FLIP, Hh, Ww, fx, fy, cx, cy, zfar=far).cpu().numpy()
    assert np.array_equal(d, g["depths"])
    cv, cf, valid, counts = tnt_cull.cull_mesh(g["vertices"], g["faces"], g["c2w"], Hh, Ww, fx, fy, cx, cy, far, depth_c2w=g["c2w"] @ FLIP)
    ms = M.w2c_rows(g["c2w"])
    assert np.array_equal(counts.cpu().numpy(), M.visibility_count(g["vertices"], g["depths"], ms, fx, fy, cx, cy))
    # the fixture's mask, where no view decides within a margin of a threshold (tests/test_tnt_cull_host.py)
    from test_tnt_cull_host import _margins
    certain = np.zeros(len(g["vertices"]), np.int64)
    unsure = np.zeros_like(certain)
    for D, m in zip(g["depths"], ms):
        seen, near = _margins(g["vertices"], D, m, fx, fy, cx, cy, 0.005)
        certain += seen & ~near
        unsure += near
    decided = (certain >= 20) | (certain + unsure < 20)
    assert np.array_equal(valid.cpu().numpy()[decided], g["mask"][decided])
    if np.array_equal(valid.cpu().numpy(), g["mask"]):
        assert np.array_equal(cv.cpu().numpy(), g["cull_vertices"]) and np.array_equal(cf.cpu().numpy(), g["cull_faces"])


def test_reference_main_run_end_to_end(tmp_path):
    import hashlib
    from rade_gs_b200 import ply_io, tnt_cull
    g = np.load(os.path.join(GOLDEN, "main_hd.npz"))
    ply_io.save_triangle_mesh_ply(str(tmp_path / "mesh.ply"), g["vertices"], g["faces"])
    np.save(tmp_path / "traj.npy", g["c2w"][:, :3, :])
    d = tnt_cull.render_depth(g["vertices"], g["faces"], g["c2w"] @ FLIP, 1080, 1920, tnt_cull.FX, tnt_cull.FY, tnt_cull.CX, tnt_cull.CY)
    sha = [hashlib.sha256(np.ascontiguousarray(x, np.float32).tobytes()).hexdigest() for x in d.cpu().numpy()]
    assert sha == list(g["log_depth_sha256"])
    out = tnt_cull.main(["--traj-path", str(tmp_path / "traj.npy"), "--ply-path", str(tmp_path / "mesh.ply"), "--shipped-depth-pose"])
    v, f = ply_io.load_triangle_mesh_ply(out)
    assert len(f) == len(g["npy_cull_faces"]) or abs(len(f) - len(g["npy_cull_faces"])) <= 0.01 * len(g["faces"])


def test_box_hidden_behind_a_wall_is_culled_and_the_wall_kept():
    """Consistent camera convention: a wall between every camera and a box.  The box's vertices are never seen; the
    wall's camera-facing grid is seen by every camera and kept."""
    from rade_gs_b200 import tnt_cull
    wall = grid(np.array([-3.0, -2.0, 0.0]), np.array([6.0, 0, 0]), np.array([0, 4.0, 0]), 20)
    hidden = merge(box([-0.5, -0.5, 1.0], [0.5, 0.5, 2.0], 4))
    v, f = merge([wall, hidden])
    poses = np.stack([look_at(np.array([x, y, -3.0]), np.array([0.0, 0.0, 1.0])) for x in np.linspace(-0.6, 0.6, 5) for y in (-0.3, 0.0, 0.3, 0.5)])
    cv, cf, valid, counts = tnt_cull.cull_mesh(v, f, poses, H, W, FX, FY, CX, CY, 20.0)
    nw = len(wall[0])
    valid = valid.cpu().numpy()
    assert not valid[nw:].any()
    centre = np.linalg.norm(wall[0][:, :2], axis=1) < 1.0
    assert valid[:nw][centre].all()
    assert len(cf) > 0 and int(cf.max()) < len(cv)


def test_repeat_poison_and_side_stream():
    from diff_gaussian_rasterization import _C as C
    v, f = room()
    m = [float(x) for x in M.w2c_rows(ROOM_POSES[1])[0]]
    vt = torch.as_tensor(v, device="cuda")
    ft = torch.as_tensor(f.astype(np.int32), device="cuda")

    def run():
        d = _C().mesh_depth(vt, ft, m, FX, FY, CX, CY, H, W, 0.01, 20.0)
        c = torch.zeros(len(vt), dtype=torch.int32, device="cuda")
        _C().visibility_count(vt, d, m, FX, FY, CX, CY, 0.005, c)
        return d.cpu().numpy(), c.cpu().numpy()

    d0, c0 = run()
    d1, c1 = run()
    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32)) and np.array_equal(c0, c1)
    try:
        C.set_poison(0x5a)
        d2, c2 = run()
    finally:
        C.set_poison(-1)
    assert np.array_equal(d0.view(np.uint32), d2.view(np.uint32)) and np.array_equal(c0, c2)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        vs = vt.clone()
        d = _C().mesh_depth(vs, ft, m, FX, FY, CX, CY, H, W, 0.01, 20.0)
        c = torch.zeros(len(vs), dtype=torch.int32, device="cuda")
        _C().visibility_count(vs, d, m, FX, FY, CX, CY, 0.005, c)
    torch.cuda.current_stream().wait_stream(side)
    assert np.array_equal(d.cpu().numpy().view(np.uint32), d0.view(np.uint32)) and np.array_equal(c.cpu().numpy(), c0)
