"""CPU checks of the Tanks and Temples cull: the numpy model of the header contracts (tests/tnt_cull_model.py) against
analytic scenes and against the reference's unmodified ``eval_tnt/cull_mesh.py`` (tests/golden/tnt_cull, made by
tools/gen_golden_tnt_cull.py), and the host side of rade_gs_b200.tnt_cull.  No GPU."""
import glob
import os

import numpy as np
import pytest
import torch

import tnt_cull_model as M
from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "tnt_cull")
H, W, FX, FY, CX, CY = 48, 64, 50.0, 50.0, 32.0, 24.0
EYE = M.w2c_rows(np.eye(4))[0]


def quad(z, half=5.0):
    v = np.array([[-half, -half, z], [half, -half, z], [half, half, z], [-half, half, z]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]])


def test_plane_depth_within_its_fp32_bound_at_every_pixel():
    """A tilted plane Z = 3 + 0.2 X: the model's depth is the exact ray hit within a few ulps at every pixel."""
    v = np.array([[-8, -8, 3 - 1.6], [8, -8, 3 + 1.6], [8, 8, 3 + 1.6], [-8, 8, 3 - 1.6]], np.float32)
    d = M.mesh_depth(v, [[0, 1, 2], [0, 2, 3]], EYE, FX, FY, CX, CY, H, W)
    dx = (np.arange(W) + 0.5 - CX) / FX
    exact = 3.0 / (1.0 - 0.2 * dx)[None, :].repeat(H, 0)
    assert (d > 0).all()
    assert np.abs(d - exact).max() <= 32 * np.finfo(np.float32).eps * exact.max()


def test_fronto_parallel_plane_is_exact():
    d = M.mesh_depth(*quad(2.0), EYE, FX, FY, CX, CY, H, W)
    assert (d == np.float32(2.0)).all()


def test_closed_cube_seen_from_inside_leaves_no_pixel_uncovered():
    c = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    f = np.array([t for q in quads for t in ((q[0], q[1], q[2]), (q[0], q[2], q[3]))])
    for k, pose in enumerate([np.eye(4), M_rot(0.7, 0.3), M_rot(-1.2, 2.0)]):
        d = M.mesh_depth(c, f, M.w2c_rows(pose)[0], 20.0, 20.0, CX, CY, H, W)   # wide field: every wall is on screen
        assert (d > 0).all(), k


def M_rot(a, b):
    ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(b), np.sin(b)
    R = np.array([[ca, 0, sa], [0, 1, 0], [-sa, 0, ca]]) @ np.array([[1, 0, 0], [0, cb, -sb], [0, sb, cb]])
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = [0.1, -0.2, 0.05]
    return T


@pytest.mark.parametrize("vertical", [True, False])
def test_shared_edge_through_pixel_centres_is_covered_once(vertical):
    """An edge on the line u = 32.5 (or v = 20.5) through a column (row) of pixel centres: each centre belongs to exactly
    one of the two faces, whichever winding they have."""
    z = 2.0
    e = np.float32(0.5 / FX * z) if vertical else np.float32(-3.5 / FY * z)
    if vertical:
        v = np.array([[e, -5, z], [e, 5, z], [-5, 0, z], [5, 0, z]], np.float32)
    else:
        v = np.array([[-5, e, z], [5, e, z], [0, -5, z], [0, 5, z]], np.float32)
    for f in ([[0, 1, 2], [1, 0, 3]], [[0, 1, 2], [0, 1, 3]], [[1, 0, 2], [1, 0, 3]]):
        a = M.mesh_depth(v, [f[0]], EYE, FX, FY, CX, CY, H, W) > 0
        b = M.mesh_depth(v, [f[1]], EYE, FX, FY, CX, CY, H, W) > 0
        assert not (a & b).any()
        assert (a | b).all()


def test_triangle_crossing_the_near_plane_is_clipped_not_dropped():
    v = np.array([[-1, -1, -1], [1, -1, 3], [0, 1, 3]], np.float32)
    d = M.mesh_depth(v, [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W, znear=0.5)
    assert (d > 0).sum() > 100 and d[d > 0].min() >= 0.5
    assert M.split(v, [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W, 0.5) == (0, 1, 0)
    # its box is that of the clipped polygon: no covered pixel lies outside it
    draws, box, *_ = M.setup(v, [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W, 0.5, 20.0)
    ys, xs = np.nonzero(d)
    assert draws[0] and box[0, 0] <= xs.min() and xs.max() <= box[0, 2] and box[0, 1] <= ys.min() and ys.max() <= box[0, 3]
    assert box[0, 2] - box[0, 0] < W - 1 or box[0, 3] - box[0, 1] < H - 1
    full = M.mesh_depth(v, [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W, znear=0.5, chunk=1 << 30)
    assert np.array_equal(d, full)
    # every vertex behind the near plane: nothing
    assert (M.mesh_depth(v - [0, 0, 5], [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W) == 0).all()


def test_triangle_far_beyond_the_screen_keeps_its_on_screen_pixels():
    v = np.array([[-1e6, -1e6, 4], [1e6, -1e6, 4], [0, 1e6, 4]], np.float32)
    d = M.mesh_depth(v, [[0, 1, 2]], EYE, FX, FY, CX, CY, H, W)
    assert (d == np.float32(4.0)).all()


def test_far_plane_degenerate_and_empty():
    assert (M.mesh_depth(*quad(25.0), EYE, FX, FY, CX, CY, H, W) == 0).all()
    v = np.array([[0, 0, 2], [1, 0, 2], [2, 0, 2], [0, 1, 2]], np.float32)
    assert (M.mesh_depth(v, [[0, 1, 2], [0, 0, 3], [3, 3, 3]], EYE, FX, FY, CX, CY, H, W) == 0).all()
    assert (M.mesh_depth(np.zeros((0, 3)), np.zeros((0, 3), int), EYE, FX, FY, CX, CY, H, W) == 0).all()


def test_visibility_frustum_borders_and_occlusion():
    D = np.zeros((H, W), np.float32)
    D[:, : W // 2] = 3.0
    pts = np.array([[(W - 1 - CX) / FX * 2, 0, 2],     # u = W - 1 (border, in)
                    [(W - 1 - CX) / FX * 2 + 1e-3, 0, 2],   # just outside
                    [0, 0, 0], [0, 0, -1],            # z = 1e-8 (in: z > 0), behind
                    [-0.5, 0, 2.0], [-0.5, 0, 3.1], [-0.5, 0, 3.004]], np.float32)
    seen, fr, z, s = M.visibility(pts, D, EYE, FX, FY, CX, CY)
    assert list(seen) == [True, False, True, False, True, False, True]


def _margins(p, D, m, fx, fy, cx, cy, eps):
    """Views whose decision lies within a margin of a threshold, where the reference (torch fp32 inverse, matmul order,
    CPU division) may decide otherwise."""
    seen, fr, z, s = M.visibility(p, D, m, fx, fy, cx, cy, eps)
    X, Y, Z = M.to_camera(m, np.asarray(p, np.float32))
    with np.errstate(all="ignore"):
        u, v = fx * X / Z + cx, fy * Y / Z + cy
    Hh, Ww = D.shape
    near = (np.abs(u) < 1e-3) | (np.abs(u - (Ww - 1)) < 1e-3) | (np.abs(v) < 1e-3) | (np.abs(v - (Hh - 1)) < 1e-3)
    near |= fr & (s > 0) & (np.abs(z - (s + np.float32(eps))) < 1e-4 * np.maximum(1.0, np.abs(z)))
    return seen, near


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "small_*.npz"))), ids=os.path.basename)
def test_model_against_the_reference_script(path):
    g = np.load(path)
    Hh, Ww, fx, fy, cx, cy, far = g["camera"]
    Hh, Ww = int(Hh), int(Ww)
    ms = M.w2c_rows(g["c2w"] @ np.diag([1.0, -1.0, -1.0, 1.0]))
    for k, m in enumerate(ms):   # the shipped pose: pyrender's camera is the flipped OpenCV pose
        assert np.array_equal(M.mesh_depth(g["vertices"], g["faces"], m, fx, fy, cx, cy, Hh, Ww, 0.01, far), g["depths"][k]), k
    certain = np.zeros(len(g["vertices"]), np.int64)
    unsure = np.zeros_like(certain)
    for D, m in zip(g["depths"], M.w2c_rows(g["c2w"])):
        seen, near = _margins(g["vertices"], D, m, fx, fy, cx, cy, 0.005)
        certain += seen & ~near
        unsure += near
    decided = (certain >= 20) | (certain + unsure < 20)
    assert decided.mean() > 0.97, f"{(~decided).sum()} undecided"
    assert np.array_equal((certain >= 20)[decided], g["mask"][decided])
    # the face and vertex filter of update_faces + remove_unreferenced_vertices
    keep = g["mask"][g["faces"]].all(1)
    used = np.zeros(len(g["vertices"]), bool)
    used[g["faces"][keep].reshape(-1)] = True
    assert np.array_equal(g["cull_vertices"], g["vertices"][used])
    assert np.array_equal(g["cull_faces"], (np.cumsum(used) - 1)[g["faces"][keep]])


def test_main_run_of_the_reference_script():
    g = np.load(os.path.join(GOLDEN, "main_hd.npz"))
    assert np.array_equal(g["log_mask"], g["npy_mask"]) and np.array_equal(g["log_cull_faces"], g["npy_cull_faces"])
    assert 0 < g["log_mask"].sum() < len(g["log_mask"])
    assert len(g["log_depth_sha256"]) == len(g["c2w"])


# ---- host side of rade_gs_b200.tnt_cull -------------------------------------------------------------------------------------

def test_load_poses_pads_3x4_npy_and_reads_log(tmp_path):
    from rade_gs_b200 import tnt_cull
    c = np.stack([M_rot(0.1 * k, 0.2) for k in range(3)])
    np.save(tmp_path / "t.npy", c[:, :3, :])
    assert np.array_equal(tnt_cull.load_poses(str(tmp_path / "t.npy")), c)
    np.save(tmp_path / "u.npy", c)
    assert np.array_equal(tnt_cull.load_poses(str(tmp_path / "u.npy")), c)
    with open(tmp_path / "t.log", "w") as f:
        for k, T in enumerate(c):
            f.write(f"{k} {k} 0\n" + "\n".join(" ".join(repr(float(x)) for x in r) for r in T) + "\n")
    assert np.array_equal(tnt_cull.load_poses(str(tmp_path / "t.log")), c)
    with pytest.raises(ValueError, match="json"):
        tnt_cull.load_poses(str(tmp_path / "t.json"))
    np.save(tmp_path / "bad.npy", np.zeros((2, 2, 4)))
    with pytest.raises(ValueError):
        tnt_cull.load_poses(str(tmp_path / "bad.npy"))


def test_w2c_is_the_fp64_inverse_of_the_fp32_pose():
    from rade_gs_b200 import tnt_cull
    c = np.stack([M_rot(0.3, -0.4), M_rot(1.0, 0.1)])
    assert np.array_equal(np.array(tnt_cull._w2c(c), np.float32), M.w2c_rows(c))


def test_host_side_rejections():
    from rade_gs_b200 import tnt_cull
    v, f = quad(2.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        tnt_cull.cull_mesh(v, f, np.eye(4)[None], device="cpu")
    bad = v.copy()
    bad[0, 0] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        tnt_cull._mesh(torch.as_tensor(bad), torch.as_tensor(f), "cpu")
    with pytest.raises(ValueError, match="face index"):
        tnt_cull._mesh(torch.as_tensor(v), torch.as_tensor([[0, 1, 4]]), "cpu")
    with pytest.raises(ValueError, match="NaN"):
        tnt_cull._poses(np.full((1, 4, 4), np.inf))
    with pytest.raises(ValueError):
        tnt_cull._poses(np.eye(3))
    with pytest.raises(ValueError, match="znear"):
        tnt_cull._check_camera(10, 10, 0.0, 1.0)
    with pytest.raises(ValueError, match="znear"):
        tnt_cull._check_camera(10, 10, 2.0, 1.0)
    with pytest.raises(ValueError):
        tnt_cull._check_camera(1, 10, 0.01, 1.0)


def test_cli_parses_the_reference_arguments(monkeypatch, tmp_path):
    from rade_gs_b200 import tnt_cull
    seen = {}

    def fake(vertices, faces, c2w, H, W, fx, fy, cx, cy, far, eps, min_views, depth_c2w):
        seen.update(H=H, W=W, fx=fx, far=far, eps=eps, min_views=min_views, depth_c2w=depth_c2w, n=len(c2w))
        return torch.as_tensor(vertices), torch.as_tensor(faces), torch.ones(len(vertices), dtype=torch.bool), None

    monkeypatch.setattr(tnt_cull, "cull_mesh", fake)
    from rade_gs_b200 import ply_io
    v, f = quad(2.0)
    ply_io.save_triangle_mesh_ply(str(tmp_path / "m.ply"), v, f)
    np.save(tmp_path / "t.npy", np.eye(4)[None, :3, :].repeat(2, 0))
    out = tnt_cull.main(["--traj-path", str(tmp_path / "t.npy"), "--ply-path", str(tmp_path / "m.ply")])
    assert out == str(tmp_path / "m_cull.ply") and os.path.exists(out)
    assert seen == dict(H=1080, W=1920, fx=1163.8678928442187, far=20.0, eps=0.005, min_views=20, depth_c2w=None, n=2)
    tnt_cull.main(["--traj-path", str(tmp_path / "t.npy"), "--ply-path", str(tmp_path / "m.ply"), "--shipped-depth-pose", "--min-views", "3"])
    assert seen["min_views"] == 3 and np.array_equal(seen["depth_c2w"][0], np.diag([1.0, -1.0, -1.0, 1.0]))
