"""DTU evaluation without a GPU: the fp64 model (tests/dtu_eval_f64.py) against fixtures made by the reference's own
eval.py and cull_mesh (tools/gen_golden_dtu_eval.py), the PLY readers, and the package's imports."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import dtu_eval_f64 as model
from conftest import GOLDEN_DIR, ROOT

DTU_DIR = os.path.join(GOLDEN_DIR, "dtu_eval")
SCANS = ["mesh_a", "mesh_b", "pcd"]


def load(name):
    return dict(np.load(os.path.join(DTU_DIR, name + ".npz")))


@pytest.mark.parametrize("name", SCANS)
def test_model_equals_reference_eval(name):
    d = load(name)
    density = float(d["density"])
    if str(d["mode"]) == "mesh":
        assert np.array_equal(model.sample(d["vertices"], d["faces"], density), d["original"])
    else:
        assert np.array_equal(d["points"], d["original"])
    shuffled = d["original"][d["perm"]]
    kept = model.greedy_downsample(shuffled, density)
    assert np.array_equal(kept, d["kept"])
    down = shuffled[kept]
    idx, d2s, s2d, m_d2s, m_s2d = model.mask_and_score(down, d["stl"], d["obs_mask"], d["bb"], d["res"], d["plane"], float(d["patch"]),
                                                       float(d["max_dist"]))
    assert np.array_equal(idx, d["in_obs"])
    assert np.array_equal(d2s, d["dist_d2s"]) and np.array_equal(s2d, d["dist_s2d"])
    np.testing.assert_allclose([m_d2s, m_s2d], d["means"][:2], rtol=1e-12, atol=0)
    assert 0 < len(idx) < len(down) and 0 < len(s2d) < len(d["stl"])   # the scenes exercise both filters


def cull_cameras(d):
    W, H = (int(x) for x in d["size"])
    return [types.SimpleNamespace(world_view_transform=torch.tensor(d["w2c_t"][k]), FoVx=float(d["fov"][k, 0]), FoVy=float(d["fov"][k, 1]),
                                  image_width=W, image_height=H, gt_mask=torch.tensor(d["masks"][k])) for k in range(len(d["w2c_t"]))]


def reference_keep(d):
    rows = {tuple(r) for r in d["culled_vertices"]}
    return np.array([tuple(r) in rows for r in d["vertices"]])


def test_cull_model_against_reference_cull():
    from rade_gs_b200 import dtu_eval
    d = load("cull")
    cams = cull_cameras(d)
    proj = dtu_eval.cull_projections(cams)
    W, H = (int(x) for x in d["size"])
    dil = np.stack([model.dilate(m[0]) for m in d["masks"]])
    keep = model.cull_keep(d["vertices"], proj, dil)
    ref = reference_keep(d)
    assert len(ref) == len(keep) and ref.sum() == len(d["culled_vertices"])
    near = model.cull_near_boundary(d["vertices"], proj, W, H)
    print(f"cull: {int(near.sum())} of {len(near)} vertices within 1e-3 px of a rounding or border boundary excluded")
    assert near.sum() < 0.05 * len(near)   # 5 views x 2 axes x a 2e-3 px band: about 2 %
    assert np.array_equal(keep[~near], ref[~near])
    assert 0 < ref.sum() < len(ref)
    if np.array_equal(keep, ref):
        new = np.cumsum(keep) - 1
        faces = d["faces"][keep[d["faces"]].all(1)]
        assert np.array_equal(new[faces], d["culled_faces"])


def test_dilation_footprint_is_disk6():
    assert model.DISK6.sum() == 113
    m = np.zeros((20, 20), np.uint8)
    m[10, 10] = 1
    assert model.dilate(m).sum() == 113
    m = np.zeros((20, 20), np.uint8)
    m[0, 0] = 1                                    # outside the image counts as unset
    assert model.dilate(m).sum() == sum(1 for y in range(7) for x in range(7) if x * x + y * y <= 36)


# ---- PLY readers ----------------------------------------------------------------------------------------------------------

PTS = np.array([[1.5, -2.25, 3.0], [500.125, 499.875, 501.0], [0.0, 1e-3, -7.0]])
TRIS = np.array([[0, 1, 2], [2, 1, 0]])


def _write(path, fmt, xyz_type, count_type, with_faces=True, ascii_=False):
    order = {"binary_little_endian": "<", "binary_big_endian": ">"}.get(fmt)
    np_t = {"float": "f4", "double": "f8", "int": "i4"}[xyz_type]
    cnt_t = {"uchar": "u1", "ushort": "u2", "int": "i4"}[count_type]
    xyz = PTS.astype(np_t)
    hdr = ["ply", f"format {fmt} 1.0", "comment hand-built", "element camera 1", "property float k",
           f"element vertex {len(PTS)}", f"property {xyz_type} x", "property uchar red", f"property {xyz_type} y", f"property {xyz_type} z",
           "property float nx"]
    if with_faces:
        hdr += [f"element face {len(TRIS)}", f"property list {count_type} int vertex_indices", "property uchar flags"]
    hdr += ["element edge 1", "property int a", "property int b", "end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(hdr) + "\n").encode())
        if ascii_:
            lines = ["0.5"] + [f"{x} 7 {y} {z} 0.25" for x, y, z in xyz.tolist()]
            if with_faces:
                lines += [f"3 {a} {b} {c} 1" for a, b, c in TRIS]
            lines += ["0 1"]
            f.write(("\n".join(lines) + "\n").encode())
            return
        f.write(np.array([0.5], order + "f4").tobytes())
        vrec = np.empty(len(PTS), [("x", order + np_t), ("r", "u1"), ("y", order + np_t), ("z", order + np_t), ("nx", order + "f4")])
        vrec["x"], vrec["y"], vrec["z"], vrec["r"], vrec["nx"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], 7, 0.25
        f.write(vrec.tobytes())
        if with_faces:
            frec = np.empty(len(TRIS), [("n", order + cnt_t), ("i", order + "i4", (3,)), ("fl", "u1")])
            frec["n"], frec["i"], frec["fl"] = 3, TRIS, 1
            f.write(frec.tobytes())
        f.write(np.array([0, 1], order + "i4").tobytes())


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian", "binary_big_endian"])
@pytest.mark.parametrize("xyz_type", ["float", "double", "int"])
@pytest.mark.parametrize("count_type", ["uchar", "ushort", "int"])
def test_ply_readers_round_trip(tmp_path, fmt, xyz_type, count_type):
    from rade_gs_b200 import ply_io
    p = str(tmp_path / "m.ply")
    _write(p, fmt, xyz_type, count_type, ascii_=fmt == "ascii")
    want = PTS.astype({"float": np.float32, "double": np.float64, "int": np.int32}[xyz_type]).astype(np.float64)
    v, f = ply_io.load_triangle_mesh_ply(p)
    assert v.dtype == np.float64 and np.array_equal(v, want)
    assert f.dtype == np.int64 and np.array_equal(f, TRIS)
    assert np.array_equal(ply_io.load_point_cloud_ply(p), want)
    _write(p, fmt, xyz_type, count_type, with_faces=False, ascii_=fmt == "ascii")
    v, f = ply_io.load_triangle_mesh_ply(p)
    assert np.array_equal(v, want) and f.shape == (0, 3)


def test_ply_reader_rejects_polygons(tmp_path):
    from rade_gs_b200 import ply_io
    p = str(tmp_path / "quad.ply")
    hdr = "ply\nformat ascii 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\nelement face 1\nproperty list uchar int vertex_indices\nend_header\n"
    with open(p, "w") as f:
        f.write(hdr + "0 0 0\n1 0 0\n1 1 0\n0 1 0\n4 0 1 2 3\n")
    with pytest.raises(ValueError, match="triangle"):
        ply_io.load_triangle_mesh_ply(p)


def test_save_point_cloud_ply_layout(tmp_path):
    from rade_gs_b200 import ply_io
    p = str(tmp_path / "vis.ply")
    colors = np.array([[1.0, 0.5, 0.0], [0.2, 1.0, 0.998], [0.0, 0.0, 1.0]])
    ply_io.save_point_cloud_ply(p, PTS, colors)
    raw = open(p, "rb").read()
    body = raw[raw.index(b"end_header\n") + len(b"end_header\n"):]
    rec = np.frombuffer(body, [("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"]], 1), PTS)
    assert rec["r"].tolist() == [255, 51, 0] and rec["g"].tolist() == [128, 255, 0] and rec["b"].tolist() == [0, 254, 255]
    assert np.array_equal(ply_io.load_point_cloud_ply(p), PTS)


def test_dtu_eval_imports_no_open3d_trimesh_skimage_or_sklearn():
    pkg = os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200")
    for f in ("dtu_eval.py", "ply_io.py"):
        text = open(os.path.join(pkg, f)).read()
        for mod in ("open3d", "trimesh", "skimage", "sklearn"):
            assert f"import {mod}" not in text and f"from {mod}" not in text, (f, mod)
    code = ("import sys; sys.path.insert(0, %r); from rade_gs_b200 import dtu_eval, ply_io; "
            "print(sorted(m for m in sys.modules if m.split('.')[0] in ('open3d', 'trimesh', 'skimage', 'sklearn')))") % os.path.join(ROOT, "rade-gs_b200")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
    assert out == "[]"
