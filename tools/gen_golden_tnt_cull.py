"""Fixtures of the Tanks and Temples mesh cull, made by the reference's own code on the CPU: tests/golden/tnt_cull/*.npz.

Runs the UNMODIFIED ``eval_tnt/cull_mesh.py`` from the reference checkout (beside the repository, or $RADE_GS_REFERENCE,
or --reference) with in-process stand-ins:

* ``pyrender``: its renderer returns the depth of tests/tnt_cull_model.py (the header's contract) under pyrender's
  documented camera, which looks down -z: the scene pose ``c2w`` is the OpenCV pose ``c2w @ diag(1, -1, -1, 1)``;
* ``trimesh``: ``load`` (through ply_io; the meshes here have no duplicate vertices or degenerate faces, so
  ``process=True`` and ``merge_vertices`` change nothing, and the stand-in checks that), ``update_faces``,
  ``remove_unreferenced_vertices`` (referenced vertices kept in order, faces renumbered) and ``export`` (recorded);
* import-only ``open3d``, and ``cv2`` when it is absent.

The small cases construct ``Mesher`` and set ``mesher.device = "cpu"`` after construction, then call ``cull_mesh``; the
mask ``point_masks`` returns is recorded by a profile hook and the depth maps are stored.  The last case runs the script's ``__main__``
through ``runpy`` at 1920x1080 with a ``.log`` and a 3x4 ``.npy`` trajectory; there ``.to("cuda:0")`` means the CPU for
the run.  It stores the masks, the culled mesh and the SHA-256 of every depth map.  Archives are byte-reproducible.

Usage:  python tools/gen_golden_tnt_cull.py [--reference /path/to/RaDe-GS] [--out DIR]
"""
from __future__ import annotations

import argparse
import contextlib
import hashlib
import io
import os
import runpy
import sys
import tempfile
import types
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tnt_cull_model as M  # noqa: E402
from rade_gs_b200 import ply_io  # noqa: E402

FLIP = np.diag([1.0, -1.0, -1.0, 1.0])
_REC = {"depth": [], "export": None, "mask": None}


# ---- stand-ins -------------------------------------------------------------------------------------------------------------

class _Trimesh:
    def __init__(self, vertices, faces):
        self.vertices = np.asarray(vertices, np.float64)
        self.faces = np.asarray(faces, np.int64).reshape(-1, 3)

    def merge_vertices(self):
        assert len(np.unique(self.vertices, axis=0)) == len(self.vertices), "the fixtures' meshes have no duplicate vertices"

    def update_faces(self, mask):
        self.faces = self.faces[np.asarray(mask)]

    def remove_unreferenced_vertices(self):
        used = np.zeros(len(self.vertices), bool)
        used[self.faces.reshape(-1)] = True
        new = np.cumsum(used) - 1
        self.faces = new[self.faces]
        self.vertices = self.vertices[used]

    def export(self, path):
        _REC["export"] = (path, self.vertices.copy(), self.faces.copy())


def _trimesh_module():
    m = types.ModuleType("trimesh")

    def load(path, process=True):
        v, f = ply_io.load_triangle_mesh_ply(path)
        a = np.sort(v[f], axis=1)
        assert ((a[:, 0] != a[:, 1]).any(1) & (a[:, 1] != a[:, 2]).any(1)).all(), "no degenerate faces: process=True would drop them"
        return _Trimesh(v, f)

    m.load = load
    m.Trimesh = _Trimesh
    return m


def _pyrender_module():
    m = types.ModuleType("pyrender")

    class Scene:
        def __init__(self):
            self.mesh, self.pose = None, {}

        def add(self, mesh):
            self.mesh = mesh

        def add_node(self, node):
            self.pose[id(node)] = node.matrix

        def set_pose(self, node, pose):
            self.pose[id(node)] = np.asarray(pose)
            self.camera_node = node

    class Mesh:
        @staticmethod
        def from_trimesh(mesh):
            return mesh

    class IntrinsicsCamera:
        def __init__(self, fx, fy, cx, cy, znear=0.05, zfar=None):
            self.fx, self.fy, self.cx, self.cy, self.znear, self.zfar = fx, fy, cx, cy, znear, zfar

    class Node:
        def __init__(self, camera=None, matrix=None):
            self.camera, self.matrix = camera, matrix

    class OffscreenRenderer:
        def __init__(self, viewport_width, viewport_height):
            self.W, self.H = viewport_width, viewport_height

        def render(self, scene, flags):
            node = scene.camera_node
            cam = node.camera
            gl_pose = np.asarray(scene.pose[id(node)], np.float64)     # pyrender: the camera looks down -z of this pose
            m = M.w2c_rows(gl_pose @ FLIP)[0]
            d = M.mesh_depth(scene.mesh.vertices, scene.mesh.faces, m, cam.fx, cam.fy, cam.cx, cam.cy, self.H, self.W, cam.znear, cam.zfar)
            _REC["depth"].append(d)
            return d

        def delete(self):
            pass

    class RenderFlags:
        OFFSCREEN, DEPTH_ONLY, SKIP_CULL_FACES = 1, 2, 4

    for k, v in dict(Scene=Scene, Mesh=Mesh, IntrinsicsCamera=IntrinsicsCamera, Node=Node, OffscreenRenderer=OffscreenRenderer,
                     RenderFlags=RenderFlags).items():
        setattr(m, k, v)
    return m


@contextlib.contextmanager
def reference_env(reference):
    mods = {"pyrender": _pyrender_module(), "trimesh": _trimesh_module(), "open3d": types.ModuleType("open3d")}
    try:
        import cv2  # noqa: F401
    except ImportError:
        mods["cv2"] = types.ModuleType("cv2")
    saved = {k: sys.modules.get(k) for k in list(mods) + ["cull_mesh", "help_func"]}
    sys.modules.update(mods)
    sys.path.insert(0, os.path.join(reference, "eval_tnt"))
    try:
        yield
    finally:
        sys.path.remove(os.path.join(reference, "eval_tnt"))
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


@contextlib.contextmanager
def record_point_masks():
    """Records the mask Mesher.point_masks returns (a profile hook on its return; the source is not touched)."""
    def hook(frame, event, arg):
        if event == "return" and frame.f_code.co_name == "point_masks" and frame.f_code.co_filename.endswith("cull_mesh.py"):
            _REC["mask"] = arg[0]

    sys.setprofile(hook)
    try:
        yield
    finally:
        sys.setprofile(None)


@contextlib.contextmanager
def cuda_means_cpu():
    to = torch.Tensor.to

    def to_cpu(self, *a, **k):
        a = tuple("cpu" if isinstance(x, str) and x.startswith("cuda") else x for x in a)
        return to(self, *a, **k)

    torch.Tensor.to = to_cpu
    try:
        yield
    finally:
        torch.Tensor.to = to


# ---- scenes ------------------------------------------------------------------------------------------------------------------

def grid(origin, du, dv, n):
    """An (n+1)^2-vertex grid of 2 n^2 triangles spanning origin + [0,1] du + [0,1] dv."""
    s = np.linspace(0.0, 1.0, n + 1)
    a, b = np.meshgrid(s, s, indexing="ij")
    v = origin + a.reshape(-1, 1) * du + b.reshape(-1, 1) * dv
    i = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    q = np.stack([i[:-1, :-1], i[1:, :-1], i[1:, 1:], i[:-1, 1:]], -1).reshape(-1, 4)
    return v, np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])


def box(lo, hi, n, inset=0.0):
    """Six separate grids (no shared vertices: each wall is inset by `inset` at its border)."""
    lo, hi = np.asarray(lo, float), np.asarray(hi, float)
    parts = []
    for ax in range(3):
        for side in (lo[ax], hi[ax]):
            u, w = [k for k in range(3) if k != ax]
            o = lo.copy()
            o[ax] = side
            o[u] += inset
            o[w] += inset
            du, dv = np.zeros(3), np.zeros(3)
            du[u] = hi[u] - lo[u] - 2 * inset
            dv[w] = hi[w] - lo[w] - 2 * inset
            parts.append(grid(o, du, dv, n))
    return parts


def merge(parts):
    vs, fs, off = [], [], 0
    for v, f in parts:
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    return np.concatenate(vs).astype(np.float32).astype(np.float64), np.concatenate(fs).astype(np.int64)


def look_at(eye, target, up=(0.0, 1.0, 0.0)):
    """OpenCV camera-to-world: +z towards the target, +y down."""
    z = np.asarray(target, float) - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, -np.asarray(up, float))
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, eye
    return T


def scene(seed, n_obj, n_wall):
    """A subdivided box around the origin in front of the cameras, an occluder panel before part of it, and a wall behind
    the cameras that covers part of what pyrender's backward-looking camera sees."""
    rng = np.random.default_rng(seed)
    parts = box([-0.5, -0.5, -0.5], [0.5, 0.5, 0.5], n_obj, inset=0.005)
    parts.append(grid(np.array([-0.3, -0.6, -1.2]), np.array([0.5, 0.0, 0.0]), np.array([0.0, 0.7, 0.0]), 3))
    parts.append(grid(np.array([-1.2, -0.9, -4.6]), np.array([2.2, 0.0, 0.0]), np.array([0.0, 1.6, 0.0]), n_wall))
    v, f = merge(parts)
    return v, f, rng


def cameras(rng, n):
    """On an arc 3 units from the origin, within 35 degrees of -z, looking at the origin (OpenCV poses)."""
    out = []
    for _ in range(n):
        a, e = rng.uniform(-0.6, 0.6), rng.uniform(-0.3, 0.3)
        eye = 3.0 * np.array([np.sin(a) * np.cos(e), np.sin(e), -np.cos(a) * np.cos(e)])
        out.append(look_at(eye, rng.uniform(-0.1, 0.1, 3)))
    return np.stack(out).astype(np.float32).astype(np.float64)


SMALL = [  # name, seed, views, H, W, fx, fy, cx, cy, box / wall subdivisions
    ("small_a", 41, 20, 60, 80, 58.3, 61.1, 40.27, 29.61, 10, 6),
    ("small_b", 42, 36, 48, 64, 45.0, 44.0, 31.5, 23.5, 12, 8),
    ("small_c", 43, 60, 72, 96, 80.9, 79.4, 47.83, 36.12, 8, 4),
]
HD = dict(H=1080, W=1920, fx=1163.8678928442187, fy=1172.793101201448, cx=962.3120628412543, cy=542.0667209577691)


def save_npz(path, **arrays):
    """np.savez_compressed with fixed timestamps, so the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


def run_small(reference, name, seed, views, H, W, fx, fy, cx, cy, n_wall, n_box):
    v, f, rng = scene(seed, n_wall, n_box)
    c2w = cameras(rng, views)
    _REC["depth"].clear()
    with reference_env(reference):
        cm = __import__("cull_mesh")
        mesher = cm.Mesher(H, W, fx, fy, cx, cy, 20.0, points_batch_size=5e5)
        mesher.device = "cpu"
        with record_point_masks(), contextlib.redirect_stdout(io.StringIO()):
            cull, _ = mesher.cull_mesh(_Trimesh(v, f), [torch.from_numpy(c).float() for c in c2w])
    return dict(vertices=v, faces=f, c2w=c2w, camera=np.array([H, W, fx, fy, cx, cy, 20.0]), depths=np.stack(_REC["depth"]),
                mask=np.asarray(_REC["mask"], bool), cull_vertices=cull.vertices, cull_faces=cull.faces)


def run_main(reference):
    v, f, rng = scene(44, 12, 4)
    c2w = cameras(rng, 22)
    out = {"vertices": v, "faces": f, "c2w": c2w}
    with tempfile.TemporaryDirectory() as tmp:
        ply = os.path.join(tmp, "mesh.ply")
        ply_io.save_triangle_mesh_ply(ply, v, f)
        log = os.path.join(tmp, "traj.log")
        with open(log, "w") as fh:
            for k, c in enumerate(c2w):
                fh.write(f"{k} {k} 0\n")
                for r in c:
                    fh.write(" ".join(repr(float(x)) for x in r) + "\n")
        npy = os.path.join(tmp, "traj.npy")
        np.save(npy, c2w[:, :3, :])
        for tag, traj in (("log", log), ("npy", npy)):
            _REC["depth"].clear()
            saved_argv = sys.argv
            sys.argv = ["cull_mesh.py", "--traj-path", traj, "--ply-path", ply]
            try:
                with reference_env(reference), cuda_means_cpu(), record_point_masks(), contextlib.redirect_stdout(io.StringIO()):
                    runpy.run_path(os.path.join(reference, "eval_tnt", "cull_mesh.py"), run_name="__main__")
            finally:
                sys.argv = saved_argv
            path, cv, cf = _REC["export"]
            assert os.path.basename(path) == "mesh_cull.ply"
            out[f"{tag}_mask"] = np.asarray(_REC["mask"], bool)
            out[f"{tag}_cull_vertices"], out[f"{tag}_cull_faces"] = cv, cf
            out[f"{tag}_depth_sha256"] = np.array([hashlib.sha256(np.ascontiguousarray(d, np.float32).tobytes()).hexdigest() for d in _REC["depth"]])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference")))
    ap.add_argument("--out", default=os.path.join(ROOT, "golden_out", "tnt_cull"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    for name, *args in SMALL:
        r = run_small(a.reference, name, *args)
        save_npz(os.path.join(a.out, name + ".npz"), **r)
        print(name, "vertices", len(r["vertices"]), "faces", len(r["faces"]), "views", len(r["c2w"]), "valid", int(r["mask"].sum()),
              "kept faces", len(r["cull_faces"]), flush=True)
    r = run_main(a.reference)
    save_npz(os.path.join(a.out, "main_hd.npz"), **r)
    print("main_hd vertices", len(r["vertices"]), "valid", int(r["log_mask"].sum()), int(r["npy_mask"].sum()), "kept faces",
          len(r["log_cull_faces"]), len(r["npy_cull_faces"]), flush=True)


if __name__ == "__main__":
    main()
