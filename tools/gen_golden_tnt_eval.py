"""Fixtures of the Tanks and Temples evaluation, made by the reference's own control flow on the CPU:
tests/golden/tnt_eval/*.npz.

Runs the UNMODIFIED ``eval_tnt/run.py::run_evaluation`` (loaded with runpy, its siblings registration.py, evaluation.py,
trajectory_io.py and config.py imported as they are) on seeded synthetic scenes.  Each dataset directory is named after a
``scenes_tau_dict`` scene, so the reference picks tau itself.  In-process stand-ins replace what is not installed:

* ``open3d``: point clouds whose transform, crop, voxel_down_sample, uniform_down_sample, compute_point_cloud_distance,
  registration_icp and registration_ransac_based_on_correspondence are the numpy model of the header contracts
  (tests/tnt_eval_f64.py, seeded RANSAC); read_point_cloud returns the registered arrays and write_point_cloud is captured;
* ``trimesh.load_mesh``: the registered vertices and faces;
* ``matplotlib.pyplot.get_cmap``: matplotlib's lookup of the hot_r table derived in rade_gs_b200.tnt_eval;
* ``plot.plot_graph``: captured (the figure is out of scope).

This pins everything the reference itself decides: the stage order and thresholds, the uniform-downsample rule,
``read_trajectory``, ``get_f1_score_histo2`` and the files it writes.  It cannot pin Open3D's internals (its crop boundary
rule, voxel output order, ICP sums, RANSAC sampling): those are the model's, i.e. the header's.

Usage:  python tools/gen_golden_tnt_eval.py [--reference /path/to/RaDe-GS] [--out DIR]
Copy the files to tests/golden/tnt_eval/.  Writing is deterministic: the archives carry fixed timestamps.
"""
from __future__ import annotations

import argparse
import copy
import io
import json
import os
import runpy
import sys
import tempfile
import types
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "rade-gs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tnt_eval_f64 as model  # noqa: E402


# ---- scenes ---------------------------------------------------------------------------------------------------------------

def _rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _similarity(rng, scale, shift):
    T = np.eye(4)
    T[:3, :3] = scale * _rotation(rng)
    T[:3, 3] = rng.normal(0, shift, 3)
    return T


def _height(x, y):
    return 0.06 * np.sin(3.0 * x) * np.cos(2.0 * y) + 0.03 * np.cos(5.0 * x + 1.0)


def make_scene(seed, tau, extent, n_gt=20000, grid=72, n_cams=60):
    """A bumpy surface in the GT frame; the mesh and the estimated trajectory live in a frame related to it by an unknown
    similarity (scale != 1); the COLMAP trajectory in a frame related by gt_trans."""
    rng = np.random.default_rng(seed)
    e = extent
    xy = rng.uniform(-e, e, (n_gt, 2))
    gt = np.column_stack([xy, _height(xy[:, 0], xy[:, 1])])
    gt = np.concatenate([gt, rng.uniform(-3 * e, 3 * e, (200, 3))])                 # clutter, mostly outside the crop
    xs = np.linspace(-0.9 * e, 0.9 * e, grid)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    verts = np.column_stack([X.ravel(), Y.ravel(), _height(X.ravel(), Y.ravel())]) + rng.normal(0, tau / 3, (grid * grid, 3))
    faces = []
    for i in range(grid - 1):
        for j in range(grid - 1):
            if (i - grid // 3) ** 2 + (j - grid // 2) ** 2 < (grid // 8) ** 2:
                continue                                                            # a hole: recall < 1
            a, b, c, d = i * grid + j, (i + 1) * grid + j, i * grid + j + 1, (i + 1) * grid + j + 1
            faces += [(a, b, c), (b, d, c)]
    faces = np.array(faces, np.int32)
    verts = np.concatenate([verts, rng.uniform(-2 * e, 2 * e, (100, 3))])          # floaters
    A = _similarity(rng, 1.7, 0.5)                                                  # estimated -> GT
    gt_trans = _similarity(rng, 1.0, 0.3)                                           # COLMAP -> GT
    ang = np.linspace(0, 2 * np.pi, n_cams, endpoint=False)
    centres = np.column_stack([2.2 * e * np.cos(ang), 2.2 * e * np.sin(ang), 0.8 * e + 0.2 * e * np.sin(3 * ang)]) + rng.normal(0, 0.02 * e, (n_cams, 3))
    Ainv, Ginv = np.linalg.inv(A), np.linalg.inv(gt_trans)

    def poses(T, c, noise):
        P = np.tile(np.eye(4), (len(c), 1, 1))
        P[:, :3, :3] = _rotation(rng)
        P[:, :3, 3] = model.transform(T, c) + rng.normal(0, noise, c.shape)
        return P
    gt_traj = poses(Ginv, centres, 0.0)
    traj = poses(Ainv, centres, 2e-4 * e)
    out = rng.choice(n_cams, n_cams // 10, replace=False)
    traj[out, :3, 3] += rng.normal(0, 1.0, (len(out), 3))                          # ~10 % outlier cameras
    verts = model.transform(Ainv, verts)
    poly = np.array([[-0.8, -0.8], [0.8, -0.8], [0.8, 0.8], [0.05, 0.15], [-0.8, 0.8], [-0.8, 0.1], [-0.5, 0.1], [-0.5, -0.2], [-0.8, -0.2]]) * e
    crop = {"class_name": "SelectionPolygonVolume", "orthogonal_axis": "Z", "axis_min": -0.3 * e, "axis_max": 0.3 * e, "version_major": 1, "version_minor": 0,
            "bounding_polygon": [[u, v, 0.0] for u, v in poly]}
    return dict(vertices=verts, faces=faces, gt=gt, gt_trans=gt_trans, traj=traj, gt_traj=gt_traj, crop=crop, planted=A)


def write_log(path, poses):
    with open(path, "w") as f:
        for k, P in enumerate(poses):
            f.write(f"{k} {k} 0\n")
            f.write("\n".join(" ".join("{0:.12f}".format(x) for x in row) for row in P))
            f.write("\n")


# ---- stand-ins ----------------------------------------------------------------------------------------------------------------

class _Cloud:
    def __init__(self, points=None):
        self.points = [] if points is None else np.asarray(points, np.float64).reshape(-1, 3)
        self.colors = None

    def _p(self):
        return np.asarray(self.points, np.float64).reshape(-1, 3)

    def transform(self, T):
        self.points = model.transform(np.asarray(T, np.float64), self._p())
        return self

    def voxel_down_sample(self, voxel):
        return _Cloud(model.voxel_down_sample(self._p(), voxel)[0])

    def uniform_down_sample(self, k):
        return _Cloud(self._p()[::k])

    def estimate_normals(self, search_param=None):
        return True

    def compute_point_cloud_distance(self, other):
        return model.nearest(other._p(), self._p())[0]


def _open3d_standin(registry, written, record, seed):
    o3d = types.ModuleType("open3d")

    class _Volume:
        def __init__(self, d):
            axis = "XYZ".index(d["orthogonal_axis"].upper())
            poly = np.asarray(d["bounding_polygon"], np.float64)[:, [a for a in range(3) if a != axis]]
            self.v = (axis, float(d["axis_min"]), float(d["axis_max"]), poly)

        def crop_point_cloud(self, pcd):
            return _Cloud(model.crop(pcd._p(), self.v)[0])

    def read_selection_polygon_volume(path):
        with open(path) as f:
            return _Volume(json.load(f))

    class _Result:
        pass

    def ransac(source, target, corres, max_dist, estimation, ransac_n, criteria=None):
        c = np.asarray(corres)
        T, n_in, rmse, k = model.ransac(source._p()[c[:, 0]], target._p()[c[:, 1]], seed, criteria.max_iteration, max_dist, ransac_n)
        record["ransac"] = dict(T=T, inliers=n_in, rmse=rmse, hypothesis=k, max_distance=max_dist, ransac_n=ransac_n, iterations=criteria.max_iteration,
                                with_scaling=estimation.with_scaling)
        r = _Result()
        r.transformation = T
        return r

    def icp(source, target, threshold, init, estimation, criteria):
        s = source._p() if np.array_equal(init, np.eye(4)) else model.transform(init, source._p())
        T, fit, rmse, it, hist, counts = model.icp(s, target._p(), threshold, criteria.max_iteration, criteria.relative_fitness, criteria.relative_rmse)
        record.setdefault("icp", []).append(dict(T=T, fitness=fit, rmse=rmse, iterations=it, threshold=threshold, source_n=len(s), target_n=len(target._p()),
                                                 with_scaling=estimation.with_scaling))
        r = _Result()
        r.transformation, r.fitness, r.inlier_rmse = T, fit, rmse
        return r

    def write_point_cloud(path, pcd):
        written[os.path.basename(path)] = (pcd._p().copy(), np.asarray(pcd.colors, np.float64).copy())
        return True

    class _RansacCriteria:
        def __init__(self, max_iteration=100000, confidence=0.999):
            self.max_iteration, self.confidence = max_iteration, confidence

    class _ICPCriteria:
        def __init__(self, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30):
            self.relative_fitness, self.relative_rmse, self.max_iteration = relative_fitness, relative_rmse, max_iteration

    class _P2P:
        def __init__(self, with_scaling=False):
            self.with_scaling = with_scaling

    o3d.geometry = types.SimpleNamespace(PointCloud=_Cloud, KDTreeSearchParamKNN=lambda knn=30: None)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64), Vector2iVector=lambda a: np.asarray(a),
                                        set_verbosity_level=lambda level: None, VerbosityLevel=types.SimpleNamespace(Debug=0))
    o3d.io = types.SimpleNamespace(read_point_cloud=lambda path: _Cloud(registry[os.path.basename(path)].copy()), write_point_cloud=write_point_cloud)
    o3d.visualization = types.SimpleNamespace(read_selection_polygon_volume=read_selection_polygon_volume, draw_geometries=lambda g: None)
    o3d.pipelines = types.SimpleNamespace(registration=types.SimpleNamespace(
        RANSACConvergenceCriteria=_RansacCriteria, ICPConvergenceCriteria=_ICPCriteria, TransformationEstimationPointToPoint=_P2P,
        registration_ransac_based_on_correspondence=ransac, registration_icp=icp))
    return o3d


def _matplotlib_standin():
    from rade_gs_b200.tnt_eval import _hot_r_table
    lut = _hot_r_table()

    def get_cmap(name):
        assert name == "hot_r", name

        def cmap(x):   # Colormap.__call__ on floats: index floor(x * N), N -> N - 1, RGBA
            xa = np.array(x, np.float64) * 256
            xa[xa == 256] = 255
            xa = np.clip(xa, -1, 256).astype(int)
            return np.concatenate([lut[xa], np.ones(xa.shape + (1,))], axis=-1)
        return cmap
    mpl = types.ModuleType("matplotlib")
    plt = types.ModuleType("matplotlib.pyplot")
    plt.get_cmap = get_cmap
    mpl.pyplot = plt
    return mpl, plt


def run_reference(reference, sc, scene, seed, traj_ext):
    registry, written, record, plotted = {}, {}, {}, {}
    tnt_dir = os.path.join(reference, "eval_tnt")
    mods = ("open3d", "trimesh", "matplotlib", "matplotlib.pyplot", "plot", "config", "registration", "evaluation", "trajectory_io", "util")
    saved = {m: sys.modules.get(m) for m in mods}
    with tempfile.TemporaryDirectory() as d:
        ds = os.path.join(d, scene)
        os.makedirs(ds)
        out = os.path.join(d, "out")
        with open(os.path.join(ds, scene + ".json"), "w") as f:
            json.dump(sc["crop"], f)
        np.savetxt(os.path.join(ds, scene + "_trans.txt"), sc["gt_trans"])
        write_log(os.path.join(ds, scene + "_COLMAP_SfM.log"), sc["gt_traj"])
        traj_path = os.path.join(d, "traj" + traj_ext)
        if traj_ext == ".npy":
            np.save(traj_path, sc["traj"])
        else:
            write_log(traj_path, sc["traj"])
        registry[scene + ".ply"] = sc["gt"]
        registry["recon.ply"] = sc["vertices"]
        sys.modules["open3d"] = _open3d_standin(registry, written, record, seed)
        sys.modules["trimesh"] = types.SimpleNamespace(load_mesh=lambda path: types.SimpleNamespace(vertices=sc["vertices"].copy(), faces=sc["faces"].copy()))
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = _matplotlib_standin()
        sys.modules["plot"] = types.SimpleNamespace(plot_graph=lambda *a, **k: plotted.update(args=a))
        for m in ("config", "registration", "evaluation", "trajectory_io", "util"):
            sys.modules.pop(m, None)
        sys.path.insert(0, tnt_dir)
        try:
            g = runpy.run_path(os.path.join(tnt_dir, "run.py"), run_name="tnt_run")
            g["run_evaluation"](dataset_dir=ds, traj_path=traj_path, ply_path=os.path.join(d, "recon.ply"), out_dir=out, view_crop=False)
            texts = {f: open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))}
        finally:
            sys.path.remove(tnt_dir)
            for m, v in saved.items():
                if v is None:
                    sys.modules.pop(m, None)
                else:
                    sys.modules[m] = v
    return record, written, plotted, texts


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


SCENES = [  # fixture name, scene (sets tau), seed, scene extent, trajectory format
    ("barn", "Barn", 31, 0.6, ".log"),
    ("caterpillar", "Caterpillar", 32, 0.3, ".npy"),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE", os.path.join(os.path.dirname(ROOT), "reference")))
    ap.add_argument("--out", default=os.path.join(ROOT, "golden_out"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    for name, scene, seed, extent, ext in SCENES:
        tau = {"Barn": 0.01, "Caterpillar": 0.005}[scene]
        sc = make_scene(seed, tau, extent)
        record, written, plotted, texts = run_reference(a.reference, copy.deepcopy(sc), scene, seed, ext)
        icp = record["icp"]
        composed, T = [], record["ransac"]["T"]
        for r in icp:   # registration.py: reg.transformation = reg.transformation @ init_trans
            T = r["T"] @ T
            composed.append(T)
        prec_pts, _ = written[scene + ".precision.ply"]
        rec_pts, _ = written[scene + ".recall.ply"]
        args = plotted["args"]   # scene, fscore, tau, edges_source, cum_source, edges_target, cum_target, stretch, out
        prf = np.loadtxt(io.StringIO(texts[scene + ".prf_tau_plotstr.txt"]))
        save_npz(os.path.join(a.out, name + ".npz"),
                 scene=np.array(scene), seed=np.array(seed), tau=np.array(tau), traj_format=np.array(ext),
                 vertices=sc["vertices"], faces=sc["faces"], gt=sc["gt"], gt_trans=sc["gt_trans"], traj=sc["traj"], gt_traj=sc["gt_traj"],
                 crop_json=np.array(json.dumps(sc["crop"])), planted=sc["planted"],
                 alignment=record["ransac"]["T"], ransac_inliers=np.array(record["ransac"]["inliers"]),
                 stage_T=np.stack(composed), stage_fitness=np.array([r["fitness"] for r in icp]),
                 stage_rmse=np.array([r["rmse"] for r in icp]), stage_iterations=np.array([r["iterations"] for r in icp]),
                 stage_threshold=np.array([r["threshold"] for r in icp]), stage_sizes=np.array([[r["source_n"], r["target_n"]] for r in icp]),
                 prf=prf, edges_source=args[3], cum_source=args[4], edges_target=args[5], cum_target=args[6],
                 ply_sizes=np.array([len(prec_pts), len(rec_pts)]),
                 files=np.array(sorted(list(texts) + [scene + ".precision.ply", scene + ".recall.ply"])),
                 txt_names=np.array(sorted(texts)), txt_contents=np.array([texts[k] for k in sorted(texts)]))
        print(name, "alignment inliers", record["ransac"]["inliers"], "stages", [(r["iterations"], round(r["fitness"], 4)) for r in icp],
              "prf", prf[:3], flush=True)


if __name__ == "__main__":
    main()
