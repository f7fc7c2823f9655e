"""Fixture of the bounded TSDF and the image export, made by the reference's own code on the CPU:
tests/golden/bounded/bounded.npz.

Imports the UNMODIFIED ``utils/mesh_utils.py`` and ``utils/render_utils.py`` from the reference checkout (beside the
repository, or $RADE_GS_REFERENCE, or --reference) with in-process stand-ins for ``open3d``, ``trimesh``, ``mediapy`` and
``matplotlib``; ``.cuda()`` means the CPU for the run.  Three things of the reference's class do not run as shipped, and
the script works around each without editing it:
  * ``reconstruction`` calls ``render`` without ``kernel_size`` and reads ``middepth``: the extractor's ``rgbmaps``,
    ``depthmaps``, ``normals``, ``depth_normals`` and ``viewpoint_stack`` are set to analytic views (tests/tsdf_scenes.py);
  * ``extract_mesh_bounded`` reads ``gt_alpha_mask``, which RaDe-GS's Camera does not have: the stand-in cameras carry it;
  * ``export_image`` calls ``save_img_u8`` / ``save_img_f32`` without importing them: render_utils' functions are put
    into the module.

``export_image`` runs first (the order of the reference's render scripts), then ``extract_mesh_bounded`` with its
defaults.  The ``open3d`` stand-in records what the reference hands to Open3D: the volume's arguments, and per view the
uint8 colour image, the float depth image (masked), depth_trunc / depth_scale / convert_rgb_to_intensity, the intrinsic
(width, height, fx, fy, cx, cy) and the extrinsic.  ``PIL.Image.fromarray`` is wrapped to record the array behind every
file the export writes.  The rendered colours include values above 1 and below 0, infinities and NaNs, so the uint8 wrap
of the integration path and the clip of the export are both pinned.

Usage:  python tools/gen_golden_bounded.py [--reference /path/to/RaDe-GS] [--out DIR]
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tsdf_scenes as ts  # noqa: E402

W, H, V = 40, 32, 3
_REC = {"volume": [], "views": [], "files": {}}


class _Image:
    def __init__(self, a):
        self.array = np.array(a, copy=True)


class _Volume:
    def __init__(self, voxel_length, sdf_trunc, color_type):
        _REC["volume"].append((float(voxel_length), float(sdf_trunc), color_type))

    def integrate(self, rgbd, intrinsic, extrinsic):
        rgbd["intrinsic"] = intrinsic.args
        rgbd["extrinsic"] = np.asarray(extrinsic, np.float64)
        _REC["views"].append(rgbd)

    def extract_triangle_mesh(self):
        return types.SimpleNamespace()


class _Intrinsic:
    def __init__(self, width, height, cx, cy, fx, fy):
        self.args = np.array([width, height, fx, fy, cx, cy], np.float64)


def _rgbd(color, depth, depth_trunc, convert_rgb_to_intensity, depth_scale):
    return {"color": color.array, "depth": depth.array, "depth_trunc": float(depth_trunc), "depth_scale": float(depth_scale),
            "convert_rgb_to_intensity": bool(convert_rgb_to_intensity)}


def install_stubs(ref):
    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(Image=_Image, RGBDImage=types.SimpleNamespace(create_from_color_and_depth=_rgbd))
    o3d.camera = types.SimpleNamespace(PinholeCameraIntrinsic=_Intrinsic, PinholeCameraParameters=types.SimpleNamespace)
    o3d.pipelines = types.SimpleNamespace(integration=types.SimpleNamespace(ScalableTSDFVolume=_Volume,
                                                                            TSDFVolumeColorType=types.SimpleNamespace(RGB8="RGB8")))
    sys.modules["open3d"] = o3d
    sys.modules["trimesh"] = types.ModuleType("trimesh")
    sys.modules["mediapy"] = types.ModuleType("mediapy")
    mpl = types.ModuleType("matplotlib")
    mpl.cm = types.SimpleNamespace()
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.cm"] = mpl.cm
    sys.path[:0] = [ref]
    torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
    orig = torch.tensor

    def on_cpu(*a, **k):
        if str(k.get("device", "")).startswith("cuda"):
            k["device"] = "cpu"
        return orig(*a, **k)
    torch.tensor = on_cpu
    from PIL import Image
    fromarray = Image.fromarray

    def recording(a, *args, **kw):
        _REC["last"] = np.array(a, copy=True)
        return fromarray(a, *args, **kw)
    Image.fromarray = recording
    open_ = open

    def opening(path, mode="r", *a, **k):
        f = open_(path, mode, *a, **k)
        if "w" in mode and str(path).endswith((".png", ".tiff")):
            _REC["pending"] = os.path.relpath(path, _REC["dir"])
        return f
    import builtins
    builtins.open = opening


def scene():
    """V views of a sphere in front of a plane; colours pushed outside [0, 1] with a few NaNs and infinities."""
    g = np.random.default_rng(11)
    fov = 55.0
    K = ts.intrinsic(W, H, fov)
    cams, rgb, depth, mask, gt, normals = [], [], [], [], [], []
    for k in range(V):
        eye = (0.15 * k - 0.15, 0.05 * k, -1.1)
        E = ts.look_at(eye, (0.0, 0.0, 0.0))
        d, c = ts.render(K, E, H, W, planes=[((0.1, 0.0, 1.0), 0.45)], spheres=[((0.0, 0.0, 0.0), 0.25)])
        c = (c * 1.6 - 0.3).astype(np.float32)                      # about 1/3 of the values leave [0, 1]
        c.reshape(-1)[g.choice(c.size, 6, replace=False)] = [np.nan, np.nan, np.inf, -np.inf, 3.0e9, -1.0e10]
        d[g.random(d.shape) < 0.03] = np.nan
        rgb.append(np.transpose(c, (2, 0, 1)))
        depth.append(d[None] * np.float32(2.0 if k == 2 else 1.0))   # the last view lies partly beyond depth_trunc = 3
        mask.append((g.random((1, H, W)) > 0.2).astype(np.float32))
        gt.append(g.uniform(-0.2, 1.2, (3, H, W)).astype(np.float32))
        n = g.normal(size=(3, H, W)).astype(np.float32)
        n[0, 0, :3] = [np.nan, np.inf, -np.inf]
        normals.append(n / np.linalg.norm(n, axis=0, keepdims=True))
        f = K[0, 0]
        cams.append(dict(E=E, FoVx=fov * math.pi / 180, FoVy=2 * math.atan(H / (2 * f))))
    return cams, *(np.stack(a).astype(np.float32) for a in (rgb, depth, mask, gt, normals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference"))
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "bounded"))
    args = ap.parse_args()
    install_stubs(args.reference)
    from PIL import Image
    from utils import mesh_utils, render_utils

    cams, rgb, depth, mask, gt, normals = scene()
    views = [types.SimpleNamespace(image_width=W, image_height=H, FoVx=c["FoVx"], FoVy=c["FoVy"],
                                   world_view_transform=torch.from_numpy(c["E"].T.astype(np.float32)),
                                   gt_alpha_mask=torch.from_numpy(mask[i]), gt_mask=torch.from_numpy(mask[i]),
                                   original_image=torch.from_numpy(gt[i])) for i, c in enumerate(cams)]
    ex = mesh_utils.GaussianExtractor(types.SimpleNamespace(), render=lambda *a, **k: None, pipe=None)
    ex.viewpoint_stack = views
    ex.rgbmaps = torch.from_numpy(rgb.copy())
    ex.depthmaps = torch.from_numpy(depth.copy())
    ex.normals = [torch.from_numpy(n.copy()) for n in normals]
    ex.depth_normals = torch.zeros_like(ex.rgbmaps)
    mesh_utils.save_img_u8, mesh_utils.save_img_f32 = render_utils.save_img_u8, render_utils.save_img_f32

    saved = Image.Image.save

    def save(self, fp, *a, **k):
        _REC["files"][_REC.pop("pending")] = _REC.pop("last")
        return saved(self, fp, *a, **k)
    Image.Image.save = save
    with tempfile.TemporaryDirectory() as tmp:
        _REC["dir"] = tmp
        ex.export_image(tmp)
    ex.extract_mesh_bounded()
    (vl, st, ct), = _REC["volume"]
    assert ct == "RGB8" and len(_REC["views"]) == V
    rv = _REC["views"]
    files = _REC["files"]
    out = {f"file:{k}": v for k, v in sorted(files.items()) if "depth_normal" not in k}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "bounded.npz")
    np.savez_compressed(
        path, rgb=rgb, depth=depth, mask=mask, gt=gt, normals=normals,
        world_view=np.stack([c["E"].T.astype(np.float32) for c in cams]), fovx=np.array([c["FoVx"] for c in cams]),
        fovy=np.array([c["FoVy"] for c in cams]), size=np.array([W, H]),
        voxel_length=np.float64(vl), sdf_trunc=np.float64(st),
        rec_color=np.stack([r["color"] for r in rv]), rec_depth=np.stack([r["depth"] for r in rv]),
        rec_depth_trunc=np.array([r["depth_trunc"] for r in rv]), rec_depth_scale=np.array([r["depth_scale"] for r in rv]),
        rec_intensity=np.array([r["convert_rgb_to_intensity"] for r in rv]),
        rec_intrinsic=np.stack([r["intrinsic"] for r in rv]), rec_extrinsic=np.stack([r["extrinsic"] for r in rv]), **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.0f} KB): {V} views {W}x{H}, volume ({vl}, {st}), {len(out)} exported files")


if __name__ == "__main__":
    main()
