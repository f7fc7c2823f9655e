"""Generate tests/golden/fused_*.npz from the REFERENCE'S OWN Python functions (on CPU; the reference checkout beside the repository, or $RADE_GS_REFERENCE).

Pins the widened rows (SURVEY.md 8f-1, 8f-2, 8f-4) to the reference itself instead of to restatements:
  fused_losses.npz     utils/loss_utils.py:17-18 `l1_loss`, :35-63 `ssim`, and train.py:163's combination; values + autograd gradients
  fused_normals.npz    utils/graphics_utils.py:97-126 `depth_double_to_normal` / `point_double_to_normal` + train.py:143-156's
                       normal-consistency loss (the three-line expression around the reference function is restated here,
                       train.py has no importable function for it); values + gradients w.r.t. normal and both maps
  fused_model.npz      scene/gaussian_model.py:156-166 `get_scaling_n_opacity_with_3D_filter`, :125-126 `get_rotation` (+ autograd
                       gradients), :743-747 `add_densification_stats` + train.py:187-188's radius maximum, :179-232 `compute_3D_filter`
  fused_ply.npz        scene/gaussian_model.py:380-397 `save_ply` bytes (attribute list, transposes) and what :515-559 `load_ply`
                       reads back from them
The reference hard-codes `.cuda()` in a few places (graphics_utils.py:106,108, gaussian_model.py:65,68): this script runs it on
CPU by making `.cuda()` / `device="cuda"` mean the CPU for the duration of the run -- an environment shim, the reference files are imported as
they are.  plyfile / simple_knn / trimesh are not in this image: tests/ref_stubs/ provides import stand-ins (the PLY byte layout
pinned here is therefore "reference's writer code + our plyfile stand-in", stated in DESIGN.md).

    python tools/gen_golden_fused.py
"""
import math
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
sys.path[:0] = [os.path.join(ROOT, "tests", "ref_stubs"), REF]
torch.Tensor.cuda = lambda self, *a, **k: self            # noqa: E731  CPU run of code that says .cuda()
torch.nn.Module.cuda = lambda self, *a, **k: self         # noqa: E731
_torch_tensor = torch.tensor


def _tensor_on_cpu(*a, **k):                              # load_ply says torch.tensor(..., device="cuda")
    if str(k.get("device", "")).startswith("cuda"):
        k["device"] = "cpu"
    return _torch_tensor(*a, **k)


torch.tensor = _tensor_on_cpu

from utils.loss_utils import l1_loss, ssim                                         # noqa: E402
from utils.graphics_utils import depth_double_to_normal, point_double_to_normal   # noqa: E402
from scene.gaussian_model import GaussianModel                                    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
torch.manual_seed(0)
torch.set_num_threads(4)


def n(t):
    return t.detach().cpu().numpy().copy()          # a copy: several tensors are updated in place afterwards


def gen_losses():
    g = torch.Generator().manual_seed(101)
    H, W = 70, 93                                   # ragged: not a multiple of the kernels' 32x16 tiles
    gt = torch.rand(3, H, W, generator=g)
    img = (gt + 0.25 * torch.randn(3, H, W, generator=g)).clamp(0, 1.2)
    img[:, 10:20, 30:50] = gt[:, 10:20, 30:50]      # a region with |img - gt| = 0 (sign(0) in the L1 gradient)
    out = {"img": n(img), "gt": n(gt)}
    for name, fn in (("l1", lambda a: l1_loss(a, gt)), ("ssim", lambda a: ssim(a, gt)),
                     ("train163", lambda a: (1.0 - 0.2) * l1_loss(a, gt) + 0.2 * (1.0 - ssim(a, gt.unsqueeze(0))))):
        a = img.clone().requires_grad_(True)
        v = fn(a)
        v.backward()
        out[name], out["d_" + name] = n(v), n(a.grad)
        a64 = img.double().clone().requires_grad_(True)          # the same reference functions in fp64: the arbiter for tolerances
        gt64 = gt.double()
        v64 = {"l1": lambda: l1_loss(a64, gt64), "ssim": lambda: ssim(a64, gt64),
               "train163": lambda: 0.8 * l1_loss(a64, gt64) + 0.2 * (1.0 - ssim(a64, gt64.unsqueeze(0)))}[name]()
        v64.backward()
        out[name + "_f64"], out["d_" + name + "_f64"] = n(v64), n(a64.grad)
    np.savez_compressed(os.path.join(OUT, "fused_losses.npz"), **out)


def gen_normals():
    g = torch.Generator().manual_seed(202)
    H, W = 45, 61
    view = SimpleNamespace(image_width=W, image_height=H, FoVx=0.9, FoVy=2 * math.atan(H / W * math.tan(0.45)))
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    base = 3.0 + 0.02 * xx + 0.015 * yy + 0.3 * torch.sin(xx / 7.0) * torch.cos(yy / 5.0)
    d1 = (base + 0.01 * torch.randn(H, W, generator=g))[None]
    d2 = (base * 1.02 + 0.01 * torch.randn(H, W, generator=g))[None]
    nrm = torch.nn.functional.normalize(torch.randn(3, H, W, generator=g), dim=0)
    out = {"FoVx": view.FoVx, "FoVy": view.FoVy, "depth1": n(d1), "depth2": n(d2), "normal": n(nrm)}

    def loss_of(normal, maps):   # train.py:151-156, depth_ratio 0.6
        err = 1 - (normal.unsqueeze(0) * maps).sum(dim=1)
        return (1 - 0.6) * err[0].mean() + 0.6 * err[1].mean()

    for dt, suf in ((torch.float32, ""), (torch.float64, "_f64")):
        a, b, c = nrm.to(dt).clone().requires_grad_(True), d1.to(dt).clone().requires_grad_(True), d2.to(dt).clone().requires_grad_(True)
        maps = depth_double_to_normal(view, b, c)
        if dt == torch.float32:
            out["depth_normals"] = n(maps)
        v = loss_of(a, maps)
        v.backward()
        out["depth_loss" + suf], out["depth_d_normal" + suf], out["depth_d1" + suf], out["depth_d2" + suf] = n(v), n(a.grad), n(b.grad), n(c.grad)
    p1 = torch.stack([(xx - W / 2) * 0.01 * base, (yy - H / 2) * 0.01 * base, base]) + 0.005 * torch.randn(3, H, W, generator=g)
    p2 = p1 * 1.01 + 0.005 * torch.randn(3, H, W, generator=g)
    out["point1"], out["point2"] = n(p1), n(p2)
    for dt, suf in ((torch.float32, ""), (torch.float64, "_f64")):
        a, b, c = nrm.to(dt).clone().requires_grad_(True), p1.to(dt).clone().requires_grad_(True), p2.to(dt).clone().requires_grad_(True)
        maps = point_double_to_normal(view, b, c)
        if dt == torch.float32:
            out["point_normals"] = n(maps)
        v = loss_of(a, maps)
        v.backward()
        out["point_loss" + suf], out["point_d_normal" + suf], out["point_d1" + suf], out["point_d2" + suf] = n(v), n(a.grad), n(b.grad), n(c.grad)
    np.savez_compressed(os.path.join(OUT, "fused_normals.npz"), **out)


def _model(P, g, deg=3):
    pc = GaussianModel(deg)
    pc._xyz = torch.nn.Parameter((torch.rand(P, 3, generator=g) * 2 - 1) * 2.0)
    pc._features_dc = torch.nn.Parameter(torch.randn(P, 1, 3, generator=g))
    pc._features_rest = torch.nn.Parameter(0.1 * torch.randn(P, (deg + 1) ** 2 - 1, 3, generator=g))
    pc._scaling = torch.nn.Parameter(torch.randn(P, 3, generator=g) * 0.7 - 3.5)
    pc._rotation = torch.nn.Parameter(torch.randn(P, 4, generator=g))
    pc._opacity = torch.nn.Parameter(torch.randn(P, 1, generator=g) * 2)
    pc.filter_3D = torch.exp(torch.randn(P, 1, generator=g) * 0.8 - 4.0)
    pc.active_sh_degree = deg
    return pc


def gen_model():
    g = torch.Generator().manual_seed(303)
    P = 3000
    pc = _model(P, g)
    out = {"raw_scaling": n(pc._scaling), "raw_opacity": n(pc._opacity), "raw_rotation": n(pc._rotation), "filter_3D": n(pc.filter_3D)}
    scales, opacity = pc.get_scaling_n_opacity_with_3D_filter
    rot = pc.get_rotation
    gs, go, gr = torch.randn(P, 3, generator=g), torch.randn(P, 1, generator=g), torch.randn(P, 4, generator=g)
    ((scales * gs).sum() + (opacity * go).sum() + (rot * gr).sum()).backward()
    out.update(scales=n(scales), opacity=n(opacity), rotations=n(rot), g_scales=n(gs), g_opacity=n(go), g_rotations=n(gr),
               d_raw_scaling=n(pc._scaling.grad), d_raw_opacity=n(pc._opacity.grad), d_raw_rotation=n(pc._rotation.grad))
    # densification statistics: train.py:187-188 then add_densification_stats (scene/gaussian_model.py:743-747)
    pc.xyz_gradient_accum = torch.rand(P, 1, generator=g)
    pc.xyz_gradient_accum_abs = torch.rand(P, 1, generator=g)
    pc.xyz_gradient_accum_abs_max = torch.rand(P, 1, generator=g) * 0.5
    pc.denom = torch.randint(0, 5, (P, 1), generator=g).float()
    pc.max_radii2D = torch.randint(0, 30, (P,), generator=g).float()
    radii = torch.randint(-2, 40, (P,), generator=g).clamp_min(0).int()
    vsp = SimpleNamespace(grad=torch.randn(P, 3, generator=g) * torch.tensor([1.0, 1.0, 3.0]))
    vsp.grad[:, 2].abs_()
    out.update(stats_in_accum=n(pc.xyz_gradient_accum), stats_in_abs=n(pc.xyz_gradient_accum_abs), stats_in_absmax=n(pc.xyz_gradient_accum_abs_max),
               stats_in_denom=n(pc.denom), stats_in_maxradii=n(pc.max_radii2D), stats_radii=n(radii), stats_grad=n(vsp.grad))
    visibility_filter = radii > 0
    pc.max_radii2D[visibility_filter] = torch.max(pc.max_radii2D[visibility_filter], radii[visibility_filter])     # train.py:187
    pc.add_densification_stats(vsp, visibility_filter)                                                              # train.py:188
    out.update(stats_out_accum=n(pc.xyz_gradient_accum), stats_out_abs=n(pc.xyz_gradient_accum_abs), stats_out_absmax=n(pc.xyz_gradient_accum_abs_max),
               stats_out_denom=n(pc.denom), stats_out_maxradii=n(pc.max_radii2D))
    # compute_3D_filter over a ring of cameras, some of which see only part of the cloud
    cams, table = [], []
    for i in range(7):
        ang = 2 * math.pi * i / 7
        eye = np.array([5.0 * math.cos(ang), 0.5 * math.sin(2 * ang), 5.0 * math.sin(ang)])
        f = -eye / np.linalg.norm(eye)
        r = np.cross(np.array([0.0, -1.0, 0.0]), f)
        r /= np.linalg.norm(r)
        u = np.cross(f, r)
        Rw2c = np.stack([r, u, f])                    # world -> camera rotation
        cam = SimpleNamespace(R=Rw2c.T.copy(), T=(-Rw2c @ eye), FoVx=0.5 + 0.05 * i, FoVy=0.4 + 0.03 * i, image_width=320 + 16 * i, image_height=240)
        cams.append(cam)
        table.append(np.concatenate([cam.R.reshape(9), cam.T, [cam.FoVx, cam.FoVy, cam.image_width, cam.image_height]]))
    pc.compute_3D_filter(cams)
    out.update(filter_xyz=n(pc._xyz), filter_cams=np.asarray(table, dtype=np.float64), filter_out=n(pc.filter_3D))
    np.savez_compressed(os.path.join(OUT, "fused_model.npz"), **out)


def gen_ply():
    g = torch.Generator().manual_seed(404)
    P, deg = 41, 2
    pc = _model(P, g, deg)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sub", "point_cloud.ply")
        pc.save_ply(path)
        raw = np.frombuffer(open(path, "rb").read(), dtype=np.uint8)
        back = GaussianModel(deg)
        back.load_ply(path)
    np.savez_compressed(os.path.join(OUT, "fused_ply.npz"), file_bytes=raw, sh_degree=deg, xyz=n(pc._xyz), features_dc=n(pc._features_dc),
                        features_rest=n(pc._features_rest), opacity=n(pc._opacity), scaling=n(pc._scaling), rotation=n(pc._rotation),
                        filter_3D=n(pc.filter_3D), loaded_xyz=n(back._xyz), loaded_features_dc=n(back._features_dc),
                        loaded_features_rest=n(back._features_rest), loaded_opacity=n(back._opacity), loaded_scaling=n(back._scaling),
                        loaded_rotation=n(back._rotation), loaded_filter_3D=n(back.filter_3D))


if __name__ == "__main__":
    gen_losses()
    gen_normals()
    gen_model()
    gen_ply()
    for f in ("fused_losses", "fused_normals", "fused_model", "fused_ply"):
        print(f, os.path.getsize(os.path.join(OUT, f + ".npz")), "bytes")
