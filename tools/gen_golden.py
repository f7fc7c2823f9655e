"""Generate the golden fixtures under tests/golden/ from the UNMODIFIED reference build (oracle/_ref/ref_dgr_C.so).

Must run where a GPU is (the reference has no CPU path):   python tools/gen_golden.py [CASE ...]
The outputs land in golden_out/; copy them to tests/golden/ and commit them together with this script.
Each fixture holds a digest of the inputs (regenerated from the case's seed by tools/golden_inputs.py), the settings, every forward output, the reference's internal per-Gaussian /
binning state (decoded from its buffers, SURVEY.md appendix B) and the eight gradient tensors.  The reference's
backward uses float atomics, so gradients are stored as the mean of two runs and the observed run-to-run
difference is stored next to them (`grad_noise_*`).
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rade_gs_b200 import rawapi, scenes  # noqa: E402

import golden_inputs  # noqa: E402

# name: (P, W, H, focal, mu, seed, coord, depth, kernel_size, sh_degree, look_at, precomp)
CASES = {
    "depth_ks0": dict(P=1500, W=96, H=64, focal=80.0, mu=-2.2, seed=11, coord=False, depth=True, ks=0.0, deg=3, view="tilt"),
    "depth_ks01": dict(P=1500, W=96, H=64, focal=80.0, mu=-2.2, seed=12, coord=False, depth=True, ks=0.1, deg=3, view="tilt"),
    "coord_ks0": dict(P=1500, W=100, H=60, focal=80.0, mu=-2.2, seed=13, coord=True, depth=False, ks=0.0, deg=2, view="tilt"),
    "both_ks01": dict(P=1500, W=96, H=64, focal=80.0, mu=-2.2, seed=14, coord=True, depth=True, ks=0.1, deg=3, view="identity"),
    "none_ks0": dict(P=1500, W=96, H=64, focal=80.0, mu=-2.2, seed=15, coord=False, depth=False, ks=0.0, deg=1, view="tilt"),
    "tiny_splats": dict(P=1500, W=96, H=64, focal=80.0, mu=-4.6, seed=16, coord=False, depth=True, ks=0.0, deg=3, view="tilt"),
    "precomp": dict(P=1000, W=64, H=48, focal=60.0, mu=-2.2, seed=17, coord=True, depth=True, ks=0.0, deg=0, view="tilt", precomp=True),
}


def build_case(c):
    view = None
    if c["view"] == "tilt":
        view = scenes.look_at_view((0.4, -0.3, -0.5), (0.1, 0.05, 6.0))
    sc = scenes.make_scene(c["P"], c["W"], c["H"], c["focal"], c["mu"], seed=c["seed"], view=view, bg=(0.1, 0.2, 0.3))
    # a few hand-placed hard cases: behind the camera, on the near plane, huge, needle-like, zero opacity
    P = c["P"]
    sc.scales[0] = torch.tensor([2.0, 2.0, 2.0])
    sc.scales[1] = torch.tensor([0.5, 1e-4, 1e-4])
    sc.scales[2] = torch.tensor([1e-5, 0.3, 0.3])
    sc.opacities[3] = 0.0
    sc.opacities[4] = 1.0
    vm = sc.viewmatrix.t()  # maths convention
    cam_pts = torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, 0.2], [0.0, 0.0, 0.2001], [50.0, 0.0, 3.0]])
    world = (cam_pts - vm[:3, 3]) @ vm[:3, :3]
    sc.means3D[5:9] = world
    extra = {}
    if c.get("precomp"):
        g = torch.Generator().manual_seed(c["seed"] + 100)
        extra["colors_precomp"] = torch.rand(P, 3, generator=g)
        L = torch.randn(P, 3, 3, generator=g) * 0.08
        cov = L @ L.transpose(1, 2)
        cov[10] = torch.diag(torch.tensor([0.04, 0.04, 1e-10]))  # ill-conditioned: rank-1 inverse branch
        cov[11] = torch.zeros(3, 3)
        extra["cov3D_precomp"] = torch.stack([cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]], 1).contiguous()
    return sc, extra


def main():
    only = sys.argv[1:]
    import build_ref
    ref = build_ref.load()
    dev = torch.device("cuda:0")
    out_dir = "golden_out"
    os.makedirs(out_dir, exist_ok=True)
    for name, c in CASES.items():
        if only and name not in only:
            continue
        sc_cpu, extra = build_case(c)
        sc = sc_cpu.to(dev)
        ex = {k: v.to(dev) for k, v in extra.items()}
        grads = scenes.make_upstream_grads(sc.height, sc.width, seed=4321 + c["seed"], device=dev)
        f = rawapi.forward(ref, sc, c["coord"], c["depth"], kernel_size=c["ks"], sh_degree=c["deg"], **ex)
        b1 = rawapi.backward(ref, sc, f, grads)
        b2 = rawapi.backward(ref, sc, f, grads)
        torch.cuda.synchronize()
        v = rawapi.ref_views(f, sc)
        rec = {"meta_" + k: np.array(val) for k, val in c.items() if not isinstance(val, str)}
        rec["meta_view"] = np.array(c["view"])
        inputs = golden_inputs.rasterize_inputs(name)
        assert all(np.array_equal(inputs["gin_" + k], val.cpu().numpy()) for k, val in grads.items())
        rec["inputs_digest"] = np.array(golden_inputs.digest(inputs))
        rec["in_tanfov"] = np.array([sc_cpu.tanfovx, sc_cpu.tanfovy], dtype=np.float64)
        rec["num_rendered"] = np.array(f["num_rendered"])
        for k in ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth", "radii"):
            rec["out_" + k] = f[k].cpu().numpy()
        for k in ("depths", "camera_planes", "ray_planes", "ts", "normals", "clamped", "means2D", "view_points", "cov3D", "conic_opacity", "rgb",
                  "tiles_touched", "point_list", "keys", "n_contrib", "ranges"):
            rec["st_" + k] = v[k].cpu().numpy()
        for k in rawapi.BWD_KEYS:
            rec["grad_" + k] = (0.5 * (b1[k].double() + b2[k].double())).float().cpu().numpy()
            rec["grad_noise_" + k] = np.array((b1[k] - b2[k]).abs().max().item() if b1[k].numel() else 0.0)
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: R={f['num_rendered']} visible={(f['radii'] > 0).sum().item()} -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
