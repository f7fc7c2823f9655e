"""Golden fixtures for `integrate_gaussians_to_points` (SURVEY.md 8f row 3) from the UNMODIFIED reference build.

Must run where a GPU is:   python tools/gen_golden_integrate.py [OUT_DIR]
Outputs land in OUT_DIR (default golden_out/) as integrate_*.npz; copy them to tests/golden/ and commit them with this script.
The inputs are stored as a digest; tools/golden_inputs.py rebuilds them from the case's seed.

The reference path has undefined behaviour outside a safe envelope, which the cases stay inside:
  * its `condition` tensor is allocated with PN (points) entries but indexed by Gaussian (rasterize_points.cu:318,
    forward.cu:379) -> PN >= P here;
  * for ill-conditioned covariances the inverse ray covariance is never assigned (a shadowed local, forward.cu:214) -> no
    needle / flat splats here.
The call is made twice and must agree bit for bit (every output element has a single writer).
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rade_gs_b200 import scenes  # noqa: E402

CASES = {
    "integrate_tilt": dict(P=1200, PN=5000, W=96, H=64, focal=80.0, mu=-2.2, seed=31, deg=3, view="tilt"),
    "integrate_front": dict(P=800, PN=1500, W=64, H=48, focal=60.0, mu=-2.0, seed=32, deg=1, view="identity"),
    "integrate_dense": dict(P=3000, PN=12000, W=48, H=48, focal=70.0, mu=-1.6, seed=33, deg=0, view="tilt"),
}


def make_points(sc, PN, seed):
    """Query points the way mesh extraction makes them (get_tetra_points: centres and scaled box corners of the
    Gaussians) plus uniform points in front of the camera, a few behind it and a few far off-screen."""
    g = torch.Generator().manual_seed(seed)
    P = sc.means3D.shape[0]
    n_box = PN // 2
    idx = torch.randint(0, P, (n_box,), generator=g)
    corners = (torch.randint(0, 2, (n_box, 3), generator=g).float() * 2 - 1) * 3.0
    corners[: n_box // 4] = 0.0  # centres
    box = sc.means3D[idx] + corners * sc.scales[idx]
    n_uni = PN - n_box - 40
    vm = sc.viewmatrix.t()
    z = torch.rand(n_uni, generator=g) * 9 + 1.5
    x = (torch.rand(n_uni, generator=g) * 2 - 1) * sc.tanfovx * 1.1 * z
    y = (torch.rand(n_uni, generator=g) * 2 - 1) * sc.tanfovy * 1.1 * z
    cam = torch.stack([x, y, z], 1)
    behind = torch.stack([torch.randn(20, generator=g), torch.randn(20, generator=g), -torch.rand(20, generator=g) * 3], 1)
    far_off = torch.stack([torch.full((20,), 60.0), torch.randn(20, generator=g), torch.full((20,), 3.0)], 1)
    world = (torch.cat([cam, behind, far_off]) - vm[:3, 3]) @ vm[:3, :3]
    return torch.cat([box, world]).contiguous()


def build_case(c):
    view = scenes.look_at_view((0.4, -0.3, -0.5), (0.1, 0.05, 6.0)) if c["view"] == "tilt" else None
    sc = scenes.make_scene(c["P"], c["W"], c["H"], c["focal"], c["mu"], seed=c["seed"], view=view, bg=(0.1, 0.2, 0.3))
    sc.opacities[3] = 0.0
    sc.opacities[4] = 1.0
    vm = sc.viewmatrix.t()
    cam_pts = torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, 0.2], [0.0, 0.0, 0.2001], [50.0, 0.0, 3.0]])
    sc.means3D[5:9] = (cam_pts - vm[:3, 3]) @ vm[:3, :3]
    return sc, make_points(sc, c["PN"], c["seed"] + 500)


def call_reference(ref, sc, pts, deg):
    none = torch.Tensor([])
    M = (deg + 1) ** 2
    sub = torch.zeros((sc.height, sc.width, 2), dtype=torch.float32, device=pts.device)
    return ref.integrate_gaussians_to_points(
        sc.bg, pts, sc.means3D, none, sc.opacities, sc.scales, sc.rotations, 1.0, none, none, sc.viewmatrix, sc.projmatrix,
        sc.tanfovx, sc.tanfovy, 0.0, sub, sc.height, sc.width, sc.shs[:, :M].contiguous(), deg, sc.campos, False, False)


def main():
    import build_ref
    ref = build_ref.load()
    dev = torch.device("cuda:0")
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "golden_out"
    os.makedirs(out_dir, exist_ok=True)
    for name, c in CASES.items():
        sc_cpu, pts_cpu = build_case(c)
        assert pts_cpu.shape[0] >= sc_cpu.means3D.shape[0]
        sc, pts = sc_cpu.to(dev), pts_cpu.to(dev)
        r1 = call_reference(ref, sc, pts, c["deg"])
        r2 = call_reference(ref, sc, pts, c["deg"])
        torch.cuda.synchronize()
        names = ("color", "alpha_integrated", "color_integrated", "point_coordinate", "point_sdf", "radii")
        for k, a, b in zip(names, r1[1:7], r2[1:7]):
            assert torch.equal(a, b), f"{name}: reference output {k} differs between two runs"
        rec = {"meta_" + k: np.array(v) for k, v in c.items() if not isinstance(v, str)}
        rec["meta_view"] = np.array(c["view"])
        import golden_inputs
        rec["inputs_digest"] = np.array(golden_inputs.digest(golden_inputs.integrate_inputs(name)))
        rec["in_tanfov"] = np.array([sc_cpu.tanfovx, sc_cpu.tanfovy], dtype=np.float64)
        rec["num_rendered"] = np.array(r1[0])
        for k, a in zip(names, r1[1:7]):
            rec["out_" + k] = a.cpu().numpy()
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, **rec)
        ai = r1[2]
        print(f"{name}: R={r1[0]} points touched={(ai != 1.0).sum().item()}/{ai.numel()} alpha range [{ai.min().item():.3f}, {ai.max().item():.3f}] "
              f"max pts/pixel={int(r1[1][8].max().item())} -> {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
