"""Workload statistics that decide optimisation choices (needs a GPU):  python tools/diag_stats.py [C2]
  * visible Gaussians whose accumulator row is all-zero after backward-render (no pixel received them): backward-preprocess and
    the SH backward could skip them;
  * hits per (warp, splat) and live-lane statistics are in the ncu captures (smsp__thread_inst_executed_per_inst_executed)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
import torch  # noqa: E402

import diff_gaussian_rasterization as dgr  # noqa: E402
from rade_gs_b200 import scenes  # noqa: E402

C = dgr._C
for cfg in sys.argv[1:] or ["C2"]:
    sc, coord, depth = scenes.make_config(cfg)
    sc = sc.to("cuda")
    g = scenes.make_upstream_grads(sc.height, sc.width, device="cuda")
    E = torch.Tensor([])
    gy = (sc.height + 15) // 16
    out = C.rasterize_gaussians_slab(sc.bg, sc.means3D, E, sc.opacities, sc.scales, sc.rotations, 1.0, E, sc.viewmatrix, sc.projmatrix, sc.tanfovx, sc.tanfovy,
                                     0.0, sc.height, sc.width, sc.shs, 3, sc.campos, False, coord, depth, False, 0, gy)
    acc = C.rasterize_gaussians_backward_render(sc.bg, sc.means3D, out[8], E, sc.scales, sc.rotations, 1.0, E, sc.viewmatrix, sc.projmatrix, sc.tanfovx,
                                                sc.tanfovy, 0.0, g["color"], g["coord"], g["mcoord"], g["depth"], g["mdepth"], g["alpha"], g["normal"], out[5],
                                                sc.shs, 3, sc.campos, out[9], out[0], out[10], out[11], out[4], coord, depth, False, 0, gy)
    vis = out[8] > 0
    zero = ~(acc != 0).any(dim=1)
    print(f"{cfg}: P {vis.numel()} visible {int(vis.sum())} visible-with-all-zero-gradient-row {int((vis & zero).sum())} "
          f"({100.0 * int((vis & zero).sum()) / max(int(vis.sum()), 1):.1f}% of visible)  num_rendered {out[0]}")
