"""Run the path a few times on one config (for ncu captures and quick timing).  python tools/run_once.py [cfg] [iters]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
import torch  # noqa: E402

import diff_gaussian_rasterization as dgr  # noqa: E402
from rade_gs_b200 import rawapi, scenes  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "C2"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
ks = float(sys.argv[3]) if len(sys.argv) > 3 else 0.0
sc, coord, depth = scenes.make_config(cfg)
sc = sc.to("cuda:0")
g = scenes.make_upstream_grads(sc.height, sc.width, device="cuda:0")
dgr._C.stage_timing(True)
for _ in range(iters):
    f = rawapi.forward(dgr._C, sc, coord, depth, kernel_size=ks)
    b = rawapi.backward(dgr._C, sc, f, g)
torch.cuda.synchronize()
print({k: round(v[0] / max(v[1], 1), 4) for k, v in dgr._C.stage_times().items()}, "R =", f["num_rendered"],
      "longest tile list =", int(rawapi.ours_views(f, sc)["totals"][1]))
