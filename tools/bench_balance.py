"""Equal against balanced row slabs on one GPU: what each rank of a 2-, 4- and 8-way sharded step would spend on its slab.

For a uniform scene and a skewed one (dense splats in the image's lower third, one in twelve of the rest above it), both at
1920x1080, every slab of the equal partition (`rasterize_gaussians_slab`) and of the balanced one (`_C._slab.rasterize_balanced`,
the call `ShardedGaussianRasterizer(balance=True)` makes) is rendered forward and backward (stage 1 + stage 2, without the
exchange) on this one GPU.  Reported per partition: each slab's forward and backward milliseconds, the slowest slab (what every
rank waits for) and the sum over the slabs.  The balanced rows are also rendered through `rasterize_gaussians_slab`
("fixed_on_balanced_rows"): the difference to "balanced" is the balanced call's own cost (whole-image tile counts, the per-row
read, the restriction).  Also a least-squares fit of the per-slab time over a + b * instances + d * tiles,
whose d / b is the per-tile cost in instances that include/rgs_b200.h's RGS_BALANCE_TILE_COST states.  CUDA-event medians of
--timed runs after --warmup, with the card's name and power limit read in the same process.  Ranks on different GPUs, the
gradient exchange and a whole training step are not timed here.

Usage:  python tools/bench_balance.py [--warmup 3] [--timed 9] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))

W, H = 1920, 1080


def _scenes():
    from rade_gs_b200 import scenes
    view = scenes.look_at_view((0.1, -0.1, -0.2), (0.0, 0.0, 6.0))
    uniform = scenes.make_scene(600_000, W, H, 1100.0, -4.2, seed=3, view=view, bg=(0.1, 0.2, 0.3))
    dense = scenes.make_scene(2_400_000, W, H, 1100.0, -4.2, seed=4, view=view, bg=(0.1, 0.2, 0.3))
    hom = torch.cat([dense.means3D, torch.ones(dense.means3D.shape[0], 1)], 1) @ dense.projmatrix
    py = ((hom[:, 1] / (hom[:, 3] + 1e-7) + 1.0) * H - 1.0) * 0.5
    keep = (py >= 2 * H / 3) | (torch.arange(py.shape[0]) % 12 == 0)
    kw = {k: (v[keep] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == keep.shape[0] else v) for k, v in vars(dense).items()}
    return {"uniform": uniform, "skewed": scenes.Scene(**kw)}


def _median_ms(fn, warmup, timed):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(timed):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--timed", type=int, default=9)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_balance needs a CUDA device: nothing here has a CPU path, and a CPU time says nothing about the GPU")
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import multigpu, rawapi, scenes
    C, dev = dgr._C, torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=60).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    report = {"card": card, "image": [W, H], "tile_cost": C._slab.BALANCE_TILE_COST, "runs": []}
    fit_rows = []
    for name, sc0 in _scenes().items():
        sc = sc0.to(dev)
        grads = scenes.make_upstream_grads(H, W, seed=5, device=dev)
        call = dict(require_coord=False, require_depth=True, kernel_size=0.1, sh_degree=3, scale_modifier=1.0, debug=False, compact=True,
                    shs=sc.shs, cols=rawapi._absent(), scales=sc.scales, rots=sc.rotations, cov=rawapi._absent())
        args = rawapi._forward_args(sc, call)
        stats = C._slab.rasterize_balanced(*args, 1, 0, True)[13]
        for world in (2, 4, 8):
            cuts = C._slab.balance_partition(stats[0].tolist(), gx, world)
            parts = {"equal": multigpu.partition_tile_rows(gy, world), "balanced": [(cuts[r], cuts[r + 1]) for r in range(world)]}
            parts["fixed_on_balanced_rows"] = parts["balanced"]   # the same rows through rasterize_gaussians_slab: the balanced call's own cost
            for kind, slabs in parts.items():
                fwd_ms, bwd_ms = [], []
                for rank, (b, e) in enumerate(slabs):
                    r0, r1 = b * 16, min(e * 16, H)
                    g = {k: v[:, r0:r1].contiguous() for k, v in grads.items()}

                    def forward():
                        if kind == "balanced":
                            out = C._slab.rasterize_balanced(*args, world, rank, True)
                            assert out[12] == cuts
                        else:
                            out = C.rasterize_gaussians_slab(*args, b, e, True)
                        f = dict(zip(rawapi.FWD_KEYS, out[:12]))
                        f["_call"] = dict(call, tile_rows=(b, e))
                        return f

                    f = forward()
                    fwd_ms.append(_median_ms(forward, a.warmup, a.timed))
                    bwd_ms.append(_median_ms(lambda: rawapi.backward_preprocess(C, sc, f, rawapi.backward_render(C, sc, f, g)), a.warmup, a.timed))
                    inst = int(stats[0][b:e].sum())
                    if kind != "fixed_on_balanced_rows":
                        fit_rows.append((inst, (e - b) * gx, fwd_ms[-1] + bwd_ms[-1]))
                tot = [x + y for x, y in zip(fwd_ms, bwd_ms)]
                inst = [int(stats[0][b:e].sum()) for b, e in slabs]
                run = {"scene": name, "P": int(sc.means3D.shape[0]), "world": world, "partition": kind, "tile_rows": [list(s) for s in slabs],
                       "instances": inst, "fwd_ms": [round(x, 4) for x in fwd_ms], "bwd_ms": [round(x, 4) for x in bwd_ms],
                       "slowest_ms": round(max(tot), 4), "sum_ms": round(sum(tot), 4)}
                report["runs"].append(run)
                print(json.dumps(run), flush=True)
    X = np.array([[1.0, i, t] for i, t, _ in fit_rows])
    y = np.array([ms for _, _, ms in fit_rows])
    coef = np.linalg.lstsq(X, y, rcond=None)[0]
    report["fit"] = {"ms_intercept": float(coef[0]), "ms_per_instance": float(coef[1]), "ms_per_tile": float(coef[2]),
                     "tile_cost_in_instances": float(coef[2] / coef[1]) if coef[1] > 0 else None, "slabs": len(fit_rows)}
    print(json.dumps({"fit": report["fit"]}), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
