"""The fused training step run eagerly (INTEGRATION.md §4) against the same step replayed from a CUDA graph (rade_gs_b200.graphs).

Configs: C2 (1 M Gaussians, 1600x1200) and a DTU-recipe scene (0.3 M Gaussians, 800x600, with the decoupled-appearance loss).
Step: activate_gaussians -> split-SH depth-variant render -> l1_ssim_loss + depth_normal_consistency_loss (+ L1_loss_appearance)
-> backward(); the camera and ground truth are copied into static device tensors, cycling over 8 views.  The optimizer is
outside both arms.

  * per-step wall time: a host clock over --steps steps ending in a synchronize, the two arms alternating in --windows windows;
    median and range over the windows;
  * GPU-busy time per step and the tile_sort_kernel time per step: torch.profiler over --profile-steps steps of each arm, in a
    run of its own after the timed windows;
  * the card's name and power limit, read in the same call.

Usage: python tools/bench_graph_step.py [--configs C2,DTU] [--steps 200] [--windows 5] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))

import torch  # noqa: E402

CONFIGS = {"C2": dict(P=1_000_000, W=1600, H=1200, focal=1600.0, mu=-5.0, appearance=False),
           "DTU": dict(P=300_000, W=800, H=600, focal=700.0, mu=-4.6, appearance=True)}
VIEWS = 8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class _Up(torch.nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.shuffle = torch.nn.PixelShuffle(2)
        self.conv = torch.nn.Conv2d(cin, cout, 3, padding=1)
        self.relu = torch.nn.ReLU()


class _AppearanceNetwork(torch.nn.Module):
    """scene/appearance_network.py's layers (names and parameter order)."""

    def __init__(self):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(67, 256, 3, padding=1)
        self.up1, self.up2, self.up3, self.up4 = _Up(64, 128), _Up(32, 64), _Up(16, 32), _Up(8, 16)
        self.conv2 = torch.nn.Conv2d(16, 16, 3, padding=1)
        self.conv3 = torch.nn.Conv2d(16, 3, 3, padding=1)
        self.relu = torch.nn.ReLU()


class Model:
    def __init__(self, sc, dev):
        self._xyz = sc.means3D.clone().requires_grad_(True)
        self._scaling = torch.log(sc.scales).requires_grad_(True)
        self._opacity = torch.logit(sc.opacities.clamp(1e-4, 1 - 1e-4)).requires_grad_(True)
        self._rotation = sc.rotations.clone().requires_grad_(True)
        self._features_dc = sc.shs[:, :1].clone().requires_grad_(True)
        self._features_rest = sc.shs[:, 1:].contiguous().requires_grad_(True)
        self.filter_3D = torch.full((sc.means3D.shape[0], 1), 1e-3, device=dev)
        self.appearance_network = _AppearanceNetwork().to(dev)
        self._appearance_embeddings = torch.nn.Parameter(0.1 * torch.randn(VIEWS, 64, device=dev))

    def get_apperance_embedding(self, idx):
        return self._appearance_embeddings.index_select(0, idx.reshape(1))[0]   # no host read of a 0-dim CUDA index

    def params(self, appearance):
        extra = [self._appearance_embeddings, *self.appearance_network.parameters()] if appearance else []
        return [self._xyz, self._scaling, self._opacity, self._rotation, self._features_dc, self._features_rest, *extra]


class Step:
    def __init__(self, sc, model, appearance, reserve, dev):
        import diff_gaussian_rasterization as dgr
        self.m, self.appearance = model, appearance
        self.view, self.proj, self.campos = torch.zeros(4, 4, device=dev), torch.zeros(4, 4, device=dev), torch.zeros(3, device=dev)
        self.gt = torch.zeros(3, sc.height, sc.width, device=dev)
        self.view_idx = torch.zeros((), dtype=torch.int64, device=dev)
        self.means2D = torch.zeros_like(model._xyz, requires_grad=True)
        self.cam = type("Cam", (), {"FoVx": 2 * math.atan(sc.tanfovx), "FoVy": 2 * math.atan(sc.tanfovy)})()
        s = dgr.GaussianRasterizationSettings(sc.height, sc.width, sc.tanfovx, sc.tanfovy, 0.0, sc.bg, 1.0, self.view, self.proj, 3, self.campos,
                                              False, True, False, False)
        self.rast = dgr.GaussianRasterizer(s, reserve)

    def params(self):
        return self.m.params(self.appearance) + [self.means2D]

    def load(self, cam, gt, idx):
        with torch.no_grad():
            for s, v in zip((self.view, self.proj, self.campos), cam):
                s.copy_(v)
            self.gt.copy_(gt)
            self.view_idx.fill_(idx)

    def __call__(self):
        from rade_gs_b200.appearance import L1_loss_appearance
        from rade_gs_b200.fused import activate_gaussians
        from rade_gs_b200.losses import depth_normal_consistency_loss, l1_ssim_loss
        m = self.m
        scales, opacity, rotations = activate_gaussians(m._scaling, m._opacity, m._rotation, m.filter_3D)
        color, radii, _, _, depth, mdepth, _, normal = self.rast(m._xyz, self.means2D, opacity, shs=(m._features_dc, m._features_rest),
                                                                 scales=scales, rotations=rotations)
        loss = l1_ssim_loss(color, self.gt, 0.2) + 0.05 * depth_normal_consistency_loss(self.cam, normal, depth, mdepth)
        if self.appearance:
            loss = loss + L1_loss_appearance(color, self.gt, m, self.view_idx)
        loss.backward()
        return loss.detach()


def setup(name, dev):
    from rade_gs_b200 import scenes
    from rade_gs_b200.graphs import BinningReserve, StepGraph
    c = CONFIGS[name]
    sc = scenes.make_scene(c["P"], c["W"], c["H"], c["focal"], c["mu"], seed=2024).to(dev)
    cams = []
    for i in range(VIEWS):
        a = 2 * math.pi * i / VIEWS
        V = scenes.look_at_view((0.3 * math.sin(a), 0.2 * math.cos(a), -0.2), (0.05 * math.cos(a), 0.0, 6.0))
        view = V.t().contiguous()
        proj = scenes.projection_matrix(0.01, 100.0, 2 * math.atan(sc.tanfovx), 2 * math.atan(sc.tanfovy)).t()
        cams.append(tuple(t.to(dev) for t in (view, (view @ proj).contiguous(), view.inverse()[3, :3].contiguous())))
    gts = [torch.rand(3, sc.height, sc.width, generator=torch.Generator(device=dev).manual_seed(i), device=dev) for i in range(VIEWS)]
    torch.manual_seed(1)
    model = Model(sc, dev)
    eager = Step(sc, model, c["appearance"], None, dev)
    reserve = BinningReserve(dev)
    graphed = Step(sc, model, c["appearance"], reserve, dev)
    sg = StepGraph(reserve)
    key = (sc.height, sc.width, sc.tanfovx, sc.tanfovy, c["P"], *(p.data_ptr() for p in graphed.params()))
    state = {"i": 0}

    def eager_step():
        i = state["i"] = (state["i"] + 1) % VIEWS
        eager.load(cams[i], gts[i], i)
        for p in eager.params():
            if p.grad is not None:
                p.grad.zero_()
        return eager()

    def graph_step():
        i = state["i"] = (state["i"] + 1) % VIEWS
        graphed.load(cams[i], gts[i], i)
        return sg.run(key, graphed, graphed.params())

    return {"eager": eager_step, "graph": graph_step}, sg, reserve


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def profiled(fn, steps):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    busy = sort = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            t = e.device_time if hasattr(e, "device_time") else e.cuda_time
            busy += t
            if "tile_sort_kernel" in e.name:
                sort += t
    return busy / 1e3 / steps, sort / 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,DTU")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_step.py needs a CUDA device")
    dev = torch.device("cuda:0")
    results = {"card": card(), "steps_per_window": a.steps, "windows": a.windows, "configs": {}}
    for name in a.configs.split(","):
        arms, sg, reserve = setup(name, dev)
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
        wall = {k: [] for k in arms}
        for _ in range(a.windows):
            for k, fn in arms.items():
                wall[k].append(timed(fn, a.steps))
        prof = {k: profiled(fn, a.profile_steps) for k, fn in arms.items()}
        r = {k: {"wall_ms_median": statistics.median(v), "wall_ms_min": min(v), "wall_ms_max": max(v), "gpu_busy_ms": prof[k][0],
                 "tile_sort_ms": prof[k][1]} for k, v in wall.items()}
        r["captures"], r["fallbacks"] = sg.captures, sg.fallbacks
        r["reserve"] = {"instances": reserve.instances, "longest_list": reserve.longest_list}
        results["configs"][name] = r
        print(json.dumps({name: r}), flush=True)
        del arms, sg, reserve
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
