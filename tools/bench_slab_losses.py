"""Slab-local normal consistency on one GPU: the kernel of each slab of a 1-, 2-, 4- and 8-way row partition against the
whole-image kernel, at 1600x1200 and 979x546, depth and coordinate forms.

For every partition it reports the slowest slab (what each rank waits for) and the sum over the slabs (the halo stencils each
slab evaluates again), CUDA-event medians over --timed windows of 20 back-to-back calls, with the card's name and power limit.  The
halo exchange between ranks and a whole sharded training step are not timed here; the output says so.

Usage:  python tools/bench_slab_losses.py [--timed 50] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))


def _inputs(H, W, from_depth, dev):
    g = torch.Generator().manual_seed(H + W)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    base = 3.0 + 0.02 * xx + 0.03 * yy + 0.3 * torch.sin(xx * 0.4) * torch.cos(yy * 0.3)
    d1, d2 = base + 0.01 * torch.randn(H, W, generator=g), base + 0.05 * torch.randn(H, W, generator=g)
    n = torch.nn.functional.normalize(torch.randn(3, H, W, generator=g), dim=0)
    if from_depth:
        return n.to(dev), d1[None].to(dev), d2[None].to(dev)
    pts = lambda d: torch.stack([(xx - W / 2) * d / 500, (yy - H / 2) * d / 500, d])  # noqa: E731
    return n.to(dev), pts(d1).to(dev), pts(d2).to(dev)


def _median_ms(fn, timed, batch=20):
    """Median over `timed` windows of `batch` back-to-back calls (a single call of a few tens of microseconds is as much the
    launch as the kernel), per call."""
    for _ in range(10):
        fn()
    times = []
    for _ in range(timed):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(batch):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / batch)
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timed", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_slab_losses needs a CUDA device")
    from diff_gaussian_rasterization import _C
    from rade_gs_b200.multigpu import partition_tile_rows, tile_rows
    dev = torch.device("cuda", 0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi.splitlines()[0] if smi else torch.cuda.get_device_name(0),
           "method": f"CUDA-event median of {a.timed} windows of 20 back-to-back calls, per call, after 10 warm-up calls", "normal_consistency": {}}
    for H, W in ((1200, 1600), (546, 979)):
        for from_depth in (True, False):
            n, e, m = _inputs(H, W, from_depth, dev)
            cam = (1 / 1000.0, 1 / 1000.0, -W / 2000.0, -H / 2000.0) if from_depth else (0.0, 0.0, 0.0, 0.0)
            w_e, w_m = 0.4 / (H * W), 0.6 / (H * W)
            whole = _median_ms(lambda: _C.normal_consistency(n, e, m, from_depth, *cam, w_e, w_m), a.timed)
            row = {"whole_ms": round(whole, 4)}
            for world in (1, 2, 4, 8):
                per = []
                for b, end in partition_tile_rows(tile_rows(H), world):
                    r0, r1 = min(b * 16, H), min(end * 16, H)
                    m_lo, m_hi, n_lo, n_hi = max(0, r0 - 2), min(H, r1 + 2), max(0, r0 - 1), min(H, r1 + 1)
                    # windows as a rank holds them after the halo exchange: contiguous buffers of its rows
                    nw, ew, mw = n[:, n_lo:n_hi].contiguous(), e[:, m_lo:m_hi].contiguous(), m[:, m_lo:m_hi].contiguous()
                    per.append(_median_ms(lambda: _C._slab.normal_consistency_rows(nw, ew, mw, from_depth, *cam, w_e, w_m, H, r0, r1), a.timed))
                row[f"{world}way"] = {"slowest_slab_ms": round(max(per), 4), "sum_ms": round(sum(per), 4)}
            res["normal_consistency"][f"{W}x{H}/{'depth' if from_depth else 'coord'}"] = row
    ngpu = torch.cuda.device_count()
    res["sharded_step"] = f"not measured ({ngpu} GPU{'s' if ngpu != 1 else ''} present; this script times the kernels only)"
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
