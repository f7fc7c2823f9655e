"""Slab-local decoupled-appearance L1 loss on one GPU: the forward and backward row kernels (`_C._slab.appearance_l1_*_rows`) of
each slab of a 1-, 2-, 4- and 8-way row partition at 800x600, 979x546 and 1600x1200, against the whole-image kernels, and the
replicated cuDNN head (conv1, up1..up4 forward and backward) timed apart.

For every partition it reports the slowest slab (what each rank waits for) and the sum over the slabs (the halo rows each slab
evaluates again), CUDA-event medians over --timed windows of 20 back-to-back calls, with the card's name and power limit read in the
same run.  The halo exchange, the two all-gathers (low-resolution rows, d(up4) rows) and a whole sharded training step need several
GPUs and are not timed here; the output says so.

Usage:  python tools/bench_slab_appearance.py [--timed 50] [--out FILE.json]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_slab_losses import _median_ms  # noqa: E402

HALO = 4


def _inputs(H0, W0, dev):
    g = torch.Generator().manual_seed(H0 + W0)
    H, W = H0 // 32 * 32, W0 // 32 * 32
    gt = torch.rand(3, H0, W0, generator=g)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=g)).clamp(0, 1)
    up4 = torch.relu(torch.randn(1, 16, H // 2, W // 2, generator=g))
    w2, b2 = torch.randn(16, 16, 3, 3, generator=g) * (2.0 / 144) ** 0.5, 0.05 * torch.randn(16, generator=g)
    w3, b3 = torch.randn(3, 16, 3, 3, generator=g) * (2.0 / 144) ** 0.5, 0.05 * torch.randn(3, generator=g)
    return [t.to(dev) for t in (image, gt, up4, w2, b2, w3, b3)]


def _head_ms(H0, W0, dev, timed):
    """conv1, up1..up4 forward + backward from d(up4) at the image's low resolution, as every rank runs them."""
    from rade_gs_b200.appearance import _head, _head_input
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_appearance import _Net
    net = _Net().to(dev)
    down = torch.rand(3, H0 // 32, W0 // 32, device=dev, requires_grad=True)
    emb = torch.randn(64, device=dev, requires_grad=True)
    g = torch.randn(1, 16, H0 // 32 * 16, W0 // 32 * 16, device=dev)

    def step():
        up4 = _head(net, _head_input(down, emb))
        torch.autograd.grad(up4, [down, emb, *net.parameters()], g, allow_unused=True)
    return _median_ms(step, timed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timed", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_slab_appearance needs a CUDA device")
    from diff_gaussian_rasterization import _C
    from rade_gs_b200.multigpu import partition_tile_rows, tile_rows
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi.splitlines()[0] if smi else torch.cuda.get_device_name(0),
           "method": f"CUDA-event median of {a.timed} windows of 20 back-to-back calls, per call, after 10 warm-up calls", "appearance": {}}
    up = torch.ones(1, device=dev)
    for H0, W0 in ((600, 800), (546, 979), (1200, 1600)):
        image, gt, up4, w2, b2, w3, b3 = _inputs(H0, W0, dev)
        _, act, _ = _C.appearance_l1_forward(image, gt, up4, w2, b2, w3, b3, True, False)
        row = {"whole_forward_ms": round(_median_ms(lambda: _C.appearance_l1_forward(image, gt, up4, w2, b2, w3, b3, True, False), a.timed), 4),
               "whole_backward_ms": round(_median_ms(lambda: _C.appearance_l1_backward(image, gt, up4, act, w2, b2, w3, b3, up), a.timed), 4),
               "head_fwd_bwd_ms": round(_head_ms(H0, W0, dev, a.timed), 4)}
        for world in (1, 2, 4, 8):
            fwd, bwd = [], []
            for b, e in partition_tile_rows(tile_rows(H0), world):
                r0, r1 = min(b * 16, H0), min(e * 16, H0)
                lo, hi = max(0, r0 - HALO), min(H0, r1 + HALO)
                # windows as a rank holds them after the halo exchange: contiguous buffers of its rows
                win, gwin = image[:, lo:hi].contiguous(), gt[:, lo:hi].contiguous()
                _, act_w = _C._slab.appearance_l1_forward_rows(win, gwin, lo, H0, r0, r1, up4, w2, b2, w3, b3)
                fwd.append(_median_ms(lambda: _C._slab.appearance_l1_forward_rows(win, gwin, lo, H0, r0, r1, up4, w2, b2, w3, b3), a.timed))
                bwd.append(_median_ms(lambda: _C._slab.appearance_l1_backward_rows(win, gwin, lo, H0, r0, r1, up4, act_w, w2, b2, w3, b3, up), a.timed))
            row[f"{world}way"] = {"forward": {"slowest_slab_ms": round(max(fwd), 4), "sum_ms": round(sum(fwd), 4)},
                                  "backward": {"slowest_slab_ms": round(max(bwd), 4), "sum_ms": round(sum(bwd), 4)}}
        res["appearance"][f"{W0}x{H0}"] = row
    ngpu = torch.cuda.device_count()
    res["multi_gpu"] = (f"not measured ({ngpu} GPU{'s' if ngpu != 1 else ''} present; the halo exchange, the two all-gathers and a sharded "
                        "step need several GPUs, and this script times the kernels only)")
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
