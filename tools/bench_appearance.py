"""Fused vs eager decoupled-appearance L1 loss (train.py:37-58), forward + backward, at the recipes' image sizes.  Prints one JSON
line.

Eager is the reference expression with torch's defaults (cuDNN may use TF32), which is how the reference trains.  Times are CUDA
events, median over --iters iterations after --warmup.  Per-kernel times of the fused path come from torch.profiler in a separate
pass; achieved FLOP/s use the algorithmic FMA counts (tail forward: conv2 + conv3 = 2736 FMA per crop pixel; tail backward:
2x that for the input and weight gradients of both convolutions, not counting the conv3 recompute), 2 FLOP per FMA.

    python tools/bench_appearance.py [--iters 30] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")]

from test_gpu_appearance import _recipe_inputs, _ref_loss, _setup   # noqa: E402
from rade_gs_b200.appearance import L1_loss_appearance               # noqa: E402

SIZES = [(600, 800), (546, 979), (1200, 1600)]
TAIL_FMA = 16 * 16 * 9 + 3 * 16 * 9


def _median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def _kernel_times(step, n=10):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "rgs" in e.key and e.device_type.name == "CUDA":
            short = next((k for k in ("tail_forward", "tail_backward", "upsample_transpose", "downsample_backward", "downsample", "grad_finish",
                                      "loss_finish") if k in e.key), e.key[:40])
            out[short] = round(e.device_time_total / n / 1000.0, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_appearance needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "sizes": []}
    for H0, W0 in SIZES:
        inp = _recipe_inputs(H0, W0, H0 + W0)
        row = {"image": f"{W0}x{H0}", "crop": f"{W0 // 32 * 32}x{H0 // 32 * 32}"}
        for name, fn in (("fused", L1_loss_appearance), ("eager", _ref_loss)):
            g, image, gt = _setup(inp)

            def step():
                image.grad = None
                fn(image, gt, g, 3).backward()
            row[name + "_fwd_bwd_ms"] = round(_median_ms(step, args.iters, args.warmup), 4)
            if name == "fused":
                row["fused_kernels_ms"] = kt = _kernel_times(step)
                px = (H0 // 32 * 32) * (W0 // 32 * 32)
                for k, mult in (("tail_forward", 1), ("tail_backward", 2)):
                    if k in kt:
                        row[k + "_tflops"] = round(2 * mult * TAIL_FMA * px / (kt[k] * 1e-3) / 1e12, 2)
        row["speedup"] = round(row["eager_fwd_bwd_ms"] / row["fused_fwd_bwd_ms"], 3)
        res["sizes"].append(row)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
