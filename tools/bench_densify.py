"""Densify-and-prune on one GPU: the eager model (tests/densify_model.py, the reference's tensor operations regrouped, timed as
the reference runs it, torch.cuda.empty_cache() included) against rade_gs_b200.densify.densify_and_prune.  SH degree 3,
P = 1 M, 3 M and 10 M, with clone / split / prune fractions of a few percent each, as mid-training densification sees them.
Prints one JSON line per P and implementation: median ms per call over --reps calls, peak torch.cuda.max_memory_allocated
during the call, and the card's name and power limit.  The quantile threshold comes from a CUB radix sort of grads_abs.

    python tools/bench_densify.py [--sizes 1000000,3000000,10000000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")]

import densify_model as dm                 # noqa: E402
from rade_gs_b200 import densify           # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def make_inputs(P, seed=0):
    """Device tensors of a model: ~3 % of rows over max_grad, half of the scales over percent_dense * extent, ~2 % faint."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.rand(*s, device="cuda", generator=g)      # noqa: E731
    n = lambda *s: torch.randn(*s, device="cuda", generator=g)     # noqa: E731
    t = {"xyz": r(P, 3) * 4 - 2, "f_dc": n(P, 1, 3), "f_rest": 0.1 * n(P, 15, 3), "opacity": n(P, 1) * 1.2 + 1.5,
         "scaling": n(P, 3) * 0.6 - 3.6, "rotation": n(P, 4)}
    denom = torch.randint(1, 20, (P, 1), device="cuda", generator=g).float()
    t["denom"] = denom
    t["accum"] = (r(P, 1) ** 8) * 0.0006 * denom
    t["accum_abs"] = (r(P, 1) ** 8) * 0.004 * denom
    for k in dm.GROUPS:
        t[k + ".exp_avg"], t[k + ".exp_avg_sq"] = n(*t[k].shape) * 1e-4, r(*t[k].shape) * 1e-8
    return t


def model_from(t):
    m = dm.Model()
    for name, attr in dm.GROUPS.items():
        setattr(m, attr, torch.nn.Parameter(t[name].clone()))
    P = t["xyz"].shape[0]
    m.xyz_gradient_accum, m.xyz_gradient_accum_abs, m.denom = t["accum"].clone(), t["accum_abs"].clone(), t["denom"].clone()
    m.xyz_gradient_accum_abs_max = torch.zeros(P, 1, device="cuda")
    m.max_radii2D = torch.zeros(P, device="cuda")
    m.filter_3D = torch.zeros(P, 1, device="cuda")
    m.percent_dense = 0.01
    groups = [{"params": [getattr(m, attr)], "lr": 1e-3, "name": name} for name, attr in dm.GROUPS.items()]
    m.optimizer = torch.optim.Adam(groups, lr=0.0, eps=1e-15, fused=True)
    for name, attr in dm.GROUPS.items():
        m.optimizer.state[getattr(m, attr)] = {"step": torch.tensor(100.0, device="cuda"), "exp_avg": t[name + ".exp_avg"].clone(),
                                               "exp_avg_sq": t[name + ".exp_avg_sq"].clone()}
    return m


def reference_like(m, *args):
    out, _ = dm.densify_and_prune(m, *args)
    torch.cuda.empty_cache()
    return out


def time_one(fn, t, reps):
    times, peaks, result = [], [], None
    for i in range(reps + 1):
        m = model_from(t)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(i)
        t0 = time.perf_counter()
        result = fn(m, 0.0002, 0.05, 4.0, 20)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if i:                       # the first call warms up allocations and module loads
            times.append(dt * 1e3)
            peaks.append(torch.cuda.max_memory_allocated() - base)
        del m
        torch.cuda.empty_cache()
    times.sort()
    return times[len(times) // 2], max(peaks), result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,3000000,10000000")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_densify needs a CUDA device")
    gpu = card()
    for P in (int(s) for s in a.sizes.split(",")):
        t = make_inputs(P)
        for impl, fn in (("model_eager", reference_like), ("fused", densify.densify_and_prune)):
            ms, peak, result = time_one(fn, t, a.reps)
            print(json.dumps({"P": P, "impl": impl, "median_ms": round(ms, 3), "peak_extra_bytes": int(peak),
                              "cloned_split_pruned": list(result), "quantile": "cub_radix_sort", "gpu": gpu}), flush=True)
        del t
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
