"""Time rade_gs_b200.metrics.lpips per image pair against the reference's LPIPS-VGG computed by torch (cuDNN, TF32 on).

Arms, per size (1600x1200, 1920x1080, 979x546), median over --reps pairs after --warmup:
  ours      metrics.lpips (csrc/rgs_lpips.cu), weights loaded once per device
  cudnn     tests/lpips_f64's restatement in fp32 through cuDNN with allow_tf32=True, its weights on the device once: the fair arm
  per_call  the reference's per-call pattern (lpipsPyTorch/__init__.py builds LPIPS('vgg') on every call): build torchvision's
            vgg16, load both state dicts from the local files, move to the GPU, run; timed at the first size only
Also: achieved TF32 TFLOP/s of `ours` from the shapes (FLOP count below) against the data sheet's 495 (H100 SXM, dense),
both arms' outputs compared at the timed sizes, and the card name and power limit read in the same process.

Weights are seeded (tests/lpips_f64.seeded_weights): timings do not depend on their values.

    python tools/bench_metrics.py [--reps 20] [--warmup 3] [--out results/bench_metrics.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")]

import lpips_f64 as ref                                   # noqa: E402
from rade_gs_b200 import metrics                          # noqa: E402

SIZES = [(1200, 1600), (1080, 1920), (546, 979)]
TF32_PEAK = 495e12


def flops(H, W):
    """multiply-adds x 2 of the 13 convs for a pair (the pools floor each side); the distance is negligible."""
    total, h, w = 0, H, W
    for k, block in enumerate(ref.BLOCKS):
        if k:
            h, w = h // 2, w // 2
        for i in block:
            cin, cout = ref.CHANNELS[i]
            total += 2 * (2 * h * w) * cout * 9 * cin
    return total


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_metrics: no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    sd = ref.seeded_weights(1)
    tmp = tempfile.mkdtemp()
    vgg, lin = os.path.join(tmp, metrics.VGG_FILE), os.path.join(tmp, metrics.LIN_FILE)
    torch.save({k: v for k, v in sd.items() if k.startswith("features.")}, vgg)
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, lin)
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = False
    g = torch.Generator().manual_seed(0)
    rows = []
    for n, (H, W) in enumerate(SIZES):
        x, y = torch.rand(3, H, W, generator=g).cuda(), torch.rand(3, H, W, generator=g).cuda()
        ours = lambda: metrics.lpips(x, y, vgg_path=vgg, lin_path=lin)                       # noqa: E731
        with torch.no_grad():
            cud = lambda: ref.lpips(x, y, sd_dev, dtype=torch.float32)                        # noqa: E731
            t_ours, t_cudnn = timed(ours, args.reps, args.warmup), timed(cud, args.reps, args.warmup)
            v_ours, v_cudnn = ours().item(), cud().item()
        row = {"size": f"{W}x{H}", "ours_ms": t_ours, "cudnn_tf32_ms": t_cudnn, "tflop_per_pair": flops(H, W) / 1e12,
               "ours_tflops": flops(H, W) / (t_ours * 1e-3) / 1e12, "cudnn_tflops": flops(H, W) / (t_cudnn * 1e-3) / 1e12,
               "ours_share_of_495": flops(H, W) / (t_ours * 1e-3) / TF32_PEAK, "ours_value": v_ours, "cudnn_value": v_cudnn,
               "rel_diff": abs(v_ours - v_cudnn) / abs(v_cudnn)}
        if n == 0:
            import torchvision

            def per_call():
                m = torchvision.models.vgg16(weights=None).features
                m.load_state_dict({k[len("features."):]: v for k, v in torch.load(vgg, map_location="cpu", weights_only=True).items()})
                heads = torch.load(lin, map_location="cpu", weights_only=True)
                m = m.cuda()
                w = {f"features.{k}": v for k, v in m.state_dict().items()}
                w.update({k: v.cuda() for k, v in heads.items()})
                return ref.lpips(x, y, w, dtype=torch.float32)

            with torch.no_grad():
                row["per_call_rebuild_ms"] = timed(per_call, max(3, args.reps // 4), 1)
        rows.append(row)
        print(json.dumps(row), flush=True)
    res = {"card": card, "rows": rows}
    print(json.dumps({"card": card}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
