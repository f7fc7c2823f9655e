"""Time the decoupled-appearance L1 loss (train.py:37-58) with the head in the project's kernels against the previous
composition: the module's head on cuDNN under torch's default flags, autograd for its backward, and the same tail kernels.

    python tools/bench_appearance_head.py [--iters 200] [--out DIR]

Per image size (800 x 600, 979 x 546, 1600 x 1200): forward + backward of the whole loss and of the head alone, both
compositions alternated in one process, CUDA-event medians after a warm-up of every shape.  Then, in a separate profiled run,
each head kernel's time and the launches per call, and each kernel's achieved FLOP/s against the FP32 data-sheet rate
(67 TFLOP/s dense, H100 SXM) and its bytes against 3.35 TB/s, from the shapes.  Prints the card's name and power limit with
the numbers; with --out also writes them as JSON there.  Needs a GPU: there is no CPU path."""
import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))

from diff_gaussian_rasterization import _C  # noqa: E402
from rade_gs_b200.appearance import L1_loss_appearance, _head_params  # noqa: E402

SIZES = [(600, 800), (546, 979), (1200, 1600)]
FP32_PEAK = 67e12
HBM = 3.35e12
LAYERS = [("conv1", 67, 256, 0), ("up1", 64, 128, 1), ("up2", 32, 64, 2), ("up3", 16, 32, 3), ("up4", 8, 16, 4)]


class _Up(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.pixel_shuffle = nn.PixelShuffle(2)
        self.conv = nn.Conv2d(cin // 4, cout, 3, padding=1)
        self.relu = nn.ReLU()

    def forward(self, x):
        return self.relu(self.conv(self.pixel_shuffle(x)))


class _Net(nn.Module):
    """scene/appearance_network.py's layers and parameter order."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(67, 256, 3, padding=1)
        self.up1, self.up2, self.up3, self.up4 = _Up(256, 128), _Up(128, 64), _Up(64, 32), _Up(32, 16)
        self.conv2 = nn.Conv2d(16, 16, 3, padding=1)
        self.conv3 = nn.Conv2d(16, 3, 3, padding=1)
        self.relu = nn.ReLU()


def _module_head(net, down, emb):
    h, w = down.shape[1:]
    x = torch.cat([down, emb[:, None, None].expand(64, h, w)], dim=0)[None]
    return net.up4(net.up3(net.up2(net.up1(net.relu(net.conv1(x))))))


class _PreviousL1(torch.autograd.Function):
    """The previous composition: the module's head on cuDNN and autograd, the tail entries of csrc/rgs_appearance.cu."""

    @staticmethod
    def forward(ctx, image, gt, emb, net, *params):
        image, gt = image.contiguous(), gt.contiguous()
        down = _C.appearance_downsample(image)
        with torch.enable_grad():
            d_leaf = down.detach().requires_grad_(True)
            e_leaf = emb.detach().requires_grad_(True)
            up4 = _module_head(net, d_leaf, e_leaf)
        w2, b2, w3, b3 = (p.detach() for p in (net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias))
        loss, act, _ = _C.appearance_l1_forward(image, gt, up4.detach(), w2, b2, w3, b3, True, False)
        ctx.head = (up4, d_leaf, e_leaf, params[:-4])
        ctx.save_for_backward(image, gt, act, w2, b2, w3, b3)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        image, gt, act, w2, b2, w3, b3 = ctx.saved_tensors
        up4, d_leaf, e_leaf, head_params = ctx.head
        d_img, d_up4, d_w2, d_b2, d_w3, d_b3 = _C.appearance_l1_backward(image, gt, up4.detach(), act, w2, b2, w3, b3, grad_out.float().reshape(1))
        grads = torch.autograd.grad(up4, [d_leaf, e_leaf, *head_params], d_up4)
        _C.appearance_downsample_backward(grads[0], d_img)
        ctx.head = None
        return (d_img, None, grads[1], None, *grads[2:], d_w2, d_b2, d_w3, d_b3)


def previous_L1(image, gt, g, view):
    net = g.appearance_network
    params = _head_params(net) + [net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias]
    return _PreviousL1.apply(image, gt, g.get_apperance_embedding(view), net, *params)


def _setup(H0, W0, seed):
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H0, W0, generator=gen)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=gen)).clamp(0, 1)
    net = _Net()
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(torch.randn(p.shape, generator=gen) * ((2.0 / (p.shape[1] * 9)) ** 0.5 if p.dim() == 4 else 0.05))
    net = net.cuda()
    table = nn.Parameter(0.5 * torch.randn(8, 64, generator=gen).cuda())
    g = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: table[i])
    return g, table, image.cuda().requires_grad_(True), gt.cuda()


def _zero(g, table, image):
    for p in list(g.appearance_network.parameters()) + [table, image]:
        p.grad = None


def _loss_step(fn, g, table, image, gt):
    _zero(g, table, image)
    fn(image, gt, g, 3).backward()


def _head_inputs(g, table, image):
    down = _C.appearance_downsample(image.detach())
    emb = table[3].detach()
    params = [p.detach() for p in _head_params(g.appearance_network)]
    h, w = down.shape[1:]
    d_up4 = torch.randn(1, 16, 16 * h, 16 * w, device="cuda")
    return down, emb, params, d_up4


def _head_new(down, emb, params, d_up4):
    act, up4 = _C._appearance_head.forward(down, emb, params)
    _C._appearance_head.backward(down, emb, params, act, up4, d_up4)


def _head_old(net, down, emb, d_up4):
    d_leaf, e_leaf = down.requires_grad_(True), emb.requires_grad_(True)
    up4 = _module_head(net, d_leaf, e_leaf)
    torch.autograd.grad(up4, [d_leaf, e_leaf, *_head_params(net)], d_up4)


def _time(fn, iters):
    """Per-call CUDA-event times (ms) of `iters` calls."""
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def _alternate(fns, iters, rounds=10):
    """`rounds` alternations of `iters // rounds` calls of each function; returns the median per function."""
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k] += _time(f, max(1, iters // rounds))
    return {k: statistics.median(v) for k, v in times.items()}


def head_work(h, w):
    """Per layer: multiply-adds of the forward convolution (the data and the weight gradient each take as many) and the bytes
    each kernel must at least move (its input and output maps once, fp32)."""
    out = []
    for name, cin, cout, L in LAYERS:
        H, W = h << L, w << L
        macs = cin * cout * 9 * H * W
        in_bytes = 4 * (3 if L == 0 else cin) * H * W
        out_bytes = 4 * cout * H * W
        out.append({"layer": name, "macs": macs, "fwd_bytes": in_bytes + out_bytes, "dgrad_bytes": 2 * out_bytes + in_bytes,
                    "wgrad_bytes": 2 * out_bytes + in_bytes})
    return out


def _card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def _profile(H0, W0):
    """Kernel names, device times and launches of one new-path loss call (forward + backward), and of the head alone."""
    from torch.profiler import ProfilerActivity, profile
    g, table, image, gt = _setup(H0, W0, 1)
    down, emb, params, d_up4 = _head_inputs(g, table, image)
    for _ in range(3):
        _loss_step(L1_loss_appearance, g, table, image, gt)
        _head_new(down, emb, params, d_up4)
    torch.cuda.synchronize()
    res = {}
    for key, fn, n in (("loss", lambda: _loss_step(L1_loss_appearance, g, table, image, gt), 20), ("head", lambda: _head_new(down, emb, params, d_up4), 20)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith("Memset") and not e.name.startswith("Memcpy"):
                k = kernels.setdefault(e.name, [0, 0.0])
                k[0] += 1
                k[1] += e.device_time
        res[key] = {"launches_per_call": sum(v[0] for v in kernels.values()) / n,
                    "kernels": {k: {"calls_per_call": v[0] / n, "us_per_call": v[1] / n} for k, v in sorted(kernels.items(), key=lambda kv: -kv[1][1])}}
    return res


def _rates(prof_head, h, w):
    """Each head kernel's achieved FLOP/s and bytes/s from the shapes, against the data-sheet rates."""
    work = {x["layer"]: x for x in head_work(h, w)}
    cin_to_layer = {str(cin): name for name, cin, _, _ in LAYERS}
    rows = []
    for k, v in prof_head["kernels"].items():
        kind = "forward" if "forward_kernel" in k else "dgrad" if "dgrad_kernel" in k else "wgrad" if "wgrad_kernel" in k else None
        if kind is None:
            continue
        # the template's first argument is the layer's input channel count: "<int, ...>" in the demangled name
        cin = k.split("<", 1)[1].split(",", 1)[0].strip() if "<" in k else ""
        layer = cin_to_layer.get(cin)
        if layer is None:
            continue
        wk = work[layer]
        t = v["us_per_call"] * 1e-6
        flops = 2 * wk["macs"]
        nbytes = wk[{"forward": "fwd_bytes", "dgrad": "dgrad_bytes", "wgrad": "wgrad_bytes"}[kind]]
        t_flop, t_byte = flops / FP32_PEAK, nbytes / HBM
        rows.append({"kernel": f"{layer} {kind}", "us": v["us_per_call"], "TFLOP/s": flops / t / 1e12, "share_of_fp32_peak": t_flop / t,
                     "GB/s": nbytes / t / 1e9, "bound": "FP32 FLOP" if t_flop >= t_byte else "HBM bytes",
                     "share_of_bound": max(t_flop, t_byte) / t})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_appearance_head needs a GPU")
    card = _card()
    print(f"card: {card['name']}, power limit / max SM clock: {card['power_limit_and_max_sm_clock']}")
    print(f"torch cudnn flags: enabled={torch.backends.cudnn.enabled} allow_tf32={torch.backends.cudnn.allow_tf32} "
          f"deterministic={torch.backends.cudnn.deterministic} benchmark={torch.backends.cudnn.benchmark}")
    setups = {s: _setup(*s, 7) for s in SIZES}
    heads = {s: _head_inputs(*[setups[s][i] for i in (0, 1, 2)]) for s in SIZES}
    for s in SIZES:   # warm every shape of both compositions
        g, table, image, gt = setups[s]
        down, emb, params, d_up4 = heads[s]
        for _ in range(5):
            _loss_step(L1_loss_appearance, g, table, image, gt)
            _loss_step(previous_L1, g, table, image, gt)
            _head_new(down, emb, params, d_up4)
            _head_old(g.appearance_network, down.clone(), emb.clone(), d_up4)
    torch.cuda.synchronize()
    results = {"card": card, "sizes": []}
    for s in SIZES:
        g, table, image, gt = setups[s]
        down, emb, params, d_up4 = heads[s]
        loss = _alternate({"new": lambda: _loss_step(L1_loss_appearance, g, table, image, gt),
                           "previous": lambda: _loss_step(previous_L1, g, table, image, gt)}, args.iters)
        head = _alternate({"new": lambda: _head_new(down, emb, params, d_up4),
                           "previous": lambda: _head_old(g.appearance_network, down.clone(), emb.clone(), d_up4)}, args.iters)
        r = {"size": f"{s[1]}x{s[0]}", "loss_ms": loss, "head_ms": head}
        results["sizes"].append(r)
        print(f"{r['size']:>10}: loss fwd+bwd  new {loss['new']:.3f} ms  previous {loss['previous']:.3f} ms   |   "
              f"head fwd+bwd  new {head['new']:.3f} ms  previous {head['previous']:.3f} ms")
    for s in SIZES:
        p = _profile(*s)
        h, w = s[0] // 32, s[1] // 32
        r = next(x for x in results["sizes"] if x["size"] == f"{s[1]}x{s[0]}")
        r["profile"] = p
        r["head_kernels"] = _rates(p["head"], h, w)
        print(f"{r['size']:>10}: launches per call: loss {p['loss']['launches_per_call']:.0f}, head {p['head']['launches_per_call']:.0f}")
        for k in r["head_kernels"]:
            print(f"            {k['kernel']:<14} {k['us']:8.1f} us  {k['TFLOP/s']:6.2f} TFLOP/s ({100 * k['share_of_fp32_peak']:5.1f}% of 67)  "
                  f"{k['GB/s']:7.1f} GB/s  bound: {k['bound']}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_appearance_head.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
