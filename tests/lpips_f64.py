"""LPIPS v0.1 with the VGG16 trunk, restated in torch ops: the second checker of rade_gs_b200.metrics.lpips and its
per-layer model.

Written from the definition, not from lpipsPyTorch's source: z-score the [0, 1] images with the fp32 constants
mean = (-.030, -.088, -.188), std = (.458, .448, .450); VGG16's conv/ReLU/max-pool trunk up to relu5_3; at relu1_2,
relu2_2, relu3_3, relu4_3 and relu5_3 unit-normalise the channel vector of every pixel (f / (|f| + 1e-10)), weight the
squared difference of the two images' vectors by the layer's head and average over the pixels; sum the five means.

`seeded_weights(seed)` builds a complete weight set in torchvision's and LPIPS's key names from a torch.Generator:
He-uniform conv weights, small biases, non-negative heads (LPIPS trains its heads non-negative).  The tests rebuild it
and check `digest()` against the fixture instead of storing 59 MB of weights.
"""
from __future__ import annotations

import hashlib

import torch
import torch.nn.functional as F

# torchvision vgg16().features indices of the 13 convs, grouped into the five blocks that end at a target ReLU
BLOCKS = [[0, 2], [5, 7], [10, 12, 14], [17, 19, 21], [24, 26, 28]]
CHANNELS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256), 17: (256, 512),
            19: (512, 512), 21: (512, 512), 24: (512, 512), 26: (512, 512), 28: (512, 512)}
HEAD_CHANNELS = [64, 128, 256, 512, 512]
MEAN = (-.030, -.088, -.188)
STD = (.458, .448, .450)


def seeded_weights(seed: int) -> dict:
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (cin, cout) in CHANNELS.items():
        bound = (6.0 / (9 * cin)) ** 0.5
        w = (torch.rand(cout, cin, 3, 3, generator=g).double() * 2 - 1) * bound
        b = (torch.rand(cout, generator=g).double() * 2 - 1) * 0.05
        sd[f"features.{i}.weight"] = w.float()
        sd[f"features.{i}.bias"] = b.float()
    for k, c in enumerate(HEAD_CHANNELS):
        sd[f"lin{k}.model.1.weight"] = (torch.rand(1, c, 1, 1, generator=g).double() * (2.0 / c) ** 0.5).float()
    return sd


def digest(sd: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def zscore(x: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    """x [B, 3, H, W]; the constants are the fp32 values, as the reference's buffers hold them."""
    m = torch.tensor(MEAN, dtype=torch.float32).to(x.device, dtype).view(1, 3, 1, 1)
    s = torch.tensor(STD, dtype=torch.float32).to(x.device, dtype).view(1, 3, 1, 1)
    return (x.to(dtype) - m) / s


def conv(x: torch.Tensor, sd: dict, i: int, dtype=torch.float64) -> torch.Tensor:
    """conv i (a torchvision features index) + ReLU, NCHW."""
    w, b = sd[f"features.{i}.weight"].to(x.device, dtype), sd[f"features.{i}.bias"].to(x.device, dtype)
    return F.relu(F.conv2d(x, w, b, padding=1))


def head_map(fx: torch.Tensor, fy: torch.Tensor, lin: torch.Tensor) -> torch.Tensor:
    """per-pixel distance [B, H, W] of one target layer; lin [C]."""
    nx = fx.pow(2).sum(1, keepdim=True).sqrt() + 1e-10
    ny = fy.pow(2).sum(1, keepdim=True).sqrt() + 1e-10
    return ((fx / nx - fy / ny).pow(2) * lin.to(fx).view(1, -1, 1, 1)).sum(1)


def layer_means(x: torch.Tensor, y: torch.Tensor, sd: dict, dtype=torch.float64) -> list:
    """x, y [3, H, W] or [1, 3, H, W] in [0, 1] -> the five layer means (0-d tensors of `dtype`)."""
    f = zscore(torch.cat([x.reshape(1, 3, *x.shape[-2:]), y.reshape(1, 3, *y.shape[-2:])]), dtype)
    out = []
    for k, block in enumerate(BLOCKS):
        if k:
            f = F.max_pool2d(f, 2)
        for i in block:
            f = conv(f, sd, i, dtype)
        out.append(head_map(f[:1], f[1:], sd[f"lin{k}.model.1.weight"].reshape(-1)).mean())
    return out


def lpips(x: torch.Tensor, y: torch.Tensor, sd: dict, dtype=torch.float64) -> torch.Tensor:
    m = layer_means(x, y, sd, dtype)
    return (((m[0] + m[1]) + m[2]) + m[3]) + m[4]
