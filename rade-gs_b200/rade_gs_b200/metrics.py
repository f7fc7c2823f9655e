"""Image-quality scores of rendered test views on the GPU: the reference's metric.py without third-party models.

    lpips(x, y, net_type='vgg', version='0.1')   lpipsPyTorch.lpips: LPIPS v0.1 over VGG16's trunk, kernels in csrc/rgs_lpips.cu
    psnr(img1, img2)                             utils/image_utils.py's psnr
    ssim                                         rade_gs_b200.losses.ssim (utils/loss_utils.py's ssim)

    python -m rade_gs_b200.metrics -m <model_path> [<model_path> ...]

walks <model_path>/test/<method>/{renders,gt}/*.png and writes <model_path>/results.json and per_view.json with metric.py's
keys, nesting and indentation.

The weights are read from local files only, never downloaded: torchvision's `vgg16-397923af.pth` (keys features.N.weight /
features.N.bias) and LPIPS's `vgg.pth` (keys linK.model.1.weight), by default from torch.hub.get_dir()/checkpoints, where
the reference's own runs leave them.  They are loaded once per device and kept.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

from diff_gaussian_rasterization import _C
from rade_gs_b200.losses import ssim

__all__ = ["lpips", "psnr", "ssim", "load_lpips_weights", "evaluate"]

VGG_FILE = "vgg16-397923af.pth"
LIN_FILE = "vgg.pth"
VGG_URL = "https://download.pytorch.org/models/vgg16-397923af.pth"
LIN_URL = "https://raw.githubusercontent.com/richzhang/PerceptualSimilarity/master/lpips/weights/v0.1/vgg.pth"

# torchvision vgg16().features indices of the convs, grouped into the blocks that end at relu1_2 ... relu5_3
_BLOCKS = [[0, 2], [5, 7], [10, 12, 14], [17, 19, 21], [24, 26, 28]]
_CHANNELS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256), 17: (256, 512),
             19: (512, 512), 21: (512, 512), 24: (512, 512), 26: (512, 512), 28: (512, 512)}
_HEADS = [64, 128, 256, 512, 512]

_cache: dict = {}


def round_tf32(w: torch.Tensor) -> torch.Tensor:
    """fp32 -> the nearest TF32 value, ties away from zero (cvt.rna.tf32.f32's rule) for finite inputs."""
    bits = w.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def _default_path(name: str) -> str:
    return os.path.join(torch.hub.get_dir(), "checkpoints", name)


def _read(path: str, name: str, url: str) -> dict:
    if not os.path.isfile(path):
        raise FileNotFoundError(f"LPIPS weights not found at {path}: fetch {name} ({url}) and place it there, or pass its path")
    return torch.load(path, map_location="cpu", weights_only=True)


def load_lpips_weights(vgg_path: str | None = None, lin_path: str | None = None) -> dict:
    """The trunk and heads on the CPU in the kernels' layouts: conv1_1 as torch's [64, 3, 3, 3]; every other conv
    repacked to [C_out, 3, 3, C_in] and rounded to TF32; the heads as [C] vectors.  Raises FileNotFoundError for a
    missing file and ValueError for a missing key or a tensor of the wrong shape."""
    vgg_path = vgg_path or _default_path(VGG_FILE)
    lin_path = lin_path or _default_path(LIN_FILE)
    vgg, lin = _read(vgg_path, VGG_FILE, VGG_URL), _read(lin_path, LIN_FILE, LIN_URL)

    def take(sd, key, shape, path):
        if key not in sd:
            raise ValueError(f"{path}: no tensor {key}")
        t = sd[key]
        if tuple(t.shape) != shape:
            raise ValueError(f"{path}: {key} has shape {tuple(t.shape)}, expected {shape}")
        return t.detach().float().contiguous()

    convs = []
    for i, (cin, cout) in _CHANNELS.items():
        w = take(vgg, f"features.{i}.weight", (cout, cin, 3, 3), vgg_path)
        b = take(vgg, f"features.{i}.bias", (cout,), vgg_path)
        convs.append((w if i == 0 else round_tf32(w.permute(0, 2, 3, 1).contiguous()), b))
    heads = [take(lin, f"lin{k}.model.1.weight", (1, c, 1, 1), lin_path).reshape(c) for k, c in enumerate(_HEADS)]
    return {"convs": convs, "heads": heads}


def _weights_on(device: torch.device, vgg_path, lin_path) -> dict:
    key = (str(device), vgg_path, lin_path)
    if key not in _cache:
        w = load_lpips_weights(vgg_path, lin_path)
        _cache[key] = {"convs": [(a.to(device), b.to(device)) for a, b in w["convs"]], "heads": [h.to(device) for h in w["heads"]]}
    return _cache[key]


def _as_chw(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dim() == 4:
        if t.shape[0] != 1:
            raise ValueError(f"{name}: one image per call ([3, H, W] or [1, 3, H, W]), got batch {t.shape[0]}")
        t = t[0]
    if t.dim() != 3 or t.shape[0] != 3:
        raise ValueError(f"{name} must be [3, H, W] or [1, 3, H, W], got {list(t.shape)}")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if t.shape[1] < 16 or t.shape[2] < 16:
        raise ValueError(f"{name}: LPIPS-VGG needs at least 16 x 16 pixels (four 2x2 pools), got {t.shape[1]} x {t.shape[2]}")
    return t


def lpips(x: torch.Tensor, y: torch.Tensor, net_type: str = "vgg", version: str = "0.1", *, vgg_path: str | None = None,
          lin_path: str | None = None, layers: bool = False):
    """LPIPS distance of x and y ([3, H, W] or [1, 3, H, W], float32 in [0, 1], CUDA, H and W >= 16) as a [1, 1, 1, 1]
    float32 tensor, as lpipsPyTorch.lpips(x, y, net_type='vgg') returns it.

    Not differentiable: the result has no grad_fn (metric.py only reports the value).  The trunk runs in TF32 on the
    tensor cores, as the reference's cuDNN convolutions do with torch's default allow_tf32; the five layer means are
    summed in fp64.  With layers=True, also returns the five layer means (fp64 [5]).
    """
    if net_type != "vgg":
        raise NotImplementedError(f"net_type {net_type!r}: only 'vgg' is implemented (the one metric.py uses)")
    if version != "0.1":
        raise ValueError(f"version {version!r}: only LPIPS v0.1 exists")
    a, b = _as_chw(x, "x"), _as_chw(y, "y")
    if a.shape != b.shape:
        raise ValueError(f"x and y differ in shape: {list(a.shape)} and {list(b.shape)}")
    if not a.is_cuda or b.device != a.device:
        raise ValueError("lpips needs x and y on one CUDA device: there is no CPU path")
    L = _C._lpips
    with torch.no_grad(), torch.cuda.device(a.device):
        w = _weights_on(a.device, vgg_path, lin_path)
        bufs = [torch.empty(0, dtype=torch.uint8, device=a.device) for _ in range(2)]
        (w0, b0), convs = w["convs"][0], iter(w["convs"][1:])
        f, cur = L.input_conv(a.detach(), b.detach(), w0, b0, bufs[0]), 0
        means = []
        for k, block in enumerate(_BLOCKS):
            if k:
                cur ^= 1
                f = L.maxpool(f, bufs[cur])
            for _ in block[1:] if k == 0 else block:
                cw, cb = next(convs)
                cur ^= 1
                f = L.conv3x3(f, cw, cb, bufs[cur])
            means.append(L.distance(f, w["heads"][k])[1])
        m = torch.cat(means)
        total = ((((m[0] + m[1]) + m[2]) + m[3]) + m[4]).float().view(1, 1, 1, 1)
    return (total, m) if layers else total


def psnr(img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
    """20 log10(1 / sqrt(mse)) per image, mse over each image's elements: [B, 1] for [B, ...] inputs."""
    mse = ((img1 - img2) ** 2).view(img1.shape[0], -1).mean(1, keepdim=True)
    return 20 * torch.log10(1.0 / torch.sqrt(mse))


def _read_png(path: str, device) -> torch.Tensor:
    from PIL import Image
    with Image.open(path) as im:
        a = np.asarray(im)
    if a.ndim == 2:
        a = a[:, :, None]
    scale = 65535.0 if a.dtype == np.uint16 else 255.0
    t = torch.from_numpy(a.astype(np.float32) / np.float32(scale)).permute(2, 0, 1)[:3]
    return t.unsqueeze(0).contiguous().to(device)


def _score_method(method_dir: str, device) -> tuple:
    renders_dir, gt_dir = os.path.join(method_dir, "renders"), os.path.join(method_dir, "gt")
    names = sorted(os.listdir(renders_dir))
    ssims, psnrs, lps = [], [], []
    for name in names:
        r, g = _read_png(os.path.join(renders_dir, name), device), _read_png(os.path.join(gt_dir, name), device)
        ssims.append(ssim(r, g).item())
        psnrs.append(psnr(r, g).item())
        lps.append(lpips(r, g).item())
    s, p, lp = torch.tensor(ssims), torch.tensor(psnrs), torch.tensor(lps)
    full = {"SSIM": s.mean().item(), "PSNR": p.mean().item(), "LPIPS": lp.mean().item()}
    per_view = {"SSIM": dict(zip(names, s.tolist())), "PSNR": dict(zip(names, p.tolist())), "LPIPS": dict(zip(names, lp.tolist()))}
    return full, per_view


def evaluate(model_paths, device="cuda") -> int:
    """metric.py's evaluate: per scene, results.json (means) and per_view.json (per image) for every method under test/.
    A scene that fails is reported with the reason and skipped; returns the number of such scenes."""
    failed = 0
    for scene_dir in model_paths:
        print("Scene:", scene_dir)
        try:
            full, per_view = {}, {}
            test_dir = os.path.join(scene_dir, "test")
            for method in sorted(os.listdir(test_dir)):
                print("Method:", method)
                full[method], per_view[method] = _score_method(os.path.join(test_dir, method), device)
                for k in ("SSIM", "PSNR", "LPIPS"):
                    print(f"  {k:<5}: {full[method][k]:>12.7f}")
                print("")
            with open(os.path.join(scene_dir, "results.json"), "w") as fp:
                json.dump(full, fp, indent=True)
            with open(os.path.join(scene_dir, "per_view.json"), "w") as fp:
                json.dump(per_view, fp, indent=True)
        except Exception as e:  # noqa: BLE001 -- one scene's failure must not stop the others
            failed += 1
            print(f"Unable to compute metrics for model {scene_dir}: {type(e).__name__}: {e}", file=sys.stderr)
    return failed


def main(argv=None) -> int:
    parser = argparse.ArgumentParser(description="SSIM, PSNR and LPIPS of rendered test views (metric.py on the GPU)")
    parser.add_argument("--model_paths", "-m", required=True, nargs="+", type=str, default=[])
    args = parser.parse_args(argv)
    return 1 if evaluate(args.model_paths) else 0


if __name__ == "__main__":
    sys.exit(main())
