"""The fp64 image-loss models (tests/image_loss_f64.py) validated without a GPU: they equal fp64 autograd of the reference's
expressions, and their bounds hold an fp32 evaluation of the kernels' expressions at every pixel."""
import math

import pytest
import torch
import torch.nn.functional as F

import image_loss_f64 as il
from f32_error import check, check_shadow


# ---- reference expressions (utils/loss_utils.py:17-63, utils/graphics_utils.py:97-126, train.py:143-163) -------------------

def ref_ssim_l1(img, gt, lam):
    """(1 - lam) L1 + lam (1 - SSIM) in the dtype of img, with the kernel's fp32 window taps and C1, C2."""
    ch = img.shape[-3]
    g = torch.tensor(il.window(), dtype=img.dtype)[:, None]
    w = (g @ g.t()).expand(ch, 1, 11, 11).contiguous()
    x, y = img.reshape(1, ch, *img.shape[-2:]), gt.reshape(1, ch, *img.shape[-2:]).to(img.dtype)
    conv = lambda t: F.conv2d(t, w, padding=5, groups=ch)
    mu1, mu2 = conv(x), conv(y)
    s1, s2, s12 = conv(x * x) - mu1 ** 2, conv(y * y) - mu2 ** 2, conv(x * y) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + il.C1) * (2 * s12 + il.C2)) / ((mu1 ** 2 + mu2 ** 2 + il.C1) * (s1 + s2 + il.C2))
    return (1 - lam) * (x - y).abs().mean() + lam * (1 - ssim.mean()), ssim


def ref_normal(normal, e, m, from_depth, inv_fx, inv_fy, cx, cy, ratio):
    H, W = normal.shape[-2:]
    if from_depth:
        yy, xx = torch.meshgrid(torch.arange(H, dtype=normal.dtype), torch.arange(W, dtype=normal.dtype), indexing="ij")
        rays = torch.stack([(xx + 0.5) * inv_fx + cx, (yy + 0.5) * inv_fy + cy, torch.ones_like(xx)])
        e, m = e.reshape(1, H, W) * rays, m.reshape(1, H, W) * rays
    points = torch.stack([e, m])
    out = torch.zeros_like(points)
    dx = points[..., 2:, 1:-1] - points[..., :-2, 1:-1]
    dy = points[..., 1:-1, 2:] - points[..., 1:-1, :-2]
    out[..., 1:-1, 1:-1] = F.normalize(torch.cross(dx, dy, dim=1), dim=1)
    err = 1 - (normal.unsqueeze(0) * out).sum(dim=1)
    return (1 - ratio) * err[0].mean() + ratio * err[1].mean()


# ---- image families -------------------------------------------------------------------------------------------------------

def images(kind, shape, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(*shape, generator=g)
    if kind == "random":
        img = (gt + 0.15 * torch.randn(*shape, generator=g)).clamp(0, 1)
    elif kind == "identical":
        img = gt.clone()
    elif kind == "constant":
        gt = torch.full(shape, 0.37)
        img = torch.full(shape, 0.61)
    elif kind == "bright_close":
        gt = 0.98 + 0.02 * torch.rand(*shape, generator=g)
        img = (gt + 1e-4 * torch.randn(*shape, generator=g)).clamp(max=1.0)
    elif kind == "saturated":
        gt = (torch.rand(*shape, generator=g) > 0.5).float()
        img = (torch.rand(*shape, generator=g) > 0.5).float()
    return img, gt


KINDS = ("random", "identical", "constant", "bright_close", "saturated")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", [(3, 17, 33), (1, 5, 1), (1, 1, 31), (3, 16, 32)])
def test_ssim_model_equals_fp64_autograd(kind, shape):
    img, gt = images(kind, shape, sum(shape))
    lam = 0.2
    fw = il.ssim_l1_forward(img, gt)
    n = img.numel()
    # weights 1 and 0 are exact in fp32: combine the two parts in fp64 with the reference's weights
    d = il.ssim_l1_backward(fw, 1.0, 0.0).v * (-lam / n) + il.ssim_l1_backward(fw, 0.0, 1.0).v * ((1 - lam) / n)
    x = img.double().requires_grad_(True)
    loss, ssim = ref_ssim_l1(x, gt.double(), lam)
    loss.backward()
    # both sides round E[x^2] - mu^2 in fp64 and divide by b >= C2 = 9e-4: 121 terms x 1e-16 / C2 ~ 1e-11 at most
    torch.testing.assert_close(fw["ssim_map"].v, ssim.detach().reshape(fw["ssim_map"].v.shape), rtol=1e-12, atol=5e-11)
    model_loss = lam + (-lam / n) * fw["sums"][0][0] + ((1 - lam) / n) * fw["sums"][1][0]
    assert abs(model_loss.item() - loss.item()) <= 1e-11
    scale = x.grad.abs().max().item() + 1.0 / n
    torch.testing.assert_close(d.reshape(x.shape), x.grad, rtol=1e-9, atol=1e-9 * scale)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rows", [(0, None), (3, 4), (0, 7), (9, 17)])
def test_ssim_bounds_hold_an_fp32_evaluation(kind, rows):
    img, gt = images(kind, (3, 17, 33), 5)
    lo, hi = rows
    fw = il.ssim_l1_forward(img, gt, lo, hi, shadow=True)
    r = fw["rows"]
    for i, name in enumerate(("d/d mu1", "d/d E[x^2]", "d/d E[xy]")):
        check_shadow(fw["dmaps"][i][:, r], f"{kind} dmaps {name}")
    d = il.ssim_l1_backward(fw, -0.2 / img.numel(), 0.8 / img.numel(), upstream=1.7)
    check_shadow(d, f"{kind} d_img")


@pytest.mark.parametrize("from_depth", [True, False])
@pytest.mark.parametrize("HW", [(1, 1), (2, 3), (3, 3), (17, 15), (16, 16)])
@pytest.mark.parametrize("ratio", [0.0, 0.6, 1.0])
def test_normal_model_equals_fp64_autograd(from_depth, HW, ratio):
    H, W = HW
    inp = normal_inputs(H, W, from_depth, seed=H * 31 + W, background=False)
    cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
    n = H * W
    # weights 1 and 0 are exact in fp32: combine the two maps' parts in fp64 with the reference's weights
    a, b = (1 - ratio) / n, ratio / n
    oe = il.normal_consistency(*inp, from_depth, *cam, 1.0, 0.0)
    om = il.normal_consistency(*inp, from_depth, *cam, 0.0, 1.0)
    leaves = [t.double().requires_grad_(True) for t in inp]
    ref = ref_normal(*leaves, from_depth, *(il.f32(c) for c in cam), ratio)
    ref.backward()
    assert abs(a * oe["loss"][0].item() + b * om["loss"][0].item() - ref.item()) <= 1e-12
    got = (a * oe["d_normal"].v + b * om["d_normal"].v, a * oe["d_e"].v, b * om["d_m"].v)
    for g, leaf in zip(got, leaves):
        torch.testing.assert_close(g.reshape(leaf.shape), leaf.grad, rtol=1e-12, atol=1e-12 * (leaf.grad.abs().max().item() + 1e-30))


@pytest.mark.parametrize("from_depth", [True, False])
@pytest.mark.parametrize("background", [False, True])
@pytest.mark.parametrize("HW", [(2, 2), (3, 5), (17, 33), (16, 15)])
def test_normal_bounds_hold_an_fp32_evaluation(from_depth, background, HW):
    H, W = HW
    inp = normal_inputs(H, W, from_depth, seed=H + 7 * W, background=background)
    cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
    out = il.normal_consistency(*inp, from_depth, *cam, 0.4 / (H * W), 0.6 / (H * W), shadow=True)
    for k in ("d_normal", "d_e", "d_m"):
        check_shadow(out[k], f"{k}")


def camera(H, W, fovx=0.9, fovy=0.7):
    fx, fy = W / (2 * math.tan(fovx / 2)), H / (2 * math.tan(fovy / 2))
    return 1 / fx, 1 / fy, -W / (2 * fx), -H / (2 * fy)


def normal_inputs(H, W, from_depth, seed, background=False, plane=False):
    """(normal [3,H,W], map_e, map_m): smooth depth (or points), optionally with a zero-depth background behind a silhouette
    (where the cross product vanishes and F.normalize's clamp is active), or an exact plane."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    if plane:
        base = 2.0 + 0.125 * xx + 0.25 * yy
        d1, d2 = base.clone(), base.clone()
    else:
        base = 3.0 + 0.02 * xx + 0.03 * yy + 0.3 * torch.sin(xx * 0.4) * torch.cos(yy * 0.3)
        d1 = base + 0.01 * torch.randn(H, W, generator=g)
        d2 = base + 0.05 * torch.randn(H, W, generator=g)
    if background:
        fg = ((xx - W / 2) ** 2 / max(W / 3, 1) ** 2 + (yy - H / 2) ** 2 / max(H / 3, 1) ** 2) < 1
        d1, d2 = d1 * fg, d2 * fg
    nrm = F.normalize(torch.randn(3, H, W, generator=g), dim=0) * 0.9
    if from_depth:
        return nrm, d1[None].contiguous(), d2[None].contiguous()
    pts = lambda d: torch.stack([(xx - W / 2) * d / 50, (yy - H / 2) * d / 50, d]).contiguous()
    return nrm, pts(d1), pts(d2)
