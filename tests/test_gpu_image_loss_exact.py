"""The fused image-loss kernels at every pixel against the fp64 models of tests/image_loss_f64.py: both image sums, the three
planes of `dmaps`, every pixel of d_img, the normal-consistency loss and every pixel of its three gradients, each within its
own bound, no outlier budget.

Shapes straddle the kernels' tiles (32 x 16 for SSIM, 16 x 16 for the normals) and fall below the 11-pixel window and the
3-pixel stencil; images are identical, constant, bright and nearly identical, saturated and random; row ranges start and
end off the tile rows; depth maps have zero-depth backgrounds, where F.normalize's clamp is active."""
import pytest
import torch

import image_loss_f64 as il
from f32_error import U, check
from test_image_loss_f64_host import KINDS, camera, images, normal_inputs

pytestmark = pytest.mark.gpu

WORST = {}


def _record(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


def _check_sum(got, vb, name):
    v, e = vb
    err = abs(float(got) - v.item())
    assert err <= e.item() * (1 + 1e-6), f"{name}: {float(got)!r} vs fp64 {v.item()!r}, bound {e.item():.3g}"
    _record(name, err / e.item() if e.item() > 0 else 0.0)


def _ssim_case(img, gt, row_lo=0, row_hi=None, w=(-0.2, 0.8), upstream=None, tag=""):
    from diff_gaussian_rasterization import _C

    H = img.shape[-2]
    hi = H if row_hi is None else row_hi
    a, b = img.cuda(), gt.cuda()
    sums, dmaps = _C.ssim_l1_forward(a, b, True, row_lo, hi)
    fw = il.ssim_l1_forward(img, gt, row_lo, hi, device="cuda")
    _check_sum(sums[0], fw["sums"][0], "ssim sum")
    _check_sum(sums[1], fw["sums"][1], "l1 sum")
    r = fw["rows"]
    for i, name in enumerate(("dmaps d/d mu1", "dmaps d/d E[x^2]", "dmaps d/d E[xy]")):
        _record(name, check(dmaps[i][:, r], fw["dmaps"][i][:, r], f"{tag} {name}"))
    up = None if upstream is None else torch.tensor([upstream], device="cuda")
    d = _C.ssim_l1_backward(a, b, dmaps, w[0], w[1], up if up is not None else torch.empty(0), row_lo, hi)
    model = il.ssim_l1_backward(fw, w[0], w[1], upstream)
    _record("d_img", check(d.reshape(model.v.shape), model, f"{tag} d_img"))
    # need_grad = False: no maps, the sums within the same bounds (the fp64 atomics across CTAs may add in another order)
    s2, dm2 = _C.ssim_l1_forward(a, b, False, row_lo, hi)
    assert dm2.numel() == 0
    _check_sum(s2[0], fw["sums"][0], "ssim sum")
    _check_sum(s2[1], fw["sums"][1], "l1 sum")


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("H", [1, 5, 15, 16, 17])
@pytest.mark.parametrize("W", [1, 5, 31, 32, 33, 101])
def test_ssim_l1_every_pixel_within_bound(C, H, W):
    for kind in KINDS:
        img, gt = images(kind, (C, H, W), 100 * H + W + C)
        _ssim_case(img, gt, tag=f"{kind} {C}x{H}x{W}")


@pytest.mark.parametrize("rows", [(0, 1), (7, 8), (15, 16), (16, 17), (36, 37), (0, 21), (5, 37), (13, 30), (0, 37)])
def test_ssim_l1_row_ranges_within_bound(rows):
    for kind in ("random", "identical", "bright_close"):
        img, gt = images(kind, (3, 37, 45), 9)
        _ssim_case(img, gt, *rows, w=(-0.3, 0.7), upstream=1.7, tag=f"{kind} rows {rows}")


def test_ssim_l1_batched_input_within_bound():
    img, gt = images("random", (1, 3, 33, 47), 4)
    _ssim_case(img, gt, upstream=-0.4, tag="[1,3,H,W]")


def test_ssim_l1_full_image_within_bound():
    img, gt = images("random", (3, 1200, 1600), 12)
    _ssim_case(img, gt, w=(-0.2 / img.numel(), 0.8 / img.numel()), tag="1600x1200")


@pytest.mark.parametrize("lam", [0.2, 1.0])
def test_l1_ssim_loss_through_autograd_within_bound(lam):
    from rade_gs_b200 import losses

    for kind in KINDS:
        img, gt = images(kind, (3, 19, 37), 3)
        a = img.cuda().requires_grad_(True)
        loss = losses.l1_ssim_loss(a, gt.cuda(), lam)
        (loss * 1.3).backward()
        n = img.numel()
        fw = il.ssim_l1_forward(img, gt, device="cuda")
        ws, wl = -lam / n, (1 - lam) / n
        (vs, es), (vl, el) = fw["sums"]
        v = lam + ws * vs + wl * vl
        e = abs(ws) * es + abs(wl) * el + U * (abs(v) + 1.0) * 4   # the fp64 combination and its rounding to fp32
        assert abs(loss.item() - v.item()) <= e.item(), (kind, loss.item(), v.item(), e.item())
        model = il.ssim_l1_backward(fw, ws, wl, 1.3)
        _record("d_img", check(a.grad, R_view(model, a.grad.shape), f"l1_ssim_loss {kind} d_img"))


def R_view(r, shape):
    from f32_error import R
    return R(r.v.reshape(shape), r.e.reshape(shape))


# ---- normal consistency ----------------------------------------------------------------------------------------------------

def _normal_case(H, W, from_depth, background, plane, ratio, tag):
    from diff_gaussian_rasterization import _C

    inp = normal_inputs(H, W, from_depth, seed=H * 41 + W, background=background, plane=plane)
    cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
    w_e, w_m = (1 - ratio) / (H * W), ratio / (H * W)
    loss, dn, de, dm = _C.normal_consistency(*(t.cuda() for t in inp), from_depth, *cam, w_e, w_m)
    out = il.normal_consistency(*inp, from_depth, *cam, w_e, w_m, device="cuda")
    _check_sum(loss[0], out["loss"], "normal loss")
    for name, got in (("d_normal", dn), ("d_e", de), ("d_m", dm)):
        _record(name, check(got.reshape(out[name].v.shape), out[name], f"{tag} {name}"))
    return out


@pytest.mark.parametrize("from_depth", [True, False])
@pytest.mark.parametrize("H", [1, 2, 3, 15, 16, 17, 33])
@pytest.mark.parametrize("W", [1, 2, 3, 15, 16, 17, 33])
def test_normal_consistency_every_pixel_within_bound(from_depth, H, W):
    for background in (False, True):
        _normal_case(H, W, from_depth, background, False, 0.6, f"{H}x{W} depth={from_depth} background={background}")


@pytest.mark.parametrize("ratio", [0.0, 0.6, 1.0])
@pytest.mark.parametrize("from_depth", [True, False])
def test_normal_consistency_plane_and_ratios_within_bound(ratio, from_depth):
    _normal_case(37, 53, from_depth, False, True, ratio, f"plane ratio={ratio}")
    out = _normal_case(40, 70, from_depth, True, False, ratio, f"silhouette ratio={ratio}")
    if ratio < 1.0:
        # the silhouettes put stencils on F.normalize's clamp: there the gradients are of order w / 1e-12
        assert out["d_e"].v.abs().amax().item() > 1e6 * (1 - ratio) / (40 * 70)


def test_depth_normal_consistency_loss_within_bound():
    from types import SimpleNamespace

    from rade_gs_b200 import losses

    H, W = 33, 47
    inp = normal_inputs(H, W, True, seed=5, background=True)
    view = SimpleNamespace(FoVx=0.9, FoVy=0.7)
    leaves = [t.cuda().requires_grad_(True) for t in inp]
    v = losses.depth_normal_consistency_loss(view, *leaves)
    v.backward()
    out = il.normal_consistency(*inp, True, *camera(H, W), 0.4 / (H * W), 0.6 / (H * W), device="cuda")
    lv, le = out["loss"]
    assert abs(v.item() - lv.item()) <= le.item() + U * abs(lv.item()) * 2
    for name, leaf in (("d_normal", leaves[0]), ("d_e", leaves[1]), ("d_m", leaves[2])):
        _record(name, check(leaf.grad, R_view(out[name], leaf.grad.shape), f"loss {name}"))


def test_report_worst_ratios():
    """Runs last in this module: the worst error / bound ratio per output over the tests above."""
    print("\nimage-loss worst error/bound:", {k: f"{v:.3g}" for k, v in sorted(WORST.items())})
