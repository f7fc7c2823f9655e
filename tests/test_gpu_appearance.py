"""The fused decoupled-appearance L1 loss (rade_gs_b200.appearance) on the GPU: against the reference's own function
(tests/golden/fused_appearance.npz, fp32 and fp64 runs), against the reference expression run eagerly on the GPU in fp64 at the
recipes' image sizes, and through a training iteration.  The bar is test_fused_golden._close: ours vs fp64 within 4x the
reference's own fp32 error plus a small absolute bar."""
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import appearance_f64 as af
from conftest import GOLDEN_DIR
from test_fused_golden import _close

pytestmark = pytest.mark.gpu
DEV = "cuda"


class _Up(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.pixel_shuffle = nn.PixelShuffle(2)
        self.conv = nn.Conv2d(cin // 4, cout, 3, padding=1)
        self.relu = nn.ReLU()

    def forward(self, x):
        return self.relu(self.conv(self.pixel_shuffle(x)))


class _Net(nn.Module):
    """The architecture of scene/appearance_network.py (same layer names and parameter order)."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(67, 256, 3, padding=1)
        self.up1, self.up2, self.up3, self.up4 = _Up(256, 128), _Up(128, 64), _Up(64, 32), _Up(32, 16)
        self.conv2 = nn.Conv2d(16, 16, 3, padding=1)
        self.conv3 = nn.Conv2d(16, 3, 3, padding=1)
        self.relu = nn.ReLU()
        self.sigmoid = nn.Sigmoid()

    def forward(self, x):
        x = self.up4(self.up3(self.up2(self.up1(self.relu(self.conv1(x))))))
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        return self.sigmoid(self.conv3(self.relu(self.conv2(x))))


def _ref_loss(image, gt_image, gaussians, view_idx, return_transformed_image=False):
    """train.py:37-58 restated."""
    emb = gaussians.get_apperance_embedding(view_idx)
    H0, W0 = image.shape[1:]
    H, W = H0 // 32 * 32, W0 // 32 * 32
    left, top = W0 // 2 - W // 2, H0 // 2 - H // 2
    crop, crop_gt = image[:, top:top + H, left:left + W], gt_image[:, top:top + H, left:left + W]
    down = F.interpolate(crop[None], size=(H // 32, W // 32), mode="bilinear", align_corners=True)[0]
    down = torch.cat([down, emb[None].repeat(H // 32, W // 32, 1).permute(2, 0, 1)], dim=0)[None]
    t = gaussians.appearance_network(down) * crop
    if return_transformed_image:
        return F.interpolate(t, size=(H0, W0), mode="bilinear", align_corners=True)[0]
    return torch.abs(t - crop_gt).mean()


def _setup(inp, dtype=torch.float32):
    net = _Net().to(DEV, dtype)
    with torch.no_grad():
        for p, v in zip(net.parameters(), inp["params"]):
            p.copy_(torch.as_tensor(v))
    table = nn.Parameter(torch.as_tensor(inp["table"]).to(DEV, dtype))
    g = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: table[i], table=table)
    image = torch.as_tensor(inp["image"]).to(DEV, dtype).requires_grad_(True)
    gt = torch.as_tensor(inp["gt"]).to(DEV, dtype)
    return g, image, gt


def _run(fn, inp, dtype=torch.float32, idx=af.VIEW_IDX):
    g, image, gt = _setup(inp, dtype)
    loss = fn(image, gt, g, idx)
    loss.backward()
    with torch.no_grad():
        tr = fn(image, gt, g, idx, return_transformed_image=True)
    return {"loss": loss.item(), "d_image": image.grad.cpu().numpy(), "d_emb": g.table.grad[idx].cpu().numpy(), "transformed": tr.cpu().numpy(),
            "grads": [p.grad.cpu().numpy() for p in g.appearance_network.parameters()], "table_grad": g.table.grad.cpu().numpy()}


@pytest.fixture
def no_tf32():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


@pytest.fixture
def exact_head():
    """The fixture's fp32 run is the reference on the CPU.  At the fixtures' 1x2 .. 3x4 head resolutions cuDNN may pick
    Winograd / FFT algorithms whose fp32 error (~1e-4) would swamp the kernels' own; torch's native convolution keeps the head
    at plain fp32 accuracy, so the comparison measures the fused part."""
    old = torch.backends.cudnn.enabled
    torch.backends.cudnn.enabled = False
    yield
    torch.backends.cudnn.enabled = old


def _check_all(ours, r32, r64, sub=lambda name, a: a):
    failures = []
    checks = [(k, sub(k, ours[k]), r32[k], r64[k]) for k in ("loss", "d_image", "d_emb", "transformed")]
    checks += [(n, sub(n, o), a, b) for n, o, a, b in zip(af.PARAM_NAMES, ours["grads"], r32["grads"], r64["grads"])]
    for name, o, a, b in checks:
        try:
            _close(o, a, b, name, 2e-6)
        except AssertionError as e:
            failures.append(str(e).split("\n")[0])
    assert not failures, failures


@pytest.mark.parametrize("case", list(af.CASES))
def test_fixture_parity(case, no_tf32, exact_head):
    from rade_gs_b200.appearance import L1_loss_appearance
    d = af.load_fixture(os.path.join(GOLDEN_DIR, "fused_appearance.npz"))[case]
    inp = af.make_inputs(case)
    assert af.inputs_digest(inp) == str(d["digest"])
    ours = _run(L1_loss_appearance, inp)
    r32 = {k: d[k] for k in ("loss", "d_image", "d_emb", "transformed")}
    r64 = {k: d[k + "_f64"] for k in r32}
    r32["grads"] = [d["g_" + n] for n in af.PARAM_NAMES]
    r64["grads"] = [d["g_" + n + "_f64"] for n in af.PARAM_NAMES]
    _check_all(ours, r32, r64, sub=af.recorded)


def _recipe_inputs(H0, W0, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H0, W0, generator=g)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=g)).clamp(0, 1)
    params = [torch.randn(*s, generator=g) * (2.0 / (s[1] * 9)) ** 0.5 if len(s) == 4 else 0.05 * torch.randn(*s, generator=g) for s in af.PARAM_SHAPES]
    return {"image": image, "gt": gt, "table": 0.5 * torch.randn(8, 64, generator=g), "params": params}


@pytest.mark.parametrize("H0,W0", [(600, 800), (546, 979), (1200, 1600)])
def test_recipe_sizes_against_fp64_eager(H0, W0, no_tf32):
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = _recipe_inputs(H0, W0, H0 + W0)
    ours = _run(L1_loss_appearance, inp)
    r32 = _run(_ref_loss, inp)
    r64 = _run(_ref_loss, inp, torch.float64)
    _check_all(ours, r32, r64)


@pytest.fixture
def deterministic_head():
    """The head's gradients come from cuDNN, whose backward algorithms may accumulate in any order unless told otherwise."""
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


def test_gradient_is_zero_outside_the_crop_and_calls_are_bit_identical(deterministic_head):
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = af.make_inputs("odd_offsets")
    a, b = _run(L1_loss_appearance, inp), _run(L1_loss_appearance, inp)
    top, left, H, W = af.crop_box(*inp["image"].shape[1:])
    out = a["d_image"].copy()
    out[:, top:top + H, left:left + W] = 0
    assert not out.any()
    assert a["loss"] == b["loss"]
    for k in ("d_image", "d_emb", "transformed"):
        assert np.array_equal(a[k], b[k]), k
    for x, y in zip(a["grads"], b["grads"]):
        assert np.array_equal(x, y)


def test_two_calls_accumulate_and_only_the_view_row_gets_a_gradient(deterministic_head):
    """loss + 0.5 * loss: the second call's gradients are exactly half the first's (a power-of-two upstream), so .grad must hold
    1.5x one call's gradients up to the rounding of one addition."""
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = af.make_inputs("ragged_tiles")
    one = _run(L1_loss_appearance, inp)
    g, image, gt = _setup(inp)
    (L1_loss_appearance(image, gt, g, af.VIEW_IDX) + 0.5 * L1_loss_appearance(image, gt, g, af.VIEW_IDX)).backward()
    pairs = [("d_image", image.grad, one["d_image"])] + [(n, p.grad, r) for n, p, r in zip(af.PARAM_NAMES, g.appearance_network.parameters(), one["grads"])]
    for name, got, ref in pairs:
        err = np.abs(got.cpu().numpy() - 1.5 * ref).max()
        assert err <= 1e-6 * np.abs(ref).max(), (name, err, np.abs(ref).max())
    rows = g.table.grad.abs().sum(dim=1).cpu().numpy()
    assert rows[af.VIEW_IDX] > 0 and not np.delete(rows, af.VIEW_IDX).any()


def test_error_paths():
    from rade_gs_b200.appearance import L1_loss_appearance
    g, image, gt = _setup(af.make_inputs("odd_offsets"))
    with pytest.raises(RuntimeError, match="no CPU path"):
        L1_loss_appearance(image.detach().cpu(), gt.cpu(), g, 0)
    with pytest.raises(ValueError, match="ground truth"):
        L1_loss_appearance(image, gt.clone().requires_grad_(True), g, 0)
    with pytest.raises(ValueError, match="H, W >= 32"):
        L1_loss_appearance(image[:, :31], gt[:, :31], g, 0)
    g.appearance_network.conv3 = nn.Conv2d(16, 4, 3, padding=1).to(DEV)
    with pytest.raises(ValueError, match="conv3"):
        L1_loss_appearance(image, gt, g, 0)


def test_training_iteration_with_rasterizer_and_ssim():
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import fused, losses, scenes
    from rade_gs_b200.appearance import L1_loss_appearance
    from test_gpu_api import _settings

    sc = scenes.make_scene(20_000, 320, 240, 280.0, -2.6, seed=5).to(DEV)
    settings = _settings(dgr, sc, False, True, ks=0.1)
    P = sc.means3D.shape[0]
    filt = torch.full((P, 1), 1e-3, device=DEV)
    inp = _recipe_inputs(240, 320, 99)
    results = []
    for impl in (L1_loss_appearance, _ref_loss):
        m = {"xyz": sc.means3D.clone().requires_grad_(True), "scaling": torch.log(sc.scales).requires_grad_(True),
             "opacity": torch.logit(sc.opacities.clamp(1e-4, 1 - 1e-4)).requires_grad_(True), "rotation": sc.rotations.clone().requires_grad_(True),
             "f_dc": sc.shs[:, :1].contiguous().requires_grad_(True), "f_rest": sc.shs[:, 1:].contiguous().requires_grad_(True)}
        g, _, gt = _setup(inp)
        opt = torch.optim.Adam([{"params": [t], "lr": 1e-3} for t in m.values()] + [{"params": [g.table], "lr": 1e-3},
                                                                                   {"params": g.appearance_network.parameters(), "lr": 1e-3}], eps=1e-15)
        s, o, r = fused.activate_gaussians(m["scaling"], m["opacity"], m["rotation"], filt)
        image = dgr.GaussianRasterizer(settings)(means3D=m["xyz"], means2D=torch.zeros_like(m["xyz"]), opacities=o, shs=(m["f_dc"], m["f_rest"]),
                                                 scales=s, rotations=r)[0]
        loss = 0.8 * impl(image, gt, g, 3) + 0.2 * (1.0 - losses.ssim(image, gt))
        opt.zero_grad(set_to_none=True)
        loss.backward()
        for group in opt.param_groups:
            for t in group["params"]:
                assert t.grad is not None and torch.isfinite(t.grad).all()
        results.append({k: t.grad.clone() for k, t in m.items()})
        opt.step()
        assert math.isfinite(loss.item())
    for k in results[0]:
        a, b = results[0][k].double(), results[1][k].double()
        assert (a - b).norm() <= 1e-2 * b.norm(), (k, ((a - b).norm() / b.norm()).item())
