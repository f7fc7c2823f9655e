"""GPU checks of rade_gs_b200.metrics: every LPIPS stage at every element against fp64 (tests/lpips_f64.py), the whole
score against the reference's fixture and against what the reference computes on the GPU, determinism, and the CLI.

Bounds of the TF32 layers (contract at rgs_lpips_conv3x3 in include/rgs_b200.h).  With S = fp64 conv(|x|, |w|):
  - an input that is not a TF32 value is truncated by the tensor cores: relative error < 2^-10 per product;
  - the weights are rounded to nearest TF32 at load (2^-11), the reference conv uses the unrounded fp32 ones;
  - fp32 accumulation of K = 9 C_in products and the bias: (K + 1) 2^-23 relative to S + |b|, doubled because the
    tensor cores' adder aligns by truncation;
  - output rounding to TF32: 2^-11 |out|.
End to end the kernels are held to 4x the error of the same restatement run in fp32 through cuDNN with TF32 allowed
(torch's default, what the reference computes on the GPU), the maximum of each taken over the case set.  Observed on one
H100 80GB HBM3 at a 700 W power limit: largest error 2.0e-6 for the kernels (the 0/1-saturated 24x20 pair, 3.1e-5
relative) against 1.34e-6 for cuDNN-TF32 (the 17x31 pair): ratio 1.5.  At 1600x1200, 1920x1080 and 979x546 the kernels'
errors are 5.3e-8, 3.7e-8 and 6.5e-8 (cuDNN-TF32: 3.0e-8, 3.1e-8, 3.6e-8), about 2.5e-5 relative.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_f64 as ref

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "metrics", "lpips.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def weights(golden, tmp_path_factory):
    sd = ref.seeded_weights(int(golden["seed"]))
    assert ref.digest(sd) == str(golden["digest"])
    d = tmp_path_factory.mktemp("ckpt")
    torch.save({k: v for k, v in sd.items() if k.startswith("features.")}, d / "vgg16-397923af.pth")
    torch.save({k: v for k, v in sd.items() if k.startswith("lin")}, d / "vgg.pth")
    return sd, str(d / "vgg16-397923af.pth"), str(d / "vgg.pth")


def _L():
    from diff_gaussian_rasterization import _C
    return _C._lpips


def _lp(x, y, w, **kw):
    from rade_gs_b200 import metrics
    return metrics.lpips(x, y, vgg_path=w[1], lin_path=w[2], **kw)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2)


# (C_in, C_out) of the twelve TF32 layers, in trunk order
TF32_LAYERS = [ref.CHANNELS[i] for b in ref.BLOCKS for i in b if i]
SIZES = [(5, 7), (13, 29), (40, 33), (71, 96)]   # narrower than one 128-pixel tile, odd sides, several tiles with a ragged last one


@pytest.mark.parametrize("layer", range(12))
def test_tf32_layer_against_fp64_at_every_element(layer):
    from rade_gs_b200.metrics import round_tf32
    cin, cout = TF32_LAYERS[layer]
    g = torch.Generator().manual_seed(100 + layer)
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
    w[:3] *= 300.0                                   # a few large-magnitude output channels
    b = torch.randn(cout, generator=g) * 0.1
    wk = round_tf32(w.permute(0, 2, 3, 1).contiguous()).cuda()
    K = 9 * cin
    for H, W in SIZES[layer % 2::2] if cin >= 256 else SIZES:
        x = (torch.rand(2, cin, H, W, generator=g) * torch.rand(2, cin, 1, 1, generator=g) * 4).cuda()
        got = _nchw(_L().conv3x3(_nhwc(x), wk, b.cuda())).double()
        xd, wd, bd = x.double(), w.double().cuda(), b.double().cuda()
        exact = F.relu(F.conv2d(xd, wd, bd, padding=1))
        S = F.conv2d(xd.abs(), wd.abs(), None, padding=1) + bd.abs().view(1, -1, 1, 1)
        bound = (2.0 ** -10 + 2.0 ** -11 + 2 * (K + 1) * 2.0 ** -23) * S + 2.0 ** -11 * exact.abs() + 1e-30
        err = (got - exact).abs()
        assert (err <= bound).all(), f"{(cin, cout)} at {H}x{W}: worst err/bound {(err / bound).max().item():.3g}"


def test_tf32_operands_that_are_tf32_values_lose_nothing_but_accumulation():
    from rade_gs_b200.metrics import round_tf32
    g = torch.Generator().manual_seed(5)
    cin, cout, H, W = 64, 128, 19, 23
    x = round_tf32(torch.rand(2, cin, H, W, generator=g))
    w = round_tf32(torch.randn(cout, cin, 3, 3, generator=g) * 0.06)
    b = torch.randn(cout, generator=g) * 0.1
    got = _nchw(_L().conv3x3(_nhwc(x).cuda(), w.permute(0, 2, 3, 1).contiguous().cuda(), b.cuda())).double().cpu()
    exact = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1))
    S = F.conv2d(x.double().abs(), w.double().abs(), None, padding=1) + b.double().abs().view(1, -1, 1, 1)
    assert ((got - exact).abs() <= 2 * (9 * cin + 1) * 2.0 ** -23 * S + 2.0 ** -11 * exact.abs()).all()


@pytest.mark.parametrize("H,W", [(16, 16), (17, 31), (97, 53)])
def test_input_conv_against_fp64_at_every_element(H, W):
    g = torch.Generator().manual_seed(H * W)
    x, y = torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)
    x[:, :3, :3] = 0.0
    y[:, -2:, -4:] = 1.0
    w = torch.randn(64, 3, 3, 3, generator=g) * 0.3
    b = torch.randn(64, generator=g) * 0.1
    got = _nchw(_L().input_conv(x.cuda(), y.cuda(), w.cuda(), b.cuda())).double().cpu()
    z = ref.zscore(torch.stack([x, y]))
    exact = F.relu(F.conv2d(z, w.double(), b.double(), padding=1))
    S = F.conv2d(z.abs(), w.double().abs(), None, padding=1) + b.double().abs().view(1, -1, 1, 1)
    # z in fp32: two roundings (2^-23 |z|); 27 fused products and the bias: 28 2^-24; output rounding to TF32
    assert ((got - exact).abs() <= (2.0 ** -22 + 30 * 2.0 ** -24) * S + 2.0 ** -11 * exact.abs()).all()


@pytest.mark.parametrize("H,W,C", [(2, 2, 64), (17, 31, 64), (40, 33, 128), (9, 6, 256), (5, 7, 512)])
def test_maxpool_is_bit_equal_to_torch(H, W, C):
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(2, H, W, C, generator=g).relu()
    x[0, 0, 0, :8] = -0.0
    got = _L().maxpool(x.cuda()).cpu()
    want = _nhwc(F.max_pool2d(_nchw(x).cuda(), 2)).cpu()
    assert got.shape == want.shape and torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("H,W,C", [(16, 16, 64), (33, 20, 128), (7, 129, 256), (8, 11, 512)])
def test_distance_against_fp64_at_every_pixel_and_the_layer_mean(H, W, C):
    g = torch.Generator().manual_seed(C * H)
    f = torch.randn(2, C, H, W, generator=g).relu() * torch.rand(1, C, 1, 1, generator=g) * 3
    f[:, :, 0, 0] = 0.0                               # a zero vector: the 1e-10 guard
    lin = torch.rand(C, generator=g) * 0.1
    m, mean = _L().distance(_nhwc(f).cuda(), lin.cuda())
    fd = f.double()
    exact = ref.head_map(fd[:1], fd[1:], lin.double())[0]
    nx = fd[:1].pow(2).sum(1, keepdim=True).sqrt() + 1e-10
    ny = fd[1:].pow(2).sum(1, keepdim=True).sqrt() + 1e-10
    T = ((fd[:1] / nx).abs() + (fd[1:] / ny).abs()).pow(2).mul(lin.double().view(1, -1, 1, 1)).sum(1)[0]
    bound = (C + 16) * 2.0 ** -23 * T
    assert ((m.double().cpu() - exact).abs() <= bound).all()
    assert abs(mean.item() - exact.mean().item()) <= bound.mean().item() + 1e-15


def _cases(golden):
    out = [(str(n), torch.from_numpy(golden[f"{n}/x"]), torch.from_numpy(golden[f"{n}/y"])) for n in golden["names"]]
    g = torch.Generator().manual_seed(3)
    for H, W in [(546, 979), (1080, 1920), (1200, 1600)]:
        yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        base = 0.5 + 0.35 * torch.sin(xx / 23.0 + torch.arange(3).view(3, 1, 1)) * torch.cos(yy / 31.0)
        x = (base + 0.05 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
        out.append((f"{H}x{W}", x, (base + 0.05 * torch.randn(3, H, W, generator=g)).clamp(0, 1)))
    return out


def test_end_to_end_against_fp64_and_the_cudnn_tf32_restatement(golden, weights):
    sd = weights[0]
    ours_err, tf32_err, rows = [], [], []
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        for name, x, y in _cases(golden):
            if f"{name}/total_f64" in golden:
                exact = float(golden[f"{name}/total_f64"])
                exact_layers = golden[f"{name}/layers_f64"]
                mine = ref.layer_means(x.double(), y.double(), sd)
                assert np.allclose([v.item() for v in mine], exact_layers, rtol=1e-12, atol=1e-18)
            else:
                exact = ref.lpips(x.cuda().double(), y.cuda().double(), sd).item()
            with torch.no_grad():
                cudnn = ref.lpips(x.cuda(), y.cuda(), sd, dtype=torch.float32).item()
            got = _lp(x.cuda(), y.cuda(), weights).item()
            ours_err.append(abs(got - exact))
            tf32_err.append(abs(cudnn - exact))
            rows.append(f"{name}: fp64 {exact:.10g} ours {got:.10g} (err {ours_err[-1]:.3g}) cudnn-tf32 err {tf32_err[-1]:.3g}")
    finally:
        torch.backends.cudnn.allow_tf32 = old
    print("\n".join(rows))
    print(f"max error: ours {max(ours_err):.3g}, cudnn-tf32 {max(tf32_err):.3g}, ratio {max(ours_err) / max(tf32_err):.3g}")
    assert max(ours_err) <= 4 * max(tf32_err)


def test_identical_images_score_exactly_zero_and_repeat_bit_for_bit(weights):
    g = torch.Generator().manual_seed(9)
    x, y = torch.rand(3, 70, 91, generator=g).cuda(), torch.rand(3, 70, 91, generator=g).cuda()
    assert _lp(x, x, weights).item() == 0.0
    a, la = _lp(x, y, weights, layers=True)
    b, lb = _lp(x, y, weights, layers=True)
    assert a.shape == (1, 1, 1, 1) and a.dtype == torch.float32 and a.grad_fn is None
    assert torch.equal(a, b) and torch.equal(la, lb)


def test_poisoned_memory_and_a_late_side_stream_change_nothing(weights):
    from diff_gaussian_rasterization import _C
    g = torch.Generator().manual_seed(10)
    x, y = torch.rand(3, 131, 77, generator=g), torch.rand(3, 131, 77, generator=g)
    ref_total, ref_layers = _lp(x.cuda(), y.cuda(), weights, layers=True)
    ref_total, ref_layers = ref_total.cpu(), ref_layers.cpu()
    _C.set_poison(0x7f)
    try:
        s = torch.cuda.Stream()
        xc, yc = x.cuda(), y.cuda()
        torch.cuda._sleep(20_000_000)
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(s):
            s.wait_event(ev)
            late_total, late_layers = _lp(xc, yc, weights, layers=True)
            late_total, late_layers = late_total.cpu(), late_layers.cpu()
        s.synchronize()
    finally:
        _C.set_poison(-1)
    assert torch.equal(late_total, ref_total) and torch.equal(late_layers, ref_layers)


def test_cli_reproduces_the_reference_json(golden, weights, tmp_path):
    from PIL import Image
    scene = tmp_path / "scene"
    for sub in ("renders", "gt"):
        (scene / "test" / "ours_1" / sub).mkdir(parents=True)
    for n in golden["names"]:
        n = str(n)
        if bool(golden[f"{n}/png"]):
            for sub, key in (("renders", "x"), ("gt", "y")):
                a = np.round(golden[f"{n}/{key}"].transpose(1, 2, 0) * 255).astype(np.uint8)
                Image.fromarray(a).save(scene / "test" / "ours_1" / sub / f"{n}.png")
    hub = tmp_path / "hub" / "checkpoints"
    hub.mkdir(parents=True)
    for f in (weights[1], weights[2]):
        os.symlink(f, hub / os.path.basename(f))
    code = ("import sys, runpy, torch; sys.path.insert(0, %r); torch.hub.set_dir(%r); sys.argv = ['metrics'] + sys.argv[1:]; "
            "runpy.run_module('rade_gs_b200.metrics', run_name='__main__')") % (os.path.join(os.path.dirname(HERE), "rade-gs_b200"), str(tmp_path / "hub"))
    r = subprocess.run([sys.executable, "-c", code, "-m", str(scene)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    # the LPIPS bar of the end-to-end test on these views: 4x the largest error of the cuDNN-TF32 restatement against fp64
    views = [str(n) for n in golden["names"] if bool(golden[f"{n}/png"])]
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        with torch.no_grad():
            bar = 4 * max(abs(ref.lpips(torch.from_numpy(golden[f"{n}/x"]).cuda(), torch.from_numpy(golden[f"{n}/y"]).cuda(), weights[0],
                                        dtype=torch.float32).item() - float(golden[f"{n}/total_f64"])) for n in views)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    exact = {n + ".png": float(golden[f"{n}/total_f64"]) for n in views}
    lp = json.loads((scene / "per_view.json").read_text())["ours_1"]["LPIPS"]
    assert lp.keys() == exact.keys()
    assert max(abs(lp[k] - exact[k]) for k in exact) <= bar
    for f in ("results.json", "per_view.json"):
        text = (scene / f).read_text()
        want_text = str(golden[f])
        got, want = json.loads(text), json.loads(want_text)
        assert text.splitlines()[1].startswith(" \"") == want_text.splitlines()[1].startswith(" \"")   # indent=True: one space
        assert got.keys() == want.keys()
        for method in want:
            assert got[method].keys() == want[method].keys()
            for metric in want[method]:
                g_, w_ = got[method][metric], want[method][metric]
                if isinstance(w_, dict):
                    assert g_.keys() == w_.keys()
                    pairs = [(g_[k], w_[k]) for k in w_]
                else:
                    pairs = [(g_, w_)]
                for a, b in pairs:
                    if np.isinf(b):
                        assert a == b
                    elif metric == "LPIPS":
                        assert abs(a - b) <= bar + 1e-5 * abs(b), (method, metric, a, b)   # the reference's own fp32 error on top
                    else:
                        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (method, metric, a, b)
