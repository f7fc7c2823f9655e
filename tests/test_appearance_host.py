"""CPU checks of the decoupled-appearance L1 loss: the fp64 model in the kernels' decomposition (tests/appearance_f64.py) against
the reference's own function run in float64 (tests/golden/fused_appearance.npz), and the wrapper's argument rejections."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import appearance_f64 as af
from conftest import GOLDEN_DIR

FIXTURE = os.path.join(GOLDEN_DIR, "fused_appearance.npz")


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-300)


@pytest.mark.parametrize("case", list(af.CASES))
def test_f64_model_reproduces_the_reference_in_float64(case):
    d = af.load_fixture(FIXTURE)[case]
    inp = af.make_inputs(case)
    assert af.inputs_digest(inp) == str(d["digest"]), "the regenerated inputs differ from the fixture's"
    m = af.forward_backward(inp["image"], inp["gt"], inp["table"][af.VIEW_IDX], inp["params"])
    for key in ("loss", "d_image", "d_emb", "transformed"):
        assert _rel(af.recorded(key, m[key]), d[key + "_f64"]) < 1e-10, key
    for name, g in zip(af.PARAM_NAMES, m["grads"]):
        assert _rel(af.recorded(name, g), d["g_" + name + "_f64"]) < 1e-10, name
    # the fixture's float32 run is a distinct evaluation: it sits at fp32 noise from float64, not at zero
    assert 1e-9 < _rel(d["d_image"], d["d_image_f64"]) < 1e-5


@pytest.mark.parametrize("case", list(af.CASES))
def test_fixture_cases_keep_every_relu_input_away_from_zero(case):
    assert af.relu_margin(af.make_inputs(case)) > af.RELU_MARGIN


def test_zero_outside_the_crop_and_one_sample_axis_in_the_model():
    inp = af.make_inputs("one_sample_axis")
    m = af.forward_backward(inp["image"], inp["gt"], inp["table"][af.VIEW_IDX], inp["params"])
    top, left, H, W = af.crop_box(*inp["image"].shape[1:])
    outside = m["d_image"].copy()
    outside[:, top:top + H, left:left + W] = 0
    assert not outside.any() and H == 32


def _net(conv3_out=3):
    net = torch.nn.Module()
    for name, cin, cout in (("conv1", 67, 256), ("conv2", 16, 16), ("conv3", 16, conv3_out)):
        setattr(net, name, torch.nn.Conv2d(cin, cout, 3, padding=1))
    for i, (cin, cout) in enumerate(((64, 128), (32, 64), (16, 32), (8, 16)), 1):
        up = torch.nn.Module()
        up.conv = torch.nn.Conv2d(cin, cout, 3, padding=1)
        setattr(net, f"up{i}", up)
    return net


def test_wrapper_rejections_without_gpu():
    from rade_gs_b200.appearance import L1_loss_appearance
    table = torch.zeros(4, 64)
    g = SimpleNamespace(appearance_network=_net(), get_apperance_embedding=lambda i: table[i])
    img, gt = torch.rand(3, 40, 50), torch.rand(3, 40, 50)
    with pytest.raises(RuntimeError, match="no CPU path"):
        L1_loss_appearance(img, gt, g, 0)
    with pytest.raises(ValueError, match="ground truth"):
        L1_loss_appearance(img, gt.clone().requires_grad_(True), g, 0)
    with pytest.raises(ValueError, match="H, W >= 32"):
        L1_loss_appearance(torch.rand(3, 31, 64), torch.rand(3, 31, 64), g, 0)
    with pytest.raises(ValueError, match="conv3 must be a 16 -> 3"):
        L1_loss_appearance(img, gt, SimpleNamespace(appearance_network=_net(4), get_apperance_embedding=g.get_apperance_embedding), 0)
    bad = _net()
    bad.conv2 = torch.nn.Conv2d(16, 16, 5, padding=2)
    with pytest.raises(ValueError, match="conv2 must be a 16 -> 16"):
        L1_loss_appearance(img, gt, SimpleNamespace(appearance_network=bad, get_apperance_embedding=g.get_apperance_embedding), 0)


def test_c_abi_rejects_small_images_and_null_pointers():
    import ctypes
    from conftest import ROOT
    lib = ctypes.CDLL(os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so"))
    lib.rgs_last_error.restype = ctypes.c_char_p
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: rejected before the first CUDA call
    assert lib.rgs_appearance_downsample(ctypes.c_int32(31), ctypes.c_int32(64), fake, fake, None) == -1
    assert b"at least 32" in lib.rgs_last_error()
    assert lib.rgs_appearance_downsample(ctypes.c_int32(64), ctypes.c_int32(64), None, fake, None) == -1
    assert b"null" in lib.rgs_last_error()
    args = [ctypes.c_int32(64), ctypes.c_int32(64)] + [fake] * 16 + [None]
    args[5] = None   # image, gt, up4, act, w2 (NULL)
    assert lib.rgs_appearance_l1_backward(*args) == -1
