"""CPU checks of the appearance network's head entry points: the C ABI's host-side rejections (rgs_appearance_head_*, reported
through rgs_last_error before any CUDA call) and the Python wrappers' shape checks, in their order, on CPU tensors."""
import ctypes
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import ROOT


def _lib():
    lib = ctypes.CDLL(os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so"))
    lib.rgs_last_error.restype = ctypes.c_char_p
    return lib


def test_scratch_size_and_rejections():
    lib = _lib()
    n = ctypes.c_size_t(0)
    assert lib.rgs_appearance_head_scratch_bytes(ctypes.c_int32(37), ctypes.c_int32(50), ctypes.byref(n)) == 0
    assert 3072 * 37 * 50 * 4 < n.value <= 3072 * 37 * 50 * 4 + (16 << 20)
    for h, w in ((0, 50), (37, 0), (-1, 3), (1 << 10, 1 << 10)):
        assert lib.rgs_appearance_head_scratch_bytes(ctypes.c_int32(h), ctypes.c_int32(w), ctypes.byref(n)) == -1
        assert b"appearance head" in lib.rgs_last_error()
    assert lib.rgs_appearance_head_scratch_bytes(ctypes.c_int32(2), ctypes.c_int32(3), None) == -1
    assert b"null" in lib.rgs_last_error()


def test_forward_and_backward_reject_bad_sizes_and_null_pointers():
    lib = _lib()
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: rejected before the first CUDA call
    fwd = [ctypes.c_int32(2), ctypes.c_int32(3)] + [fake] * 14 + [None]
    bwd = [ctypes.c_int32(2), ctypes.c_int32(3)] + [fake] * 23 + [None]
    for fn, args in ((lib.rgs_appearance_head_forward, fwd), (lib.rgs_appearance_head_backward, bwd)):
        for bad in (0, -4):
            a = list(args)
            a[0] = ctypes.c_int32(bad)
            assert fn(*a) == -1
            assert b"at least 1" in lib.rgs_last_error()
        for i in range(2, len(args) - 1):   # every pointer but the stream
            a = list(args)
            a[i] = None
            assert fn(*a) == -1, i
            assert b"null" in lib.rgs_last_error()


def _net():
    net = torch.nn.Module()
    for name, cin, cout in (("conv1", 67, 256), ("conv2", 16, 16), ("conv3", 16, 3)):
        setattr(net, name, torch.nn.Conv2d(cin, cout, 3, padding=1))
    for i, (cin, cout) in enumerate(((64, 128), (32, 64), (16, 32), (8, 16)), 1):
        up = torch.nn.Module()
        up.conv = torch.nn.Conv2d(cin, cout, 3, padding=1)
        setattr(net, f"up{i}", up)
    return net


def test_python_shape_checks_in_order():
    """conv2, conv3, then conv1 and up1..up4 (each a GOF shape with a bias), then the embedding row, then the images."""
    from rade_gs_b200 import multigpu
    from rade_gs_b200.appearance import L1_loss_appearance
    table = torch.zeros(4, 64)
    img, gt = torch.rand(3, 40, 50), torch.rand(3, 40, 50)

    def call(net, tab=table, fn="whole"):
        g = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: tab[i])
        if fn == "whole":
            return L1_loss_appearance(img, gt, g, 0)
        return multigpu.slab_L1_loss_appearance(img, gt, g, 0, (0, 40), all_pixel_rows=[(0, 40)])

    for fn in ("whole", "slab"):
        with pytest.raises(RuntimeError, match="no CPU path"):
            call(_net(), fn=fn)
        net = _net()
        net.conv3 = torch.nn.Conv2d(16, 4, 3, padding=1)
        net.conv1 = torch.nn.Conv2d(67, 128, 3, padding=1)
        with pytest.raises(ValueError, match="conv3 must be a 16 -> 3"):          # the tail's checks come first
            call(net, fn=fn)
        net = _net()
        net.conv1 = torch.nn.Conv2d(67, 128, 3, padding=1)
        net.up1.conv = torch.nn.Conv2d(64, 128, 3, padding=1, bias=False)
        with pytest.raises(ValueError, match="conv1 must be a 67 -> 256 3x3 convolution with bias"):
            call(net, fn=fn)
        for i, (cin, cout) in enumerate(((64, 128), (32, 64), (16, 32), (8, 16)), 1):
            net = _net()
            getattr(net, f"up{i}").conv = torch.nn.Conv2d(cin, cout, 3, padding=1, bias=False)
            with pytest.raises(ValueError, match=f"up{i} must be a {cin} -> {cout} 3x3 convolution with bias"):
                call(net, fn=fn)
            net = _net()
            getattr(net, f"up{i}").conv = torch.nn.Conv2d(cin, cout + 1, 3, padding=1)
            with pytest.raises(ValueError, match=f"up{i} must be a {cin} -> {cout}"):
                call(net, fn=fn)
        net = _net()
        del net.up2
        with pytest.raises(ValueError, match="up2 must be"):
            call(net, fn=fn)
        with pytest.raises(ValueError, match="embedding"):                       # before the images' checks
            call(_net(), torch.zeros(4, 32), fn=fn)
