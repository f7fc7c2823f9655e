"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol the header declares,
the Python package keeps the reference's surface, and host-side helpers behave.  No GPU, no compute calls."""
import ctypes
import inspect
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT

LIB = os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so")
HEADER = os.path.join(ROOT, "include", "rgs_b200.h")


def _declared_functions():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(rgs_[a-z_0-9]+)\s*\(", text)) - {"rgs_resize_fn"})


def test_library_exports_every_declared_symbol_at_abi_4():
    assert os.path.exists(LIB), "run python rade-gs_b200/build.py"
    lib = ctypes.CDLL(LIB)
    names = _declared_functions()
    assert {"rgs_forward", "rgs_backward", "rgs_backward_render", "rgs_backward_preprocess", "rgs_mark_visible", "rgs_grad_stride",
            "rgs_debug_get_views", "rgs_last_error", "rgs_abi_version", "rgs_launch_count"} <= set(names)
    for n in names:
        assert hasattr(lib, n), n
    lib.rgs_abi_version.restype = ctypes.c_int32
    assert lib.rgs_abi_version() == 4
    lib.rgs_grad_stride.restype = ctypes.c_int32
    assert lib.rgs_grad_stride(0, 0) == 16 and lib.rgs_grad_stride(0, 1) == 16
    assert lib.rgs_grad_stride(1, 0) == 32 and lib.rgs_grad_stride(1, 1) == 32


def test_argument_validation_without_gpu():
    """Errors that are decided on the host come back as negative status + message, never as a crash."""
    lib = ctypes.CDLL(LIB)
    lib.rgs_last_error.restype = ctypes.c_char_p
    lib.rgs_mark_visible.restype = ctypes.c_int32
    assert lib.rgs_mark_visible(ctypes.c_int32(-1), None, None, None, None, None) == -1
    assert b"negative" in lib.rgs_last_error()
    assert lib.rgs_mark_visible(ctypes.c_int32(0), None, None, None, None, None) == 0
    lib.rgs_forward.restype = ctypes.c_int64
    assert lib.rgs_forward(None, None, None, None, None) == -1


def test_host_side_rejections_report_through_rgs_last_error():
    """make_params runs before any CUDA call: more than 16 SH coefficients (the SH kernels stage rows of <= 16 x 3 floats), a slab
    outside the tile grid, prefiltered=True and the exchange's argument checks come back as statuses with messages."""
    lib = ctypes.CDLL(LIB)
    lib.rgs_last_error.restype = ctypes.c_char_p
    lib.rgs_forward.restype = ctypes.c_int64

    class Cam(ctypes.Structure):
        _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float),
                    ("kernel_size", ctypes.c_float), ("scale_modifier", ctypes.c_float), ("viewmatrix", ctypes.c_void_p), ("projmatrix", ctypes.c_void_p),
                    ("cam_pos", ctypes.c_void_p), ("background", ctypes.c_void_p), ("sh_degree", ctypes.c_int32), ("sh_coeffs", ctypes.c_int32),
                    ("require_coord", ctypes.c_int32), ("require_depth", ctypes.c_int32), ("prefiltered", ctypes.c_int32), ("debug", ctypes.c_int32),
                    ("tile_row_begin", ctypes.c_int32), ("tile_row_end", ctypes.c_int32), ("compact_slab", ctypes.c_int32)]

    class Gs(ctypes.Structure):
        _fields_ = [("P", ctypes.c_int32)] + [(n, ctypes.c_void_p) for n in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations",
                                                                             "cov3D_precomp", "shs_rest")]

    fake = ctypes.c_void_p(0x1000)   # never dereferenced: every case below is rejected before the first CUDA call
    out = (ctypes.c_void_p * 8)(*[fake] * 8)
    bufs = (ctypes.c_void_p * 6)(*[fake] * 6)

    def call(**kw):
        cam = Cam(width=64, height=64, tan_fovx=0.5, tan_fovy=0.5, scale_modifier=1.0, sh_degree=3, sh_coeffs=16, tile_row_begin=0, tile_row_end=-1)
        for k, v in kw.items():
            setattr(cam, k, v)
        gs = Gs(P=4, means3D=fake, opacities=fake, shs=fake, scales=fake, rotations=fake)
        return lib.rgs_forward(ctypes.byref(cam), ctypes.byref(gs), out, bufs, None), lib.rgs_last_error()

    rc, msg = call(sh_coeffs=20)
    assert rc == -1 and b"at most 16 SH coefficients" in msg
    rc, msg = call(sh_degree=3, sh_coeffs=9)
    assert rc == -1 and b"sh_degree" in msg
    rc, msg = call(tile_row_begin=3, tile_row_end=99)
    assert rc == -1 and b"slab" in msg
    rc, msg = call(prefiltered=1)
    assert rc == -3 and b"prefiltered" in msg
    ex = ctypes.c_void_p()
    handle = (ctypes.c_char * 64)()
    assert lib.rgs_exchange_create(ctypes.c_int32(3), ctypes.c_int32(2), ctypes.c_int64(10), ctypes.c_int32(16), ctypes.byref(ex), handle) == -1
    assert b"rank / world" in lib.rgs_last_error()
    assert lib.rgs_exchange_create(ctypes.c_int32(0), ctypes.c_int32(2), ctypes.c_int64(10), ctypes.c_int32(17), ctypes.byref(ex), handle) == -1
    assert b"capacity / row size" in lib.rgs_last_error()


def test_python_surface_matches_reference():
    import diff_gaussian_rasterization as dgr
    fields = ("image_height", "image_width", "tanfovx", "tanfovy", "kernel_size", "bg", "scale_modifier", "viewmatrix", "projmatrix",
              "sh_degree", "campos", "prefiltered", "require_depth", "require_coord", "debug")
    assert dgr.GaussianRasterizationSettings._fields == fields  # reference __init__.py:171-186
    sig = inspect.signature(dgr.GaussianRasterizer.forward)
    assert list(sig.parameters)[1:] == ["means3D", "means2D", "opacities", "shs", "colors_precomp", "scales", "rotations", "cov3D_precomp"]
    for sym in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible", "integrate_gaussians_to_points"):
        assert hasattr(dgr._C, sym)  # reference ext.cpp:15-20
    assert hasattr(dgr.GaussianRasterizer, "markVisible") and hasattr(dgr.GaussianRasterizer, "integrate")


def _settings(dgr):
    z = torch.zeros(3)
    return dgr.GaussianRasterizationSettings(32, 32, 0.5, 0.5, 0.0, z, 1.0, torch.eye(4), torch.eye(4), 0, z, False, True, False, False)


def test_exactly_one_of_checks_raise_reference_messages():
    import diff_gaussian_rasterization as dgr
    r = dgr.GaussianRasterizer(_settings(dgr))
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(m, m, torch.ones(4, 1), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair or precomputed 3D covariance"):
        r(m, m, torch.ones(4, 1), colors_precomp=torch.ones(4, 3))
    with pytest.raises(Exception, match="exactly one of"):
        r(m, m, torch.ones(4, 1), colors_precomp=torch.ones(4, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4), cov3D_precomp=torch.ones(4, 6))


def test_no_cpu_fallback():
    """The product path fails loudly on CPU tensors instead of computing something else."""
    import diff_gaussian_rasterization as dgr
    r = dgr.GaussianRasterizer(_settings(dgr))
    m = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        r(m, m, torch.ones(4, 1), colors_precomp=torch.ones(4, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))
    with pytest.raises(RuntimeError, match="num_points, 3"):
        dgr._C.rasterize_gaussians(torch.zeros(3), torch.zeros(4, 2), torch.Tensor([]), torch.ones(4, 1), torch.ones(4, 3), torch.ones(4, 4), 1.0,
                                   torch.Tensor([]), torch.eye(4), torch.eye(4), 0.5, 0.5, 0.0, 32, 32, torch.zeros(4, 1, 3), 0, torch.zeros(3),
                                   False, False, True, False)
    with pytest.raises(RuntimeError, match="no CPU path"):
        r.integrate(m, m, m, torch.ones(4, 1), colors_precomp=torch.ones(4, 3), scales=torch.ones(4, 3), rotations=torch.ones(4, 4))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "rade-gs_b200")
    for dirpath, _, files in os.walk(pkg):
        if "build" in dirpath.split(os.sep):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "liboracle" not in text and "oracle/" not in text.replace("oracle/_ref", "").replace("oracle/glm_shim", ""), f


def test_scene_recipe_is_deterministic_and_calibrated():
    from rade_gs_b200 import scenes
    a = scenes.make_scene(5000, 320, 240, 300.0, -3.6)
    b = scenes.make_scene(5000, 320, 240, 300.0, -3.6)
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        assert torch.equal(getattr(a, k), getattr(b, k))
    assert torch.allclose(a.rotations.norm(dim=1), torch.ones(5000), atol=1e-6)
    assert a.shs.shape == (5000, 16, 3) and a.opacities.shape == (5000, 1)
    # projection matrix equals the reference formula (utils/graphics_utils.py:67-87) in its transposed storage
    P = a.projmatrix
    assert abs(P[0, 0].item() - 1 / a.tanfovx) < 1e-6 and abs(P[1, 1].item() - 1 / a.tanfovy) < 1e-6 and P[2, 3].item() == 1.0
    # a tilted camera keeps the recipe's camera-space distribution
    v = scenes.look_at_view((0.4, -0.3, -0.5), (0.1, 0.05, 6.0))
    c = scenes.make_scene(2000, 320, 240, 300.0, -3.6, view=v)
    cam = c.means3D @ c.viewmatrix[:3, :3] + c.viewmatrix[3, :3]
    assert cam[:, 2].min() > 1.99 and cam[:, 2].max() < 10.01


def test_partition_tile_rows():
    from rade_gs_b200.multigpu import partition_tile_rows, tile_rows
    assert tile_rows(1080) == 68 and tile_rows(1200) == 75
    assert [e - b for b, e in partition_tile_rows(68, 8)] == [9, 9, 9, 9, 8, 8, 8, 8]  # SURVEY.md 8e
    for gy, w in ((75, 1), (75, 2), (75, 4), (75, 8), (3, 8), (0, 2)):
        parts = partition_tile_rows(gy, w)
        assert len(parts) == w and parts[0][0] == 0 and parts[-1][1] == gy
        assert all(parts[i][1] == parts[i + 1][0] for i in range(w - 1))
    weights = [1.0] * 10 + [9.0] * 10
    parts = partition_tile_rows(20, 2, weights)
    assert parts[0][0] == 0 and parts[-1][1] == 20 and parts[0][1] == parts[1][0] and parts[0][1] > 10  # heavy rows split off
    with pytest.raises(ValueError):
        partition_tile_rows(10, 0)
