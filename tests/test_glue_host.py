"""Every tensor-taking entry of the torch glue (`diff_gaussian_rasterization._C`) refuses well-shaped CPU tensors with a
RuntimeError that names CUDA, before it touches a device.  No GPU needed.  The exchange's handle entries are left out: they
take integer handles, and `exchange_connect` takes CPU handles by design."""
from types import SimpleNamespace

import pytest
import torch

P, N, H, W = 4, 5, 32, 32
E = torch.Tensor([])  # the rasterizer's "absent" convention
f32 = torch.zeros
f64 = lambda *s: torch.zeros(*s, dtype=torch.float64)
i32 = lambda *s: torch.zeros(*s, dtype=torch.int32)
i64 = lambda *s: torch.zeros(*s, dtype=torch.int64)
u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8)
byte = lambda: torch.zeros(0, dtype=torch.uint8)


def _camera():
    return [torch.eye(4), torch.eye(4), 0.5, 0.5, 0.0]


def _gaussians():  # colors, opacity, scales, rotations, scale_modifier, cov3D_precomp
    return [E, f32(P, 1), f32(P, 3), f32(P, 4), 1.0, E]


def _forward(slab=False, split=False):
    sh = [f32(P, 1, 3), f32(P, 3, 3)] if split else [f32(P, 1, 3)]
    a = [f32(3), f32(P, 3)] + _gaussians() + _camera() + [H, W] + sh + [0, f32(3), False, True, True, False]
    return a + [0, -1, False] if slab else a


def _backward(split=False, render=False, exchange=False):
    sh = [f32(P, 1, 3), f32(P, 3, 3)] if split else [f32(P, 1, 3)]
    g = _gaussians()
    maps = [f32(3, H, W), f32(3, H, W), f32(3, H, W), f32(1, H, W), f32(1, H, W), f32(1, H, W), f32(3, H, W), f32(3, H, W)]
    a = [f32(3), f32(P, 3), i32(P), g[0], g[2], g[3], g[4], g[5]] + _camera() + maps + sh
    a += [0, f32(3), byte(), 0, byte(), byte(), f32(1, H, W), True, True, False]
    if render:
        a += [0, -1]
    return ([1] if exchange else []) + a


def _integrate():
    g = _gaussians()
    return [f32(3), f32(N, 3), f32(P, 3)] + g[:5] + [g[5], E] + _camera() + [E, H, W, f32(P, 1, 3), 0, f32(3), False, False]


def _preprocess():
    g = _gaussians()
    return [f32(P, 16), f32(3), f32(P, 3), i32(P)] + g + _camera() + [H, W, f32(P, 1, 3), 0, f32(3), byte(), True, True, False]


def _grid():
    return SimpleNamespace(voxel_size=0.1, hash_keys=i64(16), hash_values=i32(16), tsdf=f32(4 * 512), weight=f32(4 * 512), color=f32(4 * 512, 3),
                           stamps=i32(4), frame_keys=i64(8), frame_list=i64(8), counters=i32(4))


_K, _T = f64(3, 3), torch.eye(4, dtype=torch.float64)

ENTRIES = {
    "rasterize_gaussians": _forward,
    "rasterize_gaussians_slab": lambda: _forward(slab=True),
    "rasterize_gaussians_split_sh": lambda: _forward(split=True),
    "rasterize_gaussians_backward": _backward,
    "rasterize_gaussians_backward_split_sh": lambda: _backward(split=True),
    "rasterize_gaussians_backward_render": lambda: _backward(render=True),
    "rasterize_gaussians_backward_render_exchange": lambda: _backward(render=True, exchange=True),
    "rasterize_gaussians_backward_preprocess": _preprocess,
    "integrate_gaussians_to_points": _integrate,
    "mark_visible": lambda: [f32(P, 3), torch.eye(4), torch.eye(4)],
    "exchange_rows": lambda: [1, i32(P), i32(P)],
    "compute_3d_filter": lambda: [f32(P, 3), f32(2, 16), 1.0],
    "ssim_l1_forward": lambda: [f32(3, H, W), f32(3, H, W), True],
    "ssim_l1_backward": lambda: [f32(3, H, W), f32(3, H, W), f32(3, 3, H, W), 0.2, 0.8, torch.ones(())],
    "normal_consistency": lambda: [f32(3, H, W), f32(3, H, W), f32(3, H, W), False, 1.0, 1.0, 16.0, 16.0, 1.0, 1.0],
    "appearance_downsample": lambda: [f32(3, 64, 64)],
    "appearance_downsample_backward": lambda: [f32(3, 2, 2), f32(3, 64, 64)],
    "appearance_l1_forward": lambda: [f32(3, 64, 64), f32(3, 64, 64), f32(1, 16, 32, 32), f32(16, 16, 3, 3), f32(16), f32(3, 16, 3, 3), f32(3), True, False],
    "appearance_l1_backward": lambda: [f32(3, 64, 64), f32(3, 64, 64), f32(1, 16, 32, 32), f32(16, 64, 64), f32(16, 16, 3, 3), f32(16), f32(3, 16, 3, 3),
                                       f32(3), torch.ones(())],
    "activate_forward": lambda: [f32(P, 3), f32(P, 1), f32(P, 4), f32(P, 1)],
    "activate_backward": lambda: [f32(P, 3), f32(P, 1), f32(P, 4), f32(P, 1), f32(P, 3), f32(P, 1), f32(P, 4)],
    "densification_stats": lambda: [f32(P, 3), i32(P), f32(P, 1), f32(P, 1), f32(P, 1), f32(P, 1), f32(P)],
    "knn_mean_dist2": lambda: [f32(P, 3)],
    "tsdf_touch": lambda: [_grid(), f32(H, W), _K, _T, 1.0, 3.0, 4.0],
    "tsdf_integrate": lambda: [_grid(), i32(2, 3), f32(H, W), f32(H, W, 3), _K, _T, 1.0, 3.0, 4.0, 1],
    "tsdf_rehash": lambda: [_grid(), i64(16), i32(16)],
    "tsdf_active_blocks": lambda: [_grid()],
    "tsdf_extract": lambda: [_grid(), 0.0],
    "tsdf_vertex_normals": lambda: [f32(N, 3), i32(2, 3)],
    "dtu_sample_mesh": lambda: [f64(N, 3), i32(2, 3), 1.0],
    "dtu_radius_downsample": lambda: [f64(N, 3), 0.1],
    "dtu_nearest": lambda: [f64(N, 3), f64(N, 3)],
    "dtu_dilate_masks": lambda: [u8(2, H, W)],
    "dtu_cull_vertices": lambda: [f64(N, 3), f64(2, 3, 4), u8(2, H, W)],
    "tnt_crop": lambda: [f64(N, 3), _T, 2, -1.0, 1.0, f64(4, 2)],
    "tnt_transform": lambda: [f64(N, 3), _T],
    "tnt_voxel_downsample": lambda: [f64(N, 3), 0.1],
    "tnt_icp_moments": lambda: [f64(N, 3), f64(N, 3), f64(N), i64(N), 0.1],
    "tetra_points": lambda: [f32(P, 3), f32(P, 3), f32(P, 4)],
    "tetra_cull_add": lambda: [f32(N), f32(N, 2), f32(H, W), E, f32(N), i32(N)],
    "tetra_cull_finish": lambda: [f32(N), i32(N)],
    "tetra_marching": lambda: [f32(N, 3), f32(N), f32(N), i64(2, 4)],
    "tetra_bisect": lambda: [f32(N), f32(N, 3), f32(N, 3), f32(N), f32(N), f32(N, 3)],
    "tetra_filter": lambda: [f32(N, 3), f32(N, 2, 3), f32(N, 2), i64(2, 3)],
}


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_cpu_tensors_are_refused_with_a_cuda_message(name):
    import diff_gaussian_rasterization as dgr
    with pytest.raises(RuntimeError, match="CUDA"):
        getattr(dgr._C, name)(*ENTRIES[name]())


def test_every_tensor_entry_is_covered():
    import diff_gaussian_rasterization as dgr
    handles = {"exchange_create", "exchange_connect", "exchange_destroy", "exchange_accumulator", "exchange_result", "exchange_status"}
    scalars = {"grad_stride", "set_poison", "launch_count", "abi_version", "stage_timing", "stage_times"}
    exported = {n for n in dir(dgr._C) if not n.startswith("_")}
    assert exported - handles - scalars == set(ENTRIES)
