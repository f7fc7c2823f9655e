"""Slab-local normal consistency on CPU (gloo, 2 and 3 ranks): the control flow of rade_gs_b200.multigpu's
`slab_depth_normal_consistency_loss` / `slab_point_normal_consistency_loss` -- halo exchange, the all-reduced loss, gradients
placed in the rank's rows -- with an fp64 torch restatement of the reference's expressions (train.py:141-156,
utils/graphics_utils.py:97-126) standing in for the CUDA kernel.  The slabs must give the whole image's loss and, on each rank's
rows, the whole image's gradients.  No GPU."""
import math
import os
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

FOV = (0.9, 0.7)
DEPTH_RATIO = 0.6


def _points_from_depth(d, rows, W, inv_fx, inv_fy, cx, cy):
    """depths_double_to_points on image rows `rows` (global indices): depth * K^-1 (x + 0.5, y + 0.5, 1)."""
    gy = rows.to(d.dtype)[:, None] + 0.5
    gx = torch.arange(W, dtype=d.dtype)[None, :] + 0.5
    rx, ry = (inv_fx * gx + cx).expand(len(rows), W), (inv_fy * gy + cy).expand(len(rows), W)
    return torch.stack([d[0] * rx, d[0] * ry, d[0]])


def _normals(p, rows, H):
    """point_double_to_normal on a window of rows (global indices `rows`): normalize(cross(dx, dy)) at the image's interior
    pixels whose row neighbours are in the window, zero elsewhere."""
    out = torch.zeros_like(p)
    dx = p[:, 2:, 1:-1] - p[:, :-2, 1:-1]
    dy = p[:, 1:-1, 2:] - p[:, 1:-1, :-2]
    n = torch.nn.functional.normalize(torch.cross(dx, dy, dim=0), dim=0)
    inner = ((rows[1:-1] >= 1) & (rows[1:-1] <= H - 2)).to(p.dtype)[None, :, None]
    out[:, 1:-1, 1:-1] = n * inner
    return out


def _whole_loss(normal, e, m, from_depth, H, W):
    """train.py:141-156 on the whole image, fp64, differentiable."""
    rows = torch.arange(H)
    if from_depth:
        fx, fy = W / (2 * math.tan(FOV[0] / 2.)), H / (2 * math.tan(FOV[1] / 2.))
        cam = (1 / fx, 1 / fy, -W / (2 * fx), -H / (2 * fy))
        pe, pm = _points_from_depth(e, rows, W, *cam), _points_from_depth(m, rows, W, *cam)
    else:
        pe, pm = e, m
    err = [1 - (normal * _normals(p, rows, H)).sum(0) for p in (pe, pm)]
    return (1 - DEPTH_RATIO) * err[0].mean() + DEPTH_RATIO * err[1].mean()


def fp64_normal_rows(normal_win, e_win, m_win, from_depth, inv_fx, inv_fy, cx, cy, w_e, w_m, H, r0, r1):
    """The contract of `rgs_normal_consistency_rows` (include/rgs_b200.h) restated with torch autograd in fp64."""
    W = normal_win.shape[-1]
    m_lo, n_lo, n_hi = max(0, r0 - 2), max(0, r0 - 1), min(H, r1 + 1)
    m_rows = torch.arange(m_lo, m_lo + e_win.shape[1])
    with torch.enable_grad():   # called from inside an autograd forward
        n, e, m = (t.detach().clone().requires_grad_(True) for t in (normal_win, e_win, m_win))
        if from_depth:
            pe, pm = _points_from_depth(e, m_rows, W, inv_fx, inv_fy, cx, cy), _points_from_depth(m, m_rows, W, inv_fx, inv_fy, cx, cy)
        else:
            pe, pm = e, m
        err = [1 - (n * _normals(p, m_rows, H)[:, n_lo - m_lo:n_hi - m_lo]).sum(0) for p in (pe, pm)]
        # every stencil that reaches the slab's pixels drives their gradients; only the slab's rows are counted
        (w_e * err[0].sum() + w_m * err[1].sum()).backward()
    own = slice(r0 - n_lo, r1 - n_lo)
    loss = (w_e * err[0][own].sum() + w_m * err[1][own].sum()).detach().reshape(1)
    return loss, n.grad[:, own], e.grad[:, r0 - m_lo:r1 - m_lo], m.grad[:, r0 - m_lo:r1 - m_lo]


def _inputs(H, W, seed=7):
    g = torch.Generator().manual_seed(seed)
    normal = torch.nn.functional.normalize(torch.randn(3, H, W, generator=g, dtype=torch.float64), dim=0)
    depth = [2.0 + 0.3 * torch.rand(1, H, W, generator=g, dtype=torch.float64) for _ in range(2)]
    coord = [torch.randn(3, H, W, generator=g, dtype=torch.float64) for _ in range(2)]
    return normal, depth, coord


def _worker(rank, world, port, H, W, weights, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        normal, depth, coord = _inputs(H, W)
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world, weights)
        r0, r1 = min(slabs[rank][0] * 16, H), min(slabs[rank][1] * 16, H)
        view = SimpleNamespace(FoVx=FOV[0], FoVy=FOV[1], image_height=H)
        out = {"rows": (r0, r1)}
        for compact in (False, True):
            for form, maps in (("depth", depth), ("point", coord)):
                if compact:
                    leaves = [t[:, r0:r1].clone().requires_grad_(True) for t in (normal, *maps)]
                else:
                    leaves = []
                    for t in (normal, *maps):
                        z = torch.zeros_like(t)
                        z[:, r0:r1] = t[:, r0:r1]            # a full-size sharded map: only the slab's rows are filled
                        leaves.append(z.requires_grad_(True))
                if form == "depth":   # with every rank's rows: the whole partition is checked on every rank
                    everyone = [(min(b * 16, H), min(e * 16, H)) for b, e in slabs]
                    loss = multigpu.slab_depth_normal_consistency_loss(view, *leaves, (r0, r1), DEPTH_RATIO, all_pixel_rows=everyone,
                                                                       kernels=fp64_normal_rows)
                else:
                    loss = multigpu.slab_point_normal_consistency_loss(*leaves, (r0, r1), DEPTH_RATIO, image_height=None if not compact and r1 - r0 < H else H,
                                                                       kernels=fp64_normal_rows)
                (2.5 * loss).backward()
                out[(form, compact)] = (loss.detach(), [t.grad for t in leaves])
        torch.save(out, os.path.join(tmpdir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


CASES = [
    (2, 16 * 5 + 3, 37, None),       # a last slab cut mid-tile
    (3, 16 * 7, 40, None),           # 3, 2, 2 tile rows
    (3, 33, 24, None),               # a last slab of one row
    (3, 50, 20, [0.0, 0.0, 0.0, 1.0]),   # weighted: one rank holds every row, two end empty at the image's last row
]


@pytest.mark.parametrize("world,H,W,weights", CASES, ids=[f"w{c[0]}_{c[1]}x{c[2]}{'_weighted' if c[3] else ''}" for c in CASES])
def test_slab_normal_consistency_equals_the_whole_image(world, H, W, weights, tmp_path):
    port = 37500 + (os.getpid() % 1500) + 7 * world + H % 7
    mp.spawn(_worker, args=(world, port, H, W, weights, str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    normal, depth, coord = _inputs(H, W)
    covered = sum(r["rows"][1] - r["rows"][0] for r in res)
    assert covered == H
    for form, maps in (("depth", depth), ("point", coord)):
        leaves = [t.clone().requires_grad_(True) for t in (normal, *maps)]
        ref = _whole_loss(*leaves, form == "depth", H, W)
        (2.5 * ref).backward()
        ref = float(ref.detach())
        for compact in (False, True):
            for r in res:
                loss, grads = r[(form, compact)]
                assert loss.dtype == torch.float32 and abs(float(loss) - ref) <= 1e-6 * max(1.0, abs(ref))
                r0, r1 = r["rows"]
                for g, leaf in zip(grads, leaves):
                    mine = g if compact else g[:, r0:r1]
                    assert mine.shape == leaf.grad[:, r0:r1].shape
                    torch.testing.assert_close(mine, leaf.grad[:, r0:r1], rtol=1e-12, atol=1e-15)
                    if not compact:
                        rest = g.clone()
                        rest[:, r0:r1] = 0
                        assert not rest.any()        # a rank's gradient lives in its own rows only
            # the fp64 stand-in's sums before the float32 return: every rank holds the same all-reduced value
            assert len({float(r[(form, compact)][0]) for r in res}) == 1


def _fp64_total_worker(rank, world, port, H, W, tmpdir):
    """The loss before its float32 rounding: the all-reduced fp64 sum of the slabs against the whole image's to 1e-12."""
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        normal, depth, _ = _inputs(H, W)
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world)
        r0, r1 = min(slabs[rank][0] * 16, H), min(slabs[rank][1] * 16, H)
        sums = []

        def keep(*a):
            out = fp64_normal_rows(*a)
            sums.append(out[0])
            return out

        view = SimpleNamespace(FoVx=FOV[0], FoVy=FOV[1], image_height=H)
        multigpu.slab_depth_normal_consistency_loss(view, *(t[:, r0:r1] for t in (normal, *depth)), (r0, r1), DEPTH_RATIO, kernels=keep)
        total = sums[0].clone()
        dist.all_reduce(total)
        torch.save(total, os.path.join(tmpdir, f"total{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_slab_normal_consistency_fp64_total(world, tmp_path):
    H, W = 16 * 5 + 9, 31
    port = 39500 + (os.getpid() % 1500) + world
    mp.spawn(_fp64_total_worker, args=(world, port, H, W, str(tmp_path)), nprocs=world, join=True)
    normal, depth, _ = _inputs(H, W)
    ref = float(_whole_loss(normal, *depth, True, H, W))
    for r in range(world):
        assert abs(float(torch.load(tmp_path / f"total{r}.pt")[0]) - ref) <= 1e-12


def test_single_process_slab_is_the_whole_image():
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    H, W = 21, 18
    normal, _, coord = _inputs(H, W)
    leaves = [t.clone().requires_grad_(True) for t in (normal, *coord)]
    loss = multigpu.slab_point_normal_consistency_loss(*leaves, (0, H), kernels=fp64_normal_rows)
    loss.backward()
    ref_leaves = [t.clone().requires_grad_(True) for t in (normal, *coord)]
    ref = _whole_loss(*ref_leaves, False, H, W)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-6
    for a, b in zip(leaves, ref_leaves):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-12, atol=1e-15)


def _refusal_worker(rank, world, port, H, weights, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        W = 12
        normal, depth, _ = _inputs(H, W)
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world, weights)
        everyone = [(min(b * 16, H), min(e * 16, H)) for b, e in slabs]
        r0, r1 = everyone[rank]
        view = SimpleNamespace(FoVx=FOV[0], FoVy=FOV[1], image_height=H)
        try:
            multigpu.slab_depth_normal_consistency_loss(view, *(t[:, r0:r1] for t in (normal, *depth)), (r0, r1), all_pixel_rows=everyone,
                                                        kernels=fp64_normal_rows)
            what = "no error"
        except ValueError as e:
            what = str(e)
        dist.barrier()   # every rank got here: nobody waits in an exchange
        torch.save({"rows": everyone, "error": what}, os.path.join(tmpdir, f"refusal{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_every_rank_refuses_a_partition_with_a_short_middle_slab(tmp_path):
    """A weighted partition can put several cuts on one heavy tile row, leaving an empty slab inside the image.  With every
    rank's rows given, all ranks raise before any exchange."""
    world, H = 3, 50
    port = 41500 + (os.getpid() % 1500)
    mp.spawn(_refusal_worker, args=(world, port, H, [0.0, 5.0, 0.0, 0.0], str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"refusal{r}.pt") for r in range(world)]
    assert res[0]["rows"] == [(0, 32), (32, 32), (32, 50)]
    for r in res:
        assert "at least 2 pixel rows" in r["error"], r["error"]


def test_all_pixel_rows_must_tile_the_image():
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    H, W = 40, 16
    n = torch.zeros(3, H, W, dtype=torch.float64)
    for bad in ([(0, 16), (16, 40)], [(0, 16), (16, 32), (30, 40)], [(0, 16), (16, 32), (32, 39)], [(0, 8), (16, 32), (32, 40)]):
        with pytest.raises(ValueError, match="all_pixel_rows"):
            multigpu.slab_point_normal_consistency_loss(n, n, n, (16, 32), all_pixel_rows=bad, rank=1, world_size=3, kernels=fp64_normal_rows)


def test_glue_refuses_cpu_tensors():
    from diff_gaussian_rasterization import _C
    H, W = 40, 16
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._slab.normal_consistency_rows(torch.zeros(3, 18, W), torch.zeros(1, 20, W), torch.zeros(1, 20, W), True, 1.0, 1.0, 0.0, 0.0, 0.5, 0.5,
                                         H, 16, 32)
    with pytest.raises(RuntimeError, match="CUDA"):
        _C._slab.normal_consistency_rows(torch.zeros(3, 18, W), torch.zeros(3, 20, W), torch.zeros(3, 20, W), False, 0.0, 0.0, 0.0, 0.0, 0.5, 0.5,
                                         H, 16, 32)


def test_input_checks():
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    H, W = 40, 16
    n, d = torch.zeros(3, H, W), torch.zeros(1, H, W)
    view = SimpleNamespace(FoVx=1.0, FoVy=1.0, image_height=H)
    with pytest.raises(RuntimeError, match="CUDA"):
        multigpu.slab_depth_normal_consistency_loss(view, n, d, d, (0, H))
    with pytest.raises(RuntimeError, match="CUDA"):
        multigpu.slab_point_normal_consistency_loss(n, n, n, (0, H))
    # a one-row slab in the middle of the image cannot supply its neighbours' two halo rows
    with pytest.raises(ValueError, match="at least 2"):
        multigpu.slab_depth_normal_consistency_loss(view, n[:, :1], d[:, :1], d[:, :1], (16, 17), rank=1, world_size=3, kernels=fp64_normal_rows)
    with pytest.raises(ValueError, match="at least 2"):
        multigpu.slab_depth_normal_consistency_loss(view, n[:, :0], d[:, :0], d[:, :0], (16, 16), rank=1, world_size=3, kernels=fp64_normal_rows)
    with pytest.raises(ValueError, match="image_height"):
        multigpu.slab_point_normal_consistency_loss(n[:, :16], n[:, :16], n[:, :16], (16, 32), rank=1, world_size=3, kernels=fp64_normal_rows)
    with pytest.raises(ValueError, match="slab's rows"):
        multigpu.slab_point_normal_consistency_loss(n[:, :16], n, n, (16, 32), image_height=H, rank=1, world_size=3, kernels=fp64_normal_rows)
    with pytest.raises(ValueError, match=r"\[1, 40 or 16 rows"):
        multigpu.slab_depth_normal_consistency_loss(view, n[:, :16], n[:, :16], n[:, :16], (16, 32), rank=1, world_size=3, kernels=fp64_normal_rows)
    with pytest.raises(ValueError, match="not rows"):
        multigpu.slab_point_normal_consistency_loss(n, n, n, (32, 48), kernels=fp64_normal_rows)
