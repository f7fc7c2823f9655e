"""The balanced partition of `ShardedGaussianRasterizer(balance=True)` on the host: the library's rule (include/rgs_b200.h,
`rgs_balance_partition`) against a Python restatement of it, its optimality against brute force, the argument checks, and the
slab losses' row rules on every balanced partition of images whose last tile row is 1 to 4 pixel rows tall.  No GPU."""
import itertools
import os
import re
import sys

import numpy as np
import pytest

from conftest import ROOT


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _tile_cost():
    text = open(os.path.join(ROOT, "include", "rgs_b200.h")).read()
    cost = int(re.search(r"#define RGS_BALANCE_TILE_COST (\d+)", text).group(1))
    assert _C()._slab.BALANCE_TILE_COST == cost
    return cost


def _weights(rows, grid_x):
    return [int(i) + _tile_cost() * grid_x for i in rows]


def optimal_largest(rows, grid_x, world):
    """B*: the least largest slab weight over all partitions into `world` contiguous slabs of at least one row, by dynamic
    programming over (slabs, rows) -- not the library's bisection."""
    w = _weights(rows, grid_x)
    gy = len(w)
    if gy < world:
        raise ValueError("fewer tile rows than ranks")
    pre = [0]
    for x in w:
        pre.append(pre[-1] + x)
    inf = float("inf")
    best = [0] + [inf] * gy          # best[j]: rows [0, j) in k slabs
    for k in range(1, world + 1):
        nxt = [inf] * (gy + 1)
        for j in range(k, gy - (world - k) + 1):
            nxt[j] = min(max(best[i], pre[j] - pre[i]) for i in range(k - 1, j))
        best = nxt
    return best[gy]


def restated_partition(rows, grid_x, world):
    """The header's cut, read literally: rank by rank, the longest run of rows from where the previous rank stopped whose weight is
    at most B* and that leaves one row for every later rank; the last rank takes the rest."""
    w = _weights(rows, grid_x)
    gy = len(w)
    best = optimal_largest(rows, grid_x, world)
    cuts = [0]
    for r in range(world - 1):
        b = cuts[-1]
        cuts.append(max(e for e in range(b + 1, gy - (world - r - 1) + 1) if sum(w[b:e]) <= best))
    cuts.append(gy)
    return cuts, best


def slab_weights(cuts, rows, grid_x):
    w = _weights(rows, grid_x)
    return [sum(w[cuts[r]:cuts[r + 1]]) for r in range(len(cuts) - 1)]


def library(rows, grid_x, world):
    return list(_C()._slab.balance_partition([int(i) for i in rows], grid_x, world))


def _histograms():
    rng = np.random.default_rng(5)
    out = []
    for gy in (1, 2, 3, 5, 8, 13, 34, 68, 75):
        gx = int(rng.integers(1, 121))
        out.append((f"zeros{gy}", [0] * gy, gx))
        out.append((f"random{gy}", rng.integers(0, 200_000, gy).tolist(), gx))
        hot = [0] * gy
        hot[int(rng.integers(0, gy))] = 3_000_000
        out.append((f"hot{gy}", hot, gx))
        out.append((f"ties{gy}", [5000] * gy, gx))
        out.append((f"lower_third{gy}", [100] * (gy - gy // 3) + [400_000] * (gy // 3), gx))
        out.append((f"alternate{gy}", [(y % 2) * 77_777 for y in range(gy)], gx))
    return out


@pytest.mark.parametrize("name,rows,grid_x", _histograms(), ids=[h[0] for h in _histograms()])
def test_library_partition_is_the_stated_rule(name, rows, grid_x):
    for world in (1, 2, 3, 4, 8, len(rows)):
        if world > len(rows):
            continue
        cuts, best = restated_partition(rows, grid_x, world)
        got = library(rows, grid_x, world)
        assert got == cuts, (world, got, cuts)
        assert all(got[r] < got[r + 1] for r in range(world)), "every slab holds a tile row"
        weights = slab_weights(got, rows, grid_x)
        assert max(weights) == best
        w = _weights(rows, grid_x)
        assert best <= -(-sum(w) // world) + max(w)


def test_grid_y_equal_to_world_gives_one_row_each():
    rows = [9, 0, 123456, 7, 7, 0]
    assert library(rows, 40, len(rows)) == list(range(len(rows) + 1))


def _brute_best(rows, grid_x, world):   # every composition of the rows into `world` slabs
    w = _weights(rows, grid_x)
    gy = len(w)
    best = None
    for inner in itertools.combinations(range(1, gy), world - 1):
        cuts = (0, *inner, gy)
        m = max(sum(w[cuts[r]:cuts[r + 1]]) for r in range(world))
        best = m if best is None else min(best, m)
    return best


def test_largest_slab_is_optimal_by_brute_force():
    rng = np.random.default_rng(11)
    for trial in range(300):
        gy = int(rng.integers(1, 10))
        world = int(rng.integers(1, gy + 1))
        grid_x = int(rng.integers(1, 6))
        kind = trial % 3
        if kind == 0:
            rows = rng.integers(0, 3000, gy).tolist()
        elif kind == 1:
            rows = (rng.integers(0, 3, gy) * 1000).tolist()   # many ties
        else:
            rows = [0] * gy
            rows[int(rng.integers(0, gy))] = int(rng.integers(1, 10**6))
        got = library(rows, grid_x, world)
        assert max(slab_weights(got, rows, grid_x)) == _brute_best(rows, grid_x, world) == optimal_largest(rows, grid_x, world), (rows, grid_x, world, got)
        assert got == restated_partition(rows, grid_x, world)[0]


def test_fewer_tile_rows_than_ranks_raises():
    with pytest.raises(RuntimeError, match="fewer tile rows than ranks"):
        library([1, 2, 3], 10, 4)
    with pytest.raises(RuntimeError, match="positive"):
        library([1, 2, 3], 10, 0)


def _settings(H):
    import torch

    import diff_gaussian_rasterization as dgr
    z = torch.zeros(3)
    return dgr.GaussianRasterizationSettings(H, 64, 0.5, 0.5, 0.0, z, 1.0, torch.eye(4), torch.eye(4), 0, z, False, True, False, False)


def test_sharded_rasterizer_balance_arguments():
    from rade_gs_b200.multigpu import ShardedGaussianRasterizer
    with pytest.raises(ValueError, match="row_weights"):
        ShardedGaussianRasterizer(_settings(128), rank=0, world_size=2, balance=True, row_weights=[1.0] * 8)
    with pytest.raises(ValueError, match="tile rows"):
        ShardedGaussianRasterizer(_settings(48), rank=0, world_size=4, balance=True)
    r = ShardedGaussianRasterizer(_settings(128), rank=1, world_size=2, balance=True)
    assert r.all_pixel_rows() == [(0, 64), (64, 128)] and r.pixel_rows() == (64, 128)


# ---- images whose last tile row holds 1 to 4 pixel rows (979x546 of the Tanks and Temples recipe, and others) ----------------

@pytest.mark.parametrize("H,W", [(546, 979), (1073, 1920), (49, 64), (180, 333)])
def test_every_balanced_partition_suits_the_slab_losses(H, W):
    """The greedy cut fills the earlier ranks first, so the last rank often takes only the image's last tile row, which here is
    shorter than the SSIM halo: the row checks of all three slab losses accept it (it ends at the image's last row), on every rank."""
    from rade_gs_b200 import multigpu
    gx, gy = (W + 15) // 16, (H + 15) // 16
    assert 1 <= H % 16 <= 4
    rng = np.random.default_rng(H)
    for kind in ("uniform", "random", "top_heavy", "bottom_heavy"):
        rows = {"uniform": [1000] * gy, "random": rng.integers(0, 300_000, gy).tolist(),
                "top_heavy": [400_000] * (gy // 3) + [50] * (gy - gy // 3), "bottom_heavy": [50] * (gy - gy // 3) + [400_000] * (gy // 3)}[kind]
        for world in range(2, min(8, gy) + 1):
            cuts = library(rows, gx, world)
            everyone = [(min(cuts[r] * 16, H), min(cuts[r + 1] * 16, H)) for r in range(world)]
            for rank in range(world):
                mine = everyone[rank]
                multigpu._check_ssim_rows(mine, H, world)
                multigpu._check_slab_rows(mine, everyone, H, rank, world)
                multigpu._check_slab_rows(mine, everyone, H, rank, world, multigpu.APPEARANCE_HALO, "the slab-local appearance loss")
    cuts = library([1000] * 35, 62, 8)
    assert cuts[-2:] == [34, 35], "979x546 at 8 ranks: the last rank holds only the 2-row tile row"


def test_ssim_row_check_still_refuses_short_inner_and_empty_last_slabs():
    from rade_gs_b200 import multigpu
    with pytest.raises(ValueError, match="5 pixel rows"):
        multigpu._check_ssim_rows((96, 98), 100, 3)      # short, not at the image's last row
    with pytest.raises(ValueError, match="5 pixel rows"):
        multigpu._check_ssim_rows((98, 98), 98, 3)       # empty
    with pytest.raises(ValueError, match="not rows of a 100-row image"):
        multigpu._check_ssim_rows((96, 104), 100, 3)     # past the image's last row: refused before the halo exchange
    multigpu._check_ssim_rows((96, 98), 98, 3)


def _short_tail_worker(rank, world, port, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist

    from rade_gs_b200 import multigpu
    from test_multigpu_host import _torch_slab_kernels
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W = 16 * 6 + 2, 40                  # slabs of 3 and 3 tile rows, then the 2-row last tile row
        rows = [(0, 48), (48, 96), (96, 98)]
        g = torch.Generator().manual_seed(7)
        gt = torch.rand(3, H, W, generator=g, dtype=torch.float64)
        whole = (gt + 0.2 * torch.randn(3, H, W, generator=g, dtype=torch.float64)).clamp(0, 1)
        r0, r1 = rows[rank]
        mine = torch.zeros_like(whole)
        mine[:, r0:r1] = whole[:, r0:r1]
        mine.requires_grad_(True)
        loss = multigpu.slab_l1_ssim_loss(mine, gt, 0.2, (r0, r1), kernels=_torch_slab_kernels())
        loss.backward()
        torch.save({"loss": loss.detach(), "grad": mine.grad, "rows": (r0, r1), "whole": whole, "gt": gt}, os.path.join(tmpdir, f"tail{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_slab_ssim_with_a_short_last_slab_equals_the_whole_image_loss(tmp_path):
    """Three ranks over gloo, torch expressions standing in for the CUDA kernels: a 2-row last slab gives the whole image's loss and
    gradient, as the halo exchange with it is sized by the image's edge."""
    import torch
    import torch.multiprocessing as mp

    from test_multigpu_host import _ssim_map
    world = 3
    mp.spawn(_short_tail_worker, args=(world, 37600 + os.getpid() % 2000, str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"tail{r}.pt") for r in range(world)]
    x = res[0]["whole"].clone().requires_grad_(True)
    gt = res[0]["gt"]
    ref = 0.8 * (x - gt).abs().mean() + 0.2 * (1 - _ssim_map(x, gt).mean())
    ref.backward()
    grad = torch.zeros_like(x)
    for r in res:
        assert abs(float(r["loss"]) - float(ref)) < 1e-6, (float(r["loss"]), float(ref))
        r0, r1 = r["rows"]
        grad[:, r0:r1] = r["grad"][:, r0:r1]
    assert torch.allclose(grad, x.grad, rtol=1e-9, atol=1e-12)
