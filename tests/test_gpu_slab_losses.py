"""Slab-local normal consistency on the GPU.

One process: each image (1600x1200, 979x546, a 33-row one) is split into 2, 3, 4 and 8 slabs, equal and weighted
(`partition_tile_rows`).  `_C._slab.normal_consistency_rows` runs on each slab with the halo rows cut from the whole maps.
The stitched gradients must equal the whole-image `_C.normal_consistency` bit for bit.  The summed loss must lie within the fp64
model's bound (tests/image_loss_f64.py), as the whole-image kernel's does.  Repeat calls, poisoned memory and a late-ready side
stream give the same bits.

Several GPUs (NCCL, world 2/4/8, skipped when the box has fewer): one whole sharded training step, `ShardedGaussianRasterizer
(compact=True)` with the slab-local L1 + SSIM and normal-consistency losses, against the single-GPU rasterizer with the
whole-image losses."""
import os
import sys

import numpy as np
import pytest
import torch

import image_loss_f64 as il
from conftest import ROOT
from test_gpu_stale_memory import Case, check_case, poisoned_allocator  # noqa: F401  (the fixture)
from test_image_loss_f64_host import camera, normal_inputs

pytestmark = pytest.mark.gpu


def _C():
    from diff_gaussian_rasterization import _C
    return _C


def _partitions(H, world):
    from rade_gs_b200.multigpu import partition_tile_rows, tile_rows
    n = tile_rows(H)
    g = np.random.default_rng(H * 10 + world)
    out = {"equal": partition_tile_rows(n, world)}
    if n >= world:
        out["weighted"] = partition_tile_rows(n, world, list(g.uniform(0.2, 3.0, n)))
    rows = {}
    for name, slabs in out.items():
        px = [(min(b * 16, H), min(e * 16, H)) for b, e in slabs]
        # a slab of fewer than 2 rows that does not end at the last row cannot be used: the Python layer refuses such a partition
        # (tests/test_slab_losses_host.py), so the kernel is never called on it
        if all(e - b >= 2 or e == H for b, e in px):
            rows[name] = px
    return rows


def _slab_call(inp, from_depth, cam, w_e, w_m, H, r0, r1):
    n, e, m = inp
    m_lo, m_hi, n_lo, n_hi = max(0, r0 - 2), min(H, r1 + 2), max(0, r0 - 1), min(H, r1 + 1)
    return _C()._slab.normal_consistency_rows(n[:, n_lo:n_hi], e[:, m_lo:m_hi], m[:, m_lo:m_hi], from_depth, *cam, w_e, w_m, H, r0, r1)


def _int(t):
    return t.contiguous().view(torch.int32)


SIZES = [(1200, 1600), (546, 979), (33, 50)]


@pytest.mark.parametrize("from_depth", [True, False], ids=["depth", "coord"])
@pytest.mark.parametrize("H,W", SIZES, ids=[f"{w}x{h}" for h, w in SIZES])
def test_slabs_stitch_to_the_whole_image_bit_for_bit(H, W, from_depth):
    inp = tuple(t.cuda() for t in normal_inputs(H, W, from_depth, seed=H + 7 * W, background=True))
    cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
    w_e, w_m = 0.4 / (H * W), 0.6 / (H * W)
    loss, dn, de, dm = _C().normal_consistency(*inp, from_depth, *cam, w_e, w_m)
    model = il.normal_consistency(*(t.cpu() for t in inp), from_depth, *cam, w_e, w_m, device="cuda") if H * W < 10 ** 6 else None
    tried = 0
    for world in (2, 3, 4, 8):
        for name, rows in _partitions(H, world).items():
            tried += 1
            total = 0.0
            parts = [[], [], []]
            for r0, r1 in rows:
                if r1 == r0:
                    continue
                s, *g = _slab_call(inp, from_depth, cam, w_e, w_m, H, r0, r1)
                total += float(s[0])
                for p, t in zip(parts, g):
                    assert t.shape[1] == r1 - r0
                    p.append(t)
            for got, ref, what in zip(parts, (dn, de, dm), ("d_normal", "d_expected", "d_median")):
                got = torch.cat(got, 1)
                bad = int((_int(got) != _int(ref)).sum())
                assert bad == 0, f"{world} slabs ({name}): {what} differs at {bad} of {ref.numel()} elements"
            # the per-block fp32 partials are the whole image's; only their fp64 order differs
            assert abs(total - float(loss[0])) <= 1e-12 * max(1.0, abs(float(loss[0]))), (world, name, total, float(loss[0]))
            if model is not None:
                v, e = model["loss"]
                assert abs(total - v.item()) <= e.item() * (1 + 1e-6), (world, name, total, v.item(), e.item())
    assert tried >= 4


def test_row_ranges_off_tile_rows_and_single_rows():
    """Ranges that start and end anywhere, one-row ranges at both borders and a range covering the whole image."""
    H, W = 37, 41
    for from_depth in (True, False):
        inp = tuple(t.cuda() for t in normal_inputs(H, W, from_depth, seed=5))
        cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
        _, *whole = _C().normal_consistency(*inp, from_depth, *cam, 0.3, 0.7)
        for r0, r1 in ((0, 1), (36, 37), (0, 37), (3, 29), (15, 17), (1, 36), (20, 21)):
            _, *g = _slab_call(inp, from_depth, cam, 0.3, 0.7, H, r0, r1)
            for got, ref in zip(g, whole):
                assert torch.equal(_int(got), _int(ref[:, r0:r1])), (from_depth, r0, r1)


def test_refuses_wrong_windows():
    H, W = 40, 20
    n, e = torch.zeros(3, H, W, device="cuda"), torch.zeros(1, H, W, device="cuda")
    C = _C()._slab
    with pytest.raises(RuntimeError, match="rendered_normal"):
        C.normal_consistency_rows(n[:, 14:34], e[:, 14:34], e[:, 14:34], True, 1.0, 1.0, 0.0, 0.0, 0.5, 0.5, H, 16, 32)   # the maps' window
    with pytest.raises(RuntimeError, match="expected map"):
        C.normal_consistency_rows(n[:, 15:33], e[:, 15:33], e[:, 14:34], True, 1.0, 1.0, 0.0, 0.0, 0.5, 0.5, H, 16, 32)
    with pytest.raises(RuntimeError, match="row_lo"):
        C.normal_consistency_rows(n, e, e, True, 1.0, 1.0, 0.0, 0.0, 0.5, 0.5, H, 30, 20)


def test_repeat_poison_and_side_stream(poisoned_allocator):
    H, W = 70, 53
    out = {}
    for from_depth in (True, False):
        inp = tuple(t.cuda() for t in normal_inputs(H, W, from_depth, seed=11, background=True))
        cam = camera(H, W) if from_depth else (0.0, 0.0, 0.0, 0.0)
        out[from_depth] = (inp, cam)

    def run(x):
        res = {}
        for from_depth, (inp, cam) in x.items():
            for r0, r1 in ((0, 16), (16, 48), (48, 70)):
                s, dn, de, dm = _slab_call(inp, from_depth, cam, 0.4 / (H * W), 0.6 / (H * W), H, r0, r1)
                for k, v in (("loss", s), ("d_normal", dn), ("d_e", de), ("d_m", dm)):
                    res[f"{from_depth}/{r0}/{k}"] = v
        return res

    sums = {f"{d}/{r0}/loss": ("sum",) for d in (True, False) for r0 in (0, 16, 48)}   # fp64 atomics across blocks: order-dependent
    check_case(Case(out, run, sums), poisoned_allocator)


# ---- several GPUs: one sharded training step -----------------------------------------------------------------------------

def _step_worker(rank, world, port, outdir, coord):
    for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    from types import SimpleNamespace
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import losses, multigpu, scenes
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    ex = None
    try:
        sc = scenes.make_scene(60000, 640, 400, 500.0, -3.8, seed=21, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.2, 0.1, 0.3)).to(dev)
        sc = multigpu.broadcast_scene_(sc)
        H, W = sc.height, sc.width
        st = dgr.GaussianRasterizationSettings(H, W, sc.tanfovx, sc.tanfovy, 0.1, sc.bg, 1.0, sc.viewmatrix, sc.projmatrix, 3, sc.campos, False,
                                               not coord, coord, False)
        ex = multigpu.GradExchange(sc.means3D.shape[0], dgr._C.grad_stride(coord, not coord), dev)
        g = torch.Generator().manual_seed(9)
        gt = torch.rand(3, H, W, generator=g).to(dev)
        view = SimpleNamespace(FoVx=2 * np.arctan(sc.tanfovx), FoVy=2 * np.arctan(sc.tanfovy), image_height=H, image_width=W)

        def step(sharded):
            lv = {k: getattr(sc, k).clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
            m2 = torch.zeros_like(lv["means3D"], requires_grad=True)
            rast = multigpu.ShardedGaussianRasterizer(st, exchange=ex, compact=True) if sharded else dgr.GaussianRasterizer(st)
            color, _, co, mco, dep, mdep, _, normal = rast(lv["means3D"], m2, lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                                                           rotations=lv["rotations"])
            if sharded:
                rows = rast.pixel_rows()
                everyone = [(min(b * 16, H), min(e * 16, H)) for b, e in rast.slabs]
                full = color.new_zeros(3, H, W)        # slab_l1_ssim_loss takes full-size maps
                full[:, rows[0]:rows[1]] = color
                rgb = multigpu.slab_l1_ssim_loss(full, gt, 0.2, rows)
                if coord:
                    nc = multigpu.slab_point_normal_consistency_loss(normal, co, mco, rows, image_height=H, all_pixel_rows=everyone)
                else:
                    nc = multigpu.slab_depth_normal_consistency_loss(view, normal, dep, mdep, rows, all_pixel_rows=everyone)
            else:
                rgb = losses.l1_ssim_loss(color, gt, 0.2)
                nc = losses.point_normal_consistency_loss(normal, co, mco) if coord else losses.depth_normal_consistency_loss(view, normal, dep, mdep)
            loss = rgb + 0.05 * nc
            loss.backward()
            return float(loss), {k: v.grad for k, v in lv.items()}

        ls, gs = step(True)
        l1, g1 = step(False)
        res = {"loss": (ls, l1)}
        for k in gs:
            res[k] = (gs[k].double().cpu().numpy(), g1[k].double().cpu().numpy())
            ref = gs[k].contiguous().clone()
            dist.broadcast(ref, src=0)
            res[k + "/bits_differ_from_rank0"] = int((_int(gs[k]) != _int(ref)).sum())
        np.save(os.path.join(outdir, f"step{rank}.npy"), res, allow_pickle=True)
    finally:
        if ex is not None:
            ex.close()
        dist.destroy_process_group()


@pytest.mark.parametrize("coord", [False, True], ids=["depth", "coord"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_step_with_slab_losses_equals_single(world, coord, tmp_path):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    import tolerances as tol
    mp.spawn(_step_worker, args=(world, 29800 + os.getpid() % 1000 + world + 10 * coord, str(tmp_path), coord), nprocs=world, join=True)
    for rank in range(world):
        res = np.load(tmp_path / f"step{rank}.npy", allow_pickle=True).item()
        ls, l1 = res.pop("loss")
        assert abs(ls - l1) <= 1e-5 * max(1.0, abs(l1)), (rank, ls, l1)
        for k, v in res.items():
            if k.endswith("/bits_differ_from_rank0"):
                assert v == 0, (rank, k, v)
            else:
                tol.grad_close_gpu(v[0], v[1], f"rank {rank} {k}")
