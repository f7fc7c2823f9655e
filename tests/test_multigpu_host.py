"""World-size-2 test of the multi-GPU control flow on CPU (gloo): slab-local scatter -> ONE all-reduce of the
screen-space gradient rows -> replicated parameter gradients.  The CUDA stages are replaced by the oracle's
(oracle.render_backward / oracle.preprocess_backward), the control flow under test is
rade_gs_b200.multigpu.allreduce_sum_ / partition_tile_rows -- the same code the GPU path runs with NCCL."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN_CASES, ROOT, golden_oracle_inputs, golden_upstream, load_golden

SG_KEYS = ("mean2D", "conic", "opacity", "colors", "ts", "camera_planes", "ray_planes", "normals", "view_points")


def _slab_upstream(up, H, rows):
    """Upstream gradients restricted to a slab of pixel rows: every per-pixel term of backward-render is linear in
    that pixel's upstream gradients, so zeroing the other rows yields exactly the slab's partial sums."""
    out = {}
    for k, v in up.items():
        z = np.zeros_like(v)
        z[:, rows[0]:rows[1], :] = v[:, rows[0]:rows[1], :]
        out[k] = z
    return out


def _worker(rank, world, port, case, tmpdir):
    for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import oracle
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        d = load_golden(case)
        inp = golden_oracle_inputs(d)
        H = inp.H
        fwd = oracle.forward(inp)  # replicated on every rank, like preprocess on the GPUs
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world)
        rows = (min(slabs[rank][0] * 16, H), min(slabs[rank][1] * 16, H))
        up = _slab_upstream(golden_upstream(d), H, rows)

        def stage1():
            sg = oracle.render_backward(inp, fwd, up)
            return torch.from_numpy(np.concatenate([sg[k].reshape(inp.P, -1) for k in SG_KEYS], axis=1))

        def stage2(acc):
            a = acc.numpy()
            sg, o = {}, 0
            for k, w in zip(SG_KEYS, (3, 4, 1, 3, 1, 6, 2, 3, 3)):
                sg[k] = np.ascontiguousarray(a[:, o:o + w]).reshape(-1) if w == 1 else np.ascontiguousarray(a[:, o:o + w])
                o += w
            return oracle.preprocess_backward(inp, fwd, sg)

        out = stage2(multigpu.allreduce_sum_(stage1()))
        np.savez(os.path.join(tmpdir, f"rank{rank}.npz"), **{k: v for k, v in out.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("case", [c for c in ("depth_ks01", "coord_ks0") if c in GOLDEN_CASES])
def test_two_rank_all_reduced_backward_equals_single(case, tmp_path):
    import oracle
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, case, str(tmp_path)), nprocs=2, join=True)
    d = load_golden(case)
    inp = golden_oracle_inputs(d)
    fwd = oracle.forward(inp)
    single = oracle.backward(inp, fwd, golden_upstream(d))
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations"):
        assert np.array_equal(r0[k], r1[k]), k  # replicated result
        ref = single[k]
        err = np.abs(r0[k] - ref).max()
        assert err <= 1e-5 * max(1.0, np.abs(ref).max()), (k, err)  # float64 partial sums: association only


def test_allreduce_is_noop_without_process_group():
    from rade_gs_b200.multigpu import allreduce_sum_
    t = torch.arange(6.0)
    assert torch.equal(allreduce_sum_(t.clone()), t)


def test_unknown_exchange_mode_is_refused(monkeypatch):
    """`peer` and `dense` are the only modes; anything else is refused, also on one process where the mode becomes dense."""
    from rade_gs_b200.multigpu import GradExchange
    with pytest.raises(ValueError, match="bogus"):
        GradExchange(10, 16, "cpu", mode="bogus")
    monkeypatch.setenv("RGS_GRAD_EXCHANGE", "bogus")
    with pytest.raises(ValueError, match="bogus"):
        GradExchange(10, 16, "cpu")
    monkeypatch.setenv("RGS_GRAD_EXCHANGE", "dense")
    assert GradExchange(10, 16, "cpu").mode == "dense"


def _gather_worker(rank, world, port, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W = 40, 24  # 3 tile rows -> slabs of 2 and 1 rows
        g = torch.Generator().manual_seed(3)
        whole = torch.rand(3, H, W, generator=g)
        weight = torch.rand(3, H, W, generator=g)
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world)
        r0, r1 = min(slabs[rank][0] * 16, H), min(slabs[rank][1] * 16, H)
        mine = torch.zeros_like(whole)
        mine[:, r0:r1] = whole[:, r0:r1]
        mine.requires_grad_(True)
        rows = [(min(b * 16, H), min(e * 16, H)) for b, e in slabs]
        full = multigpu._GatherSlabs.apply(mine, None, rows, rank)
        loss = (full * full * weight).sum()  # any full-image loss, evaluated redundantly on each rank
        loss.backward()
        torch.save({"full": full.detach(), "grad": mine.grad, "rows": (r0, r1), "whole": whole, "weight": weight},
                   os.path.join(tmpdir, f"gather{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_gather_image_is_differentiable_across_two_ranks(tmp_path):
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_gather_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    covered = 0
    for rank in range(2):
        d = torch.load(tmp_path / f"gather{rank}.pt")
        assert torch.equal(d["full"], d["whole"])  # the gathered slabs reassemble the image exactly (pure copies)
        r0, r1 = d["rows"]
        want = 2 * d["whole"] * d["weight"]
        assert torch.allclose(d["grad"][:, r0:r1], want[:, r0:r1])  # the rows this rank's backward consumes
        covered += r1 - r0
    assert covered == 40


def _exchange_worker(rank, world, port, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        P, stride = 5000, 16
        out = {}
        for case, density in (("typical", 0.3), ("empty_rank", 0.0 if rank == 1 else 0.4), ("full", 1.0)):
            g = torch.Generator().manual_seed(100 + 7 * rank + len(case))
            acc = torch.randn(P, stride, generator=g)
            acc[torch.rand(P, generator=g) >= density] = 0.0  # rows of Gaussians that do not reach this rank's slab
            if density > 0:
                acc[17] = float(rank + 1)  # a row every rank contributes to
            out[case + "_in"] = acc.clone()
            out[case + "_dense"] = multigpu.allreduce_sum_(acc.clone())
            out[case + "_group"] = multigpu.allreduce_sum_(acc.clone(), dist.group.WORLD)   # an explicit group, as the rasterizer passes it
        torch.save(out, os.path.join(tmpdir, f"exchange{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_row_all_reduce_equals_the_sum_over_ranks(world, tmp_path):
    port = 33500 + (os.getpid() % 2000) + world
    mp.spawn(_exchange_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"exchange{r}.pt") for r in range(world)]
    for case in ("typical", "empty_rank", "full"):
        total = sum(r[case + "_in"].double() for r in res)
        for r in res:
            assert torch.allclose(r[case + "_dense"].double(), total, rtol=1e-6, atol=1e-6)
            assert torch.allclose(r[case + "_group"].double(), total, rtol=1e-6, atol=1e-6)


# ---- slab-local L1 + SSIM with halo rows: host logic on CPU (gloo), torch expressions standing in for the CUDA kernels -----------

def _ssim_map(a, b):
    """utils/loss_utils.py:35-63 restated (window 11, sigma 1.5, zero padding), returning the map."""
    import torch.nn.functional as F
    g = torch.tensor([math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)], dtype=a.dtype)
    g = g / g.sum()
    w = (g[:, None] @ g[None, :])[None, None].expand(a.shape[0], 1, 11, 11).contiguous()
    conv = lambda t: F.conv2d(t[None], w, padding=5, groups=a.shape[0])[0]  # noqa: E731
    mu1, mu2 = conv(a), conv(b)
    s1, s2, s12 = conv(a * a) - mu1 * mu1, conv(b * b) - mu2 * mu2, conv(a * b) - mu1 * mu2
    return ((2 * mu1 * mu2 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1 * mu1 + mu2 * mu2 + 0.01 ** 2) * (s1 + s2 + 0.03 ** 2))


def _torch_slab_kernels():
    def fwd(img, gt, r0, r1, need_grad):
        return torch.stack([_ssim_map(img, gt)[:, r0:r1].sum().double(), (img - gt).abs()[:, r0:r1].sum().double()]), ()

    def bwd(img, gt, state, w_ssim, w_l1, r0, r1):
        with torch.enable_grad():   # called from inside an autograd backward, where grad mode is off
            x = img.clone().requires_grad_(True)
            (w_ssim * _ssim_map(x, gt)[:, r0:r1].sum() + w_l1 * (x - gt).abs()[:, r0:r1].sum()).backward()
        return x.grad

    return fwd, bwd


def _slab_loss_worker(rank, world, port, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        H, W = 16 * 7, 40                     # 7 tile rows over 3 ranks: slabs of 3, 2, 2 tile rows
        g = torch.Generator().manual_seed(5)
        gt = torch.rand(3, H, W, generator=g, dtype=torch.float64)
        whole = (gt + 0.2 * torch.randn(3, H, W, generator=g, dtype=torch.float64)).clamp(0, 1)
        slabs = multigpu.partition_tile_rows(multigpu.tile_rows(H), world)
        r0, r1 = slabs[rank][0] * 16, min(slabs[rank][1] * 16, H)
        mine = torch.zeros_like(whole)
        mine[:, r0:r1] = whole[:, r0:r1]
        mine.requires_grad_(True)
        loss = multigpu.slab_l1_ssim_loss(mine, gt, 0.2, (r0, r1), kernels=_torch_slab_kernels())
        loss.backward()
        torch.save({"loss": loss.detach(), "grad": mine.grad, "rows": (r0, r1), "whole": whole, "gt": gt}, os.path.join(tmpdir, f"slabloss{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_slab_local_ssim_with_halo_rows_equals_the_whole_image_loss(tmp_path):
    world = 3
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_slab_loss_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"slabloss{r}.pt") for r in range(world)]
    x = res[0]["whole"].clone().requires_grad_(True)
    gt = res[0]["gt"]
    ref = 0.8 * (x - gt).abs().mean() + 0.2 * (1 - _ssim_map(x, gt).mean())      # train.py:163 on the whole image, one process
    ref.backward()
    grad = torch.zeros_like(x)
    for r in res:
        assert abs(float(r["loss"]) - float(ref)) < 1e-6, (float(r["loss"]), float(ref))   # the loss is returned as float32
        r0, r1 = r["rows"]
        out = r["grad"].clone()
        out[:, r0:r1] = 0
        assert not out.any()                                 # a rank's gradient lives in its own rows only
        grad[:, r0:r1] = r["grad"][:, r0:r1]
    assert torch.allclose(grad, x.grad, rtol=1e-9, atol=1e-12)  # including the rows next to slab boundaries (halo contributions)


def _bcast_worker(rank, world, port, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from types import SimpleNamespace
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(11)
        sc = SimpleNamespace(means3D=torch.randn(100, 3, generator=g), scales=torch.rand(100, 3, generator=g), width=64, name="x")
        if rank == 1:
            sc.scales = sc.scales + 1e-7        # "the same scene", one ulp off on another rank
            sc.means3D = sc.means3D.t().contiguous().t()   # and a non-contiguous view
        multigpu.broadcast_scene_(sc)
        torch.save({"means3D": sc.means3D.clone(), "scales": sc.scales.clone(), "width": sc.width}, os.path.join(tmpdir, f"bcast{rank}.pt"))
    finally:
        dist.destroy_process_group()


def test_broadcast_scene_makes_the_replicated_state_bit_identical(tmp_path):
    """Slabs only compose to the single-GPU image when every rank rasterizes the same bits."""
    port = 36500 + (os.getpid() % 2000)
    mp.spawn(_bcast_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    a, b = (torch.load(tmp_path / f"bcast{r}.pt") for r in range(2))
    assert torch.equal(a["means3D"], b["means3D"]) and torch.equal(a["scales"], b["scales"]) and a["width"] == b["width"] == 64
