"""The row forms of the decoupled-appearance L1 loss (include/rgs_b200.h's rgs_appearance_*_rows) on one GPU: every slab of 2/3/4/8
equal and weighted partitions runs the row kernels on windows cut from the whole tensors, and the stitched low-resolution map,
d_image (with the downsample's share) and d(up4) must equal the whole-image `_C.appearance_*` outputs bit for bit.  The per-slab
fp64 loss and weight-gradient rows, summed in rank order, must lie within test_fused_golden._close's bar against an fp64 eager
evaluation, as the whole-image kernel's do.  Then `multigpu.slab_L1_loss_appearance` at one rank against `L1_loss_appearance`, the
SSIM-only companion term, and the row kernels on poisoned memory and a late-ready side stream.

One sharded training step with the whole DTU / TNT recipe loss (NCCL, world 1/2/4/8, skipped when the box has fewer GPUs):
`ShardedGaussianRasterizer(compact=True)` with `slab_L1_loss_appearance`, the SSIM-only `slab_l1_ssim_loss(..., 1.0, rows)` and
the slab-local depth-normal consistency, against the single-GPU rasterizer with `L1_loss_appearance` and the whole-image losses."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from test_fused_golden import _close
from test_gpu_appearance import _recipe_inputs, _setup
from test_gpu_stale_memory import Case, check_case, poisoned_allocator  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALO = 4
SIZES = [(1200, 1600), (546, 979), (600, 800), (40, 50)]


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _partitions(H0):
    from rade_gs_b200 import multigpu
    n = multigpu.tile_rows(H0)
    out = {}
    for world in (2, 3, 4, 8):
        out[f"{world}eq"] = multigpu.partition_tile_rows(n, world)
    # weighted: most of the work in the lower third (slabs of very different heights, empty trailing slabs at the small size)
    wts = [1.0 + 20.0 * (y > 2 * n // 3) for y in range(n)]
    for world in (3, 8):
        out[f"{world}wt"] = multigpu.partition_tile_rows(n, world, wts)
    return {k: [(min(b * 16, H0), min(e * 16, H0)) for b, e in v] for k, v in out.items()}


def _inputs(H0, W0, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = H0 // 32 * 32, W0 // 32 * 32
    gt = torch.rand(3, H0, W0, generator=g)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=g)).clamp(0, 1)
    up4 = torch.relu(torch.randn(1, 16, H // 2, W // 2, generator=g))
    w2, b2 = torch.randn(16, 16, 3, 3, generator=g) * (2.0 / 144) ** 0.5, 0.05 * torch.randn(16, generator=g)
    w3, b3 = torch.randn(3, 16, 3, 3, generator=g) * (2.0 / 144) ** 0.5, 0.05 * torch.randn(3, generator=g)
    d_down = 1e-3 * torch.randn(3, H // 32, W // 32, generator=g)
    t = [x.to(DEV) for x in (image, gt, up4, w2, b2, w3, b3, d_down)]
    return dict(zip(("image", "gt", "up4", "w2", "b2", "w3", "b3", "d_down"), t)) | {"upstream": torch.tensor([0.75], device=DEV)}


def _whole(x):
    C = _C()
    down = C.appearance_downsample(x["image"])
    loss, act, _ = C.appearance_l1_forward(x["image"], x["gt"], x["up4"], x["w2"], x["b2"], x["w3"], x["b3"], True, False)
    d_img, d_up4, *dw = C.appearance_l1_backward(x["image"], x["gt"], x["up4"], act, x["w2"], x["b2"], x["w3"], x["b3"], x["upstream"])
    C.appearance_downsample_backward(x["d_down"], d_img)
    return {"down": down, "loss": loss, "act": act, "d_image": d_img, "d_up4": d_up4, "dw": dw}


def _slabs(x, rows):
    """Each slab's row kernels on windows cut from the whole tensors; the owned rows stitched, the fp64 sums added in rank order."""
    C = _C()
    image, gt = x["image"], x["gt"]
    H0, W0 = image.shape[1:]
    H, W = H0 // 32 * 32, W0 // 32 * 32
    down = torch.full((3, H // 32, W // 32), float("nan"), device=DEV)
    d_up4 = torch.full((16, H // 2, W // 2), float("nan"), device=DEV)
    d_image = torch.full_like(image, float("nan"))
    acts, loss_sum, grad_row = [], None, None
    for r0, r1 in rows:
        w = C._slab.appearance_row_windows(H0, W0, r0, r1)
        lo, hi = max(0, r0 - HALO), min(H0, r1 + HALO)
        win, gwin = image[:, lo:hi].contiguous(), gt[:, lo:hi].contiguous()
        down[:, w[2]:w[3]] = C._slab.appearance_downsample_rows(win, lo, H0, r0, r1)
        s, act = C._slab.appearance_l1_forward_rows(win, gwin, lo, H0, r0, r1, x["up4"], x["w2"], x["b2"], x["w3"], x["b3"])
        acts.append((w[6], w[7], act))
        di, du, g = C._slab.appearance_l1_backward_rows(win, gwin, lo, H0, r0, r1, x["up4"], act, x["w2"], x["b2"], x["w3"], x["b3"], x["upstream"])
        C._slab.appearance_downsample_backward_rows(x["d_down"], di, H0, r0, r1)
        d_image[:, r0:r1] = di
        d_up4[:, w[4]:w[5]] = du
        loss_sum = s if loss_sum is None else loss_sum + s
        grad_row = g if grad_row is None else grad_row + g
    return {"down": down, "d_image": d_image, "d_up4": d_up4.reshape(1, 16, H // 2, W // 2), "acts": acts,
            "loss": (loss_sum / (3.0 * H * W)).float()[0], "grad_row": grad_row.float()}


def _bits(name, a, b):
    assert a.shape == b.shape, (name, tuple(a.shape), tuple(b.shape))
    bad = int((a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).sum())
    assert bad == 0, f"{name}: {bad} of {a.numel()} elements differ"


def _eager(x, dtype):
    """The tail in torch (fp32 or fp64): loss and conv2 / conv3's weight and bias gradients."""
    H0, W0 = x["image"].shape[1:]
    H, W = H0 // 32 * 32, W0 // 32 * 32
    top, left = H0 // 2 - H // 2, W0 // 2 - W // 2
    p = [x[k].to(dtype).requires_grad_(True) for k in ("w2", "b2", "w3", "b3")]
    X = F.interpolate(x["up4"].to(dtype), scale_factor=2, mode="bilinear", align_corners=True)
    M = torch.sigmoid(F.conv2d(torch.relu(F.conv2d(X, p[0], p[1], padding=1)), p[2], p[3], padding=1))[0]
    crop, crop_gt = (x[k].to(dtype)[:, top:top + H, left:left + W] for k in ("image", "gt"))
    loss = (M * crop - crop_gt).abs().mean()
    grads = torch.autograd.grad(loss * x["upstream"].to(dtype)[0], p)
    return loss.item(), torch.cat([g.reshape(-1) for g in grads]).double().cpu().numpy()


@pytest.fixture
def no_tf32():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("H0,W0", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_stitched_slabs_are_the_whole_image_bit_for_bit(H0, W0, no_tf32):
    x = _inputs(H0, W0, H0 + W0)
    whole = _whole(x)
    l32, g32 = _eager(x, torch.float32)
    l64, g64 = _eager(x, torch.float64)
    g_whole = torch.cat([t.reshape(-1) for t in whole["dw"]]).double().cpu().numpy()
    _close(whole["loss"].item(), l32, l64, "whole loss", 2e-6)
    _close(g_whole, g32, g64, "whole weight gradients", 2e-6)
    for name, rows in _partitions(H0).items():
        s = _slabs(x, rows)
        _bits(f"{name} down", s["down"], whole["down"])
        _bits(f"{name} d_image", s["d_image"], whole["d_image"])
        _bits(f"{name} d_up4", s["d_up4"], whole["d_up4"])
        for a_lo, a_hi, act in s["acts"]:
            _bits(f"{name} act rows [{a_lo}, {a_hi})", act, whole["act"][:, a_lo:a_hi])
        _close(s["loss"].item(), l32, l64, f"{name} loss", 2e-6)
        _close(s["grad_row"].double().cpu().numpy(), g32, g64, f"{name} weight gradients", 2e-6)
    # one slab over the whole image is the whole-image call
    one = _slabs(x, [(0, H0)])
    _bits("1 slab loss", one["loss"].reshape(1), whole["loss"].reshape(1))
    _bits("1 slab weight gradients", one["grad_row"], torch.cat([t.reshape(-1) for t in whole["dw"]]))


@pytest.fixture
def deterministic_head():
    old = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = old


@pytest.mark.parametrize("H0,W0", [(546, 979), (40, 50)])
def test_one_rank_slab_loss_is_L1_loss_appearance_bit_for_bit(H0, W0, deterministic_head):
    from rade_gs_b200 import multigpu
    from rade_gs_b200.appearance import L1_loss_appearance
    inp = _recipe_inputs(H0, W0, 7 + H0)
    runs = []
    for fn in ("whole", "slab"):
        g, image, gt = _setup(inp)
        if fn == "whole":
            loss = L1_loss_appearance(image, gt, g, 2)
        else:
            loss = multigpu.slab_L1_loss_appearance(image, gt, g, 2, (0, H0), all_pixel_rows=[(0, H0)])
        loss.backward()
        runs.append([loss.detach().reshape(1), image.grad, g.table.grad] + [p.grad for p in g.appearance_network.parameters()])
    for i, (a, b) in enumerate(zip(*runs)):
        _bits(f"output {i}", a, b)


@pytest.mark.parametrize("H0,W0", [(546, 979), (40, 50)])
def test_ssim_only_companion_term_is_one_minus_ssim(H0, W0):
    """train.py:160 with --use_decoupled_appearance adds lambda * (1 - ssim): slab_l1_ssim_loss(..., 1.0, rows) weights L1 by 0."""
    from rade_gs_b200 import losses, multigpu
    C = _C()
    x = _inputs(H0, W0, 3)
    a = x["image"].clone().requires_grad_(True)
    b = x["image"].clone().requires_grad_(True)
    slab = multigpu.slab_l1_ssim_loss(a, x["gt"], 1.0, (0, H0))
    ref = 1.0 - losses.ssim(b, x["gt"])
    slab.backward()
    ref.backward()
    assert abs(slab.item() - ref.item()) <= 1e-6
    torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-9)
    # the L1 term contributes nothing, bit for bit: the same loss and gradient as the SSIM kernels called with an L1 weight of 0
    n = x["image"].numel()
    sums, dmaps = C.ssim_l1_forward(x["image"], x["gt"], True, 0, H0)
    # (the fp64 sums accumulate with atomics, so two evaluations may differ in their last bit: allow one float32 rounding)
    torch.testing.assert_close(slab.detach().reshape(1), (1.0 - sums[0:1] / n).float(), rtol=1.2e-7, atol=0.0)
    d = C.ssim_l1_backward(x["image"], x["gt"], dmaps, -1.0 / n, 0.0, torch.empty(0), 0, H0)
    _bits("gradient against the SSIM-only kernel", a.grad, d)


def _row_case():
    x = _inputs(546, 979, 21)
    rows = _partitions(546)["3eq"]

    def run(x):
        s = _slabs(x, rows)
        out = {k: s[k] for k in ("down", "d_image", "d_up4", "loss", "grad_row")}
        out.update({f"act{i}": a for i, (_, _, a) in enumerate(s["acts"])})
        return out
    return Case(x, run)


def test_row_kernels_on_poisoned_memory_and_a_side_stream(poisoned_allocator):
    check_case(_row_case(), poisoned_allocator)


# ---- several GPUs: one sharded training step of the DTU / TNT recipe ------------------------------------------------------

def _int(t):
    return t.contiguous().view(torch.int32)


def _step_worker(rank, world, port, outdir):
    for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    from types import SimpleNamespace
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import losses, multigpu, scenes
    from rade_gs_b200.appearance import L1_loss_appearance
    from test_gpu_appearance import _Net
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    torch.backends.cudnn.deterministic = True     # the head's gradients: the same bits on every rank and in both steps
    torch.backends.cudnn.allow_tf32 = False
    ex = None
    try:
        sc = scenes.make_scene(60000, 640, 400, 500.0, -3.8, seed=21, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.2, 0.1, 0.3)).to(dev)
        sc = multigpu.broadcast_scene_(sc)
        H, W = sc.height, sc.width
        st = dgr.GaussianRasterizationSettings(H, W, sc.tanfovx, sc.tanfovy, 0.1, sc.bg, 1.0, sc.viewmatrix, sc.projmatrix, 3, sc.campos, False,
                                               True, False, False)
        ex = multigpu.GradExchange(sc.means3D.shape[0], dgr._C.grad_stride(False, True), dev)
        inp = _recipe_inputs(H, W, 5)
        gt = inp["gt"].to(dev)
        dist.broadcast(gt, src=0)
        net0 = _Net().to(dev)
        with torch.no_grad():
            for p, v in zip(net0.parameters(), inp["params"]):
                p.copy_(torch.as_tensor(v))
                dist.broadcast(p, src=0)
        table0 = inp["table"].to(dev)
        dist.broadcast(table0, src=0)
        view = SimpleNamespace(FoVx=2 * np.arctan(sc.tanfovx), FoVy=2 * np.arctan(sc.tanfovy), image_height=H, image_width=W)
        lam, lam_n, uid = 0.2, 0.05, 3

        def step(sharded):
            lv = {k: getattr(sc, k).clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
            m2 = torch.zeros_like(lv["means3D"], requires_grad=True)
            net = _Net().to(dev)
            net.load_state_dict(net0.state_dict())
            table = torch.nn.Parameter(table0.clone())
            g = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: table[i])
            rast = multigpu.ShardedGaussianRasterizer(st, exchange=ex, compact=True) if sharded else dgr.GaussianRasterizer(st)
            color, _, _, _, dep, mdep, _, normal = rast(lv["means3D"], m2, lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                                                        rotations=lv["rotations"])
            if sharded:   # INTEGRATION.md section 3, the DTU / TNT recipe
                rows = rast.pixel_rows()
                everyone = [(min(b * 16, H), min(e * 16, H)) for b, e in rast.slabs]
                full = color.new_zeros(3, H, W)        # slab_l1_ssim_loss takes full-size maps
                full[:, rows[0]:rows[1]] = color
                l1 = multigpu.slab_L1_loss_appearance(color, gt, g, uid, rows, all_pixel_rows=everyone)
                ssim_term = multigpu.slab_l1_ssim_loss(full, gt, 1.0, rows)
                nc = multigpu.slab_depth_normal_consistency_loss(view, normal, dep, mdep, rows, all_pixel_rows=everyone)
            else:         # train.py:135-136, :160
                l1 = L1_loss_appearance(color, gt, g, uid)
                ssim_term = 1.0 - losses.ssim(color, gt)
                nc = losses.depth_normal_consistency_loss(view, normal, dep, mdep)
            loss = (1.0 - lam) * l1 + lam * ssim_term + lam_n * nc
            loss.backward()
            grads = {k: v.grad for k, v in lv.items()}
            grads.update({"net." + n: p.grad for n, p in net.named_parameters()})
            grads["embedding"] = table.grad[uid]
            return float(loss), grads

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


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_sharded_step_with_the_appearance_recipe_equals_single(world, tmp_path):
    """Gaussian, network and embedding gradients: the same bits on every rank, and within test_gpu_slab_losses' bars of the
    single-GPU step (world 1 runs the same code path through one slab)."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    import tolerances as tol
    mp.spawn(_step_worker, args=(world, 31800 + os.getpid() % 1000 + world, str(tmp_path)), nprocs=world, join=True)
    for rank in range(world):
        res = np.load(tmp_path / f"step{rank}.npy", allow_pickle=True).item()
        ls, l1 = res.pop("loss")
        assert abs(ls - l1) <= 1e-5 * max(1.0, abs(l1)), (rank, ls, l1)
        names = [k for k in res if not k.endswith("/bits_differ_from_rank0")]
        assert {"embedding", "net.conv1.weight", "net.conv3.bias", "means3D", "shs"} <= set(names)
        for k, v in res.items():
            if k.endswith("/bits_differ_from_rank0"):
                assert v == 0, (rank, k, v)
            else:
                tol.grad_close_gpu(v[0], v[1], f"rank {rank} {k}")
