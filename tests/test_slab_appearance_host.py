"""Slab-local decoupled-appearance L1 loss on CPU (gloo, 2 and 3 ranks): the control flow of rade_gs_b200.multigpu's
`slab_L1_loss_appearance` -- halo exchange, the gathered low-resolution rows, the replicated head, the gathered d(up4) rows, the
rank-order sums -- with fp64 stand-ins for the four row kernels, built on tests/appearance_f64.py.  Each stand-in sees only its
windows (rows outside them are zero), so a halo that is too short changes the result.  The slabs must give the single-process
fp64 model's loss and gradients.  Also the row windows of the C ABI and its host-side rejections.  No GPU."""
import ctypes
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import appearance_f64 as af
from conftest import ROOT

VIEW = 3


class _Up(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.pixel_shuffle = nn.PixelShuffle(2)
        self.conv = nn.Conv2d(cin // 4, cout, 3, padding=1)
        self.relu = nn.ReLU()

    def forward(self, x):
        return self.relu(self.conv(self.pixel_shuffle(x)))


class _Net(nn.Module):
    """scene/appearance_network.py's layers and parameter order."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(67, 256, 3, padding=1)
        self.up1, self.up2, self.up3, self.up4 = _Up(256, 128), _Up(128, 64), _Up(64, 32), _Up(32, 16)
        self.conv2 = nn.Conv2d(16, 16, 3, padding=1)
        self.conv3 = nn.Conv2d(16, 3, 3, padding=1)
        self.relu = nn.ReLU()


def _inputs(H0, W0, seed=11):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(3, H0, W0, generator=g, dtype=torch.float64)
    image = (0.8 * gt + 0.1 + 0.1 * torch.randn(3, H0, W0, generator=g, dtype=torch.float64)).clamp(0, 1)
    table = 0.5 * torch.randn(8, 64, generator=g, dtype=torch.float64)
    params = [torch.randn(*s, generator=g, dtype=torch.float64) * (2.0 / (s[1] * 9)) ** 0.5 if len(s) == 4
              else 0.05 * torch.randn(*s, generator=g, dtype=torch.float64) for s in af.PARAM_SHAPES]
    return image, gt, table, params


def _gaussians(table, params):
    net = _Net().double()
    with torch.no_grad():
        for p, v in zip(net.parameters(), params):
            p.copy_(v)
    t = nn.Parameter(table.clone())
    return SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: t[i], table=t)


def _windows(H0, W0, r0, r1):
    from diff_gaussian_rasterization import _C
    return _C._slab.appearance_row_windows(H0, W0, r0, r1)


def _embed(win, lo, H0):
    """A window of image rows [lo, lo + rows) in a full-size fp64 image that is zero elsewhere."""
    full = np.zeros((3, H0, win.shape[-1]))
    full[:, lo:lo + win.shape[1]] = win.numpy()
    return full


def _resample(x, Ry, Rx):         # af.resample as two matrix products (the same fp64 values up to summation order)
    return np.matmul(np.matmul(Ry, x), Rx.T)


def _resample_T(g, Ry, Rx):
    return np.matmul(np.matmul(Ry.T, g), Rx)


def _crop(full):
    top, left, H, W = af.crop_box(*full.shape[1:])
    return full[:, top:top + H, left:left + W]


class Fp64Rows:
    """include/rgs_b200.h's rgs_appearance_*_rows restated on the fp64 model: each reads only its windows."""

    @staticmethod
    def downsample_rows(win, lo, H0, r0, r1):
        W0 = win.shape[-1]
        _, _, oy_lo, oy_hi = _windows(H0, W0, r0, r1)[:4]
        _, _, H, W = af.crop_box(H0, W0)
        down = _resample(_crop(_embed(win, lo, H0)), af.interp_matrix(H, H // 32), af.interp_matrix(W, W // 32))
        return torch.from_numpy(down[:, oy_lo:oy_hi].copy())

    @staticmethod
    def _tail(up4, act_rows, w2, b2, w3, b3, H, W):
        X = _resample(up4.reshape(16, H // 2, W // 2).numpy(), af.interp_matrix(H // 2, H), af.interp_matrix(W // 2, W))
        A = np.maximum(af.conv(X, w2.numpy(), b2.numpy()), 0)
        if act_rows is not None:   # backward: the activations forward stored, zero outside their window
            lo, act = act_rows
            A = np.zeros_like(A)
            A[:, lo:lo + act.shape[1]] = act.numpy()
        M = 1.0 / (1.0 + np.exp(-af.conv(A, w3.numpy(), b3.numpy())))
        return X, A, M

    @staticmethod
    def l1_forward_rows(win, gt_win, lo, H0, r0, r1, up4, w2, b2, w3, b3):
        W0 = win.shape[-1]
        c0, c1, _, _, _, _, a_lo, a_hi = _windows(H0, W0, r0, r1)[:8]
        _, _, H, W = af.crop_box(H0, W0)
        _, A, M = Fp64Rows._tail(up4, None, w2, b2, w3, b3, H, W)
        err = np.abs(M * _crop(_embed(win, lo, H0)) - _crop(_embed(gt_win, lo, H0)))
        return torch.tensor([err[:, c0:c1].sum()]), torch.from_numpy(A[:, a_lo:a_hi].copy())

    @staticmethod
    def l1_backward_rows(win, gt_win, lo, H0, r0, r1, up4, act, w2, b2, w3, b3, upstream):
        W0 = win.shape[-1]
        c0, c1, _, _, u_lo, u_hi, a_lo = _windows(H0, W0, r0, r1)[:7]
        top, left, H, W = af.crop_box(H0, W0)
        X, A, M = Fp64Rows._tail(up4, (a_lo, act), w2, b2, w3, b3, H, W)
        crop = _crop(_embed(win, lo, H0))
        dT = np.sign(M * crop - _crop(_embed(gt_win, lo, H0))) * (float(upstream) / (3 * H * W))
        own = np.zeros((1, H, 1))
        own[:, c0:c1] = 1.0
        d_image = np.zeros((3, H0, W0))
        d_image[:, top:top + H, left:left + W] = dT * M * own
        dS = dT * crop * (1.0 - M) * M
        dW3, db3 = af.conv_wgrad(dS * own, A)
        dZ = af.conv_T(dS, w3.numpy()) * (A > 0)
        dW2, db2 = af.conv_wgrad(dZ * own, X)
        d_up4 = _resample_T(af.conv_T(dZ, w2.numpy()), af.interp_matrix(H // 2, H), af.interp_matrix(W // 2, W))
        row = np.concatenate([dW2.ravel(), db2, dW3.ravel(), db3])
        return torch.from_numpy(d_image[:, r0:r1].copy()), torch.from_numpy(d_up4[:, u_lo:u_hi].copy()), torch.from_numpy(row)

    @staticmethod
    def downsample_backward_rows(d_down, d_img, H0, r0, r1):
        W0 = d_img.shape[-1]
        top, left, H, W = af.crop_box(H0, W0)
        full = np.zeros((3, H0, W0))
        full[:, top:top + H, left:left + W] = _resample_T(d_down.detach().numpy(), af.interp_matrix(H, H // 32), af.interp_matrix(W, W // 32))
        d_img += torch.from_numpy(full[:, r0:r1].copy())


def _reference(H0, W0):
    image, gt, table, params = _inputs(H0, W0)
    return af.forward_backward(image.numpy(), gt.numpy(), table[VIEW].numpy(), [p.numpy() for p in params])


def _worker(rank, world, port, H0, W0, rows, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        image, gt, table, params = _inputs(H0, W0)
        r0, r1 = rows[rank]
        out = {}
        for compact, everyone in ((False, rows), (True, None)):
            g = _gaussians(table, params)
            if compact:
                leaf = image[:, r0:r1].clone().requires_grad_(True)
            else:
                leaf = torch.zeros_like(image)
                leaf[:, r0:r1] = image[:, r0:r1]   # a full-size sharded render: only the slab's rows are filled
                leaf.requires_grad_(True)
            loss = multigpu.slab_L1_loss_appearance(leaf, gt, g, VIEW, (r0, r1), all_pixel_rows=everyone, kernels=Fp64Rows)
            (2.5 * loss).backward()
            out[compact] = {"loss": loss.detach(), "d_image": leaf.grad, "table": g.table.grad,
                            "grads": [p.grad for p in g.appearance_network.parameters()]}
        torch.save(out, os.path.join(tmpdir, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


CASES = {
    "w2_546_mid_tile": (2, 546, 70, [(0, 288), (288, 546)]),               # crop offset 1, an odd crop row at the cut, last slab cut mid-tile
    "w3_600_outside": (3, 600, 70, [(0, 10), (10, 590), (590, 600)]),      # crop offset 12: two slabs without a crop row
    "w3_546_four_rows": (3, 546, 67, [(0, 101), (101, 105), (105, 546)]),  # a middle slab of exactly the halo's 4 rows
    "w3_600_weighted": (3, 600, 70, None),                                 # weighted: one rank holds every row, two end empty
}


def _rows(world, H0, rows):
    if rows is not None:
        return rows
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    n = multigpu.tile_rows(H0)
    slabs = multigpu.partition_tile_rows(n, world, [0.0] * (n - 1) + [1.0])
    return [(min(b * 16, H0), min(e * 16, H0)) for b, e in slabs]


@pytest.mark.parametrize("case", list(CASES))
def test_slab_appearance_equals_the_whole_image_fp64(case, tmp_path):
    world, H0, W0, rows = CASES[case]
    rows = _rows(world, H0, rows)
    assert rows[0][0] == 0 and rows[-1][1] == H0
    port = 43500 + (os.getpid() % 1500) + 7 * world + H0 % 7 + len(case)
    mp.spawn(_worker, args=(world, port, H0, W0, rows, str(tmp_path)), nprocs=world, join=True)
    res = [torch.load(tmp_path / f"rank{r}.pt") for r in range(world)]
    m = _reference(H0, W0)

    def close(got, ref, what):
        ref = torch.as_tensor(np.asarray(ref, np.float64)) * 2.5
        tol = 1e-12 * max(1.0, float(ref.abs().max()) if ref.numel() else 0.0)
        assert got.shape == ref.shape, what
        err = float((got - ref).abs().max()) if got.numel() else 0.0
        assert err <= tol, (what, err, tol)

    for compact in (False, True):
        outs = [r[compact] for r in res]
        for rank, (o, (r0, r1)) in enumerate(zip(outs, rows)):
            assert o["loss"].dtype == torch.float64
            assert abs(float(o["loss"]) - float(m["loss"])) <= 1e-12, (rank, float(o["loss"]), float(m["loss"]))
            d = o["d_image"] if compact else o["d_image"][:, r0:r1]
            close(d, m["d_image"][:, r0:r1], f"rank {rank} d_image")
            if not compact:
                rest = o["d_image"].clone()
                rest[:, r0:r1] = 0
                assert not rest.any()        # a rank's gradient lives in its own rows only
            close(o["table"][VIEW], m["d_emb"], f"rank {rank} embedding")
            assert not torch.cat([o["table"][:VIEW], o["table"][VIEW + 1:]]).any()
            for name, gr, ref in zip(af.PARAM_NAMES, o["grads"], m["grads"]):
                close(gr, ref, f"rank {rank} {name}")
        # the same bits on every rank
        for o in outs[1:]:
            assert torch.equal(o["loss"], outs[0]["loss"]) and torch.equal(o["table"], outs[0]["table"])
            assert all(torch.equal(a, b) for a, b in zip(o["grads"], outs[0]["grads"]))


def _refusal_worker(rank, world, port, H0, rows, give_rows, tmpdir):
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        image, gt, table, params = _inputs(H0, 40)
        r0, r1 = rows[rank]
        try:
            multigpu.slab_L1_loss_appearance(image[:, r0:r1], gt, _gaussians(table, params), VIEW, (r0, r1),
                                             all_pixel_rows=rows if give_rows else None, kernels=Fp64Rows)
            what = "no error"
        except ValueError as e:
            what = str(e)
        dist.barrier()   # every rank got here: nobody waits in an exchange
        torch.save(what, os.path.join(tmpdir, f"refusal{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("give_rows", [True, False], ids=["all_pixel_rows", "gathered_rows"])
def test_every_rank_refuses_a_short_middle_slab(give_rows, tmp_path):
    """A middle slab of 3 rows cannot send its neighbours their 4 halo rows.  Given every rank's rows, all ranks raise before any
    collective; without them, all ranks raise after gathering the rows and before the exchange."""
    world, H0, rows = 3, 96, [(0, 40), (40, 43), (43, 96)]
    port = 45500 + (os.getpid() % 1500) + int(give_rows)
    mp.spawn(_refusal_worker, args=(world, port, H0, rows, give_rows, str(tmp_path)), nprocs=world, join=True)
    for r in range(world):
        what = torch.load(tmp_path / f"refusal{r}.pt")
        assert "at least 4 pixel rows" in what, what


def test_single_process_refusals():
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    image, gt, table, params = _inputs(64, 40)
    g = _gaussians(table, params)
    with pytest.raises(ValueError, match="transformed"):
        multigpu.slab_L1_loss_appearance(image, gt, g, VIEW, (0, 64), return_transformed_image=True, kernels=Fp64Rows)
    with pytest.raises(RuntimeError, match="CUDA"):
        multigpu.slab_L1_loss_appearance(image.float(), gt.float(), g, VIEW, (0, 64))
    with pytest.raises(ValueError, match="ground truth"):
        multigpu.slab_L1_loss_appearance(image, gt.clone().requires_grad_(True), g, VIEW, (0, 64), kernels=Fp64Rows)
    with pytest.raises(ValueError, match="image_height"):
        multigpu.slab_L1_loss_appearance(image, gt, g, VIEW, (0, 64), image_height=63, kernels=Fp64Rows)
    with pytest.raises(ValueError, match="slab's rows"):
        multigpu.slab_L1_loss_appearance(image[:, :20], gt, g, VIEW, (0, 32), rank=0, world_size=2, all_pixel_rows=[(0, 32), (32, 64)], kernels=Fp64Rows)
    with pytest.raises(ValueError, match="not rows"):
        multigpu.slab_L1_loss_appearance(image, gt, g, VIEW, (32, 80), kernels=Fp64Rows)
    with pytest.raises(ValueError, match="all_pixel_rows"):
        multigpu.slab_L1_loss_appearance(image, gt, g, VIEW, (0, 32), rank=0, world_size=2, all_pixel_rows=[(0, 32), (40, 64)], kernels=Fp64Rows)


def test_single_process_slab_is_the_whole_image():
    sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
    from rade_gs_b200 import multigpu
    H0, W0 = 99, 67
    image, gt, table, params = _inputs(H0, W0)
    g = _gaussians(table, params)
    leaf = image.clone().requires_grad_(True)
    loss = multigpu.slab_L1_loss_appearance(leaf, gt, g, VIEW, (0, H0), kernels=Fp64Rows)
    loss.backward()
    m = _reference(H0, W0)
    assert abs(float(loss) - m["loss"]) <= 1e-12
    torch.testing.assert_close(leaf.grad, torch.from_numpy(m["d_image"]), rtol=1e-10, atol=1e-15)
    for p, ref in zip(g.appearance_network.parameters(), m["grads"]):
        torch.testing.assert_close(p.grad, torch.from_numpy(np.asarray(ref)), rtol=1e-10, atol=1e-14)


# ---- the row windows and the C ABI ---------------------------------------------------------------------------------------------

def _gather_reads(H):
    """For each up4 row u, the crop rows the gather (upsample_transpose_kernel) reads: those whose fp32 taps name u."""
    Hu = H // 2
    sy = np.float32(Hu - 1) / np.float32(H - 1)
    y = np.arange(H)
    i0 = (sy * y.astype(np.float32)).astype(np.int64)
    i1 = i0 + (i0 < Hu - 1)
    return [y[(i0 == u) | (i1 == u)] for u in range(Hu)]


def test_upsample_gather_reads_rows_2u_minus_2_to_2u_plus_2():
    """The tight bound the row windows rest on: the gather of up4 row u reads crop rows [2u - 2, 2u + 2] and no others, and both
    ends occur (the 2u - 2 read has weight 0: its lower tap is u - 1 exactly, so only u's weight, 0, multiplies it)."""
    lo_seen, hi_seen = set(), set()
    for H in list(range(32, 4096 + 1, 32)) + [8192, 16384]:
        for u, ys in enumerate(_gather_reads(H)):
            assert ys.min() >= 2 * u - 2 and ys.max() <= 2 * u + 2, (H, u, ys)
            lo_seen.add(int(ys.min()) - 2 * u)
            hi_seen.add(int(ys.max()) - 2 * u)
    assert min(lo_seen) == -2 and max(hi_seen) == 2


@pytest.mark.parametrize("H0,W0", [(546, 979), (600, 800), (1200, 1600), (40, 50), (33, 64)])
def test_row_windows_partition_and_cover_what_the_kernels_read(H0, W0):
    top, _, H, _ = af.crop_box(H0, W0)
    h = H // 32
    scy = np.float32(H - 1) / np.float32(h - 1) if h > 1 else np.float32(0)
    upper = (scy * np.arange(h, dtype=np.float32)).astype(np.int64)     # the downsample's upper tap, as the kernel computes it
    reads = _gather_reads(H)
    for cuts in ([0, H0], [0, H0 // 3, H0 // 2, H0], [0, 5, 17, 250 % H0 + 20, H0], [0, top + 1, H0 - 4, H0, H0]):
        cuts = sorted(set(min(c, H0) for c in cuts)) + ([H0] if cuts.count(H0) > 1 else [])
        oy_seen, u_seen = [], []
        for r0, r1 in zip(cuts[:-1], cuts[1:]):
            c0, c1, oy_lo, oy_hi, u_lo, u_hi, a_lo, a_hi, x_lo, x_hi, i_lo, i_hi = _windows(H0, W0, r0, r1)
            assert (c0, c1) == (min(max(r0 - top, 0), H), min(max(r1 - top, 0), H))
            oy_seen += range(oy_lo, oy_hi)
            u_seen += range(u_lo, u_hi)
            for oy in range(oy_lo, oy_hi):
                assert c0 <= upper[oy] < c1
            for u in range(u_lo, u_hi):
                assert c0 <= 2 * u < c1 and x_lo <= reads[u].min() and reads[u].max() < x_hi
            if c1 > c0:
                assert (x_lo, x_hi) == (max(0, c0 - 2), min(H, c1 + 2))
                assert (i_lo, i_hi) == (max(0, x_lo - 2), min(H, x_hi + 2))   # d(conv2) one row out, the loss derivative two
                assert (a_lo, a_hi) == (max(0, i_lo - 1), min(H, i_hi + 1))   # conv3 reads one row beyond the loss derivative
            else:
                assert oy_hi == oy_lo and u_hi == u_lo and a_hi == a_lo and x_hi == x_lo and i_hi == i_lo
        assert oy_seen == list(range(h)) and u_seen == list(range(H // 2))   # each row owned exactly once


def _lib():
    lib = ctypes.CDLL(os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so"))
    lib.rgs_last_error.restype = ctypes.c_char_p
    return lib


def test_c_abi_rejects_bad_rows_windows_and_null_pointers():
    lib = _lib()
    i32 = ctypes.c_int32
    fake = ctypes.c_void_p(0x1000)   # never dereferenced: rejected before the first CUDA call
    H0, W0 = 600, 800                # crop rows [12, 588)

    def fwd(r0, r1, lo, rows, **null):
        a = dict(image=fake, gt=fake, up4=fake, w2=fake, b2=fake, w3=fake, b3=fake, act=fake, partials=fake, loss_sum=fake)
        a.update(null)
        return lib.rgs_appearance_l1_forward_rows(i32(H0), i32(W0), i32(r0), i32(r1), a["image"], a["gt"], i32(lo), i32(rows), a["up4"], a["w2"],
                                                  a["b2"], a["w3"], a["b3"], a["act"], a["partials"], a["loss_sum"], None)

    def bwd(r0, r1, lo, rows, **null):
        a = dict(image=fake, gt=fake, up4=fake, act=fake, w2=fake, w3=fake, b3=fake, d_image=fake, d_up4=fake, grad_row=fake, partials=fake, d_x=fake)
        a.update(null)
        return lib.rgs_appearance_l1_backward_rows(i32(H0), i32(W0), i32(r0), i32(r1), a["image"], a["gt"], i32(lo), i32(rows), a["up4"], a["act"],
                                                   a["w2"], a["w3"], a["b3"], None, a["d_image"], a["d_up4"], a["grad_row"], a["partials"], a["d_x"],
                                                   None)

    def down(r0, r1, lo, rows, image=fake):
        return lib.rgs_appearance_downsample_rows(i32(H0), i32(W0), i32(r0), i32(r1), image, i32(lo), i32(rows), fake, None)

    def rejected(rc, text):
        assert rc == -1 and text in lib.rgs_last_error(), lib.rgs_last_error()

    # row ranges outside the image
    rejected(fwd(100, 700, 96, 500), b"row range")
    rejected(bwd(-1, 100, 0, 104), b"row range")
    rejected(down(300, 200, 296, 8), b"row range")
    rejected(lib.rgs_appearance_downsample_backward_rows(i32(H0), i32(W0), i32(0), i32(601), fake, fake, None), b"row range")
    rejected(lib.rgs_appearance_row_windows(i32(H0), i32(W0), i32(10), i32(5), fake), b"row range")
    rejected(lib.rgs_appearance_row_windows(i32(31), i32(W0), i32(0), i32(31), fake), b"at least 32")
    # null pointers
    rejected(fwd(100, 200, 96, 108, loss_sum=None), b"null")
    rejected(fwd(100, 200, 96, 108, act=None), b"null")
    rejected(bwd(100, 200, 96, 108, grad_row=None), b"null")
    rejected(bwd(100, 200, 96, 108, d_x=None), b"null")
    rejected(down(100, 200, 100, 101, image=None), b"null")
    rejected(lib.rgs_appearance_downsample_backward_rows(i32(H0), i32(W0), i32(0), i32(16), None, fake, None), b"null")
    rejected(lib.rgs_appearance_row_windows(i32(H0), i32(W0), i32(0), i32(16), None), b"null")
    # windows that are not inside the image
    rejected(fwd(100, 200, -4, 208), b"not inside")
    rejected(bwd(500, 600, 496, 108), b"not inside")
    rejected(down(0, 100, 0, 601), b"not inside")
    # halos too short: forward needs the slab's crop rows, backward 4 rows either side, the downsample one row below
    rejected(fwd(100, 200, 101, 99), b"lacks halo rows")
    rejected(bwd(100, 200, 100, 100), b"lacks halo rows")
    rejected(bwd(100, 200, 97, 107), b"lacks halo rows")
    rejected(bwd(100, 200, 96, 107), b"lacks halo rows")
    rejected(down(100, 200, 100, 100), b"lacks halo rows")
    # a slab without crop rows needs no window and launches nothing, so fake pointers are never touched
    w = (ctypes.c_int32 * 12)()
    assert lib.rgs_appearance_row_windows(i32(H0), i32(W0), i32(0), i32(10), w) == 0 and list(w)[:2] == [0, 0]
    assert down(0, 10, 0, 0) == 0
