"""Tile-row sharding of one camera across the GPUs of a box (SURVEY.md 8e; the reference is single-GPU only).

Every rank holds the full Gaussian set and runs preprocess on all of it (identical on every rank); rank r bins,
sorts and blends only the tile rows of its slab, so the union of the per-rank sorted lists is the reference's
list.  Backward has exactly one exchange step: the packed screen-space gradient rows written by
backward-render are plain sums over pixels, hence additive across slabs -- they are summed once over the ranks
and only then turned into parameter gradients.  The sum has to sit before backward-preprocess, not after it: with
kernel_size > 0 that stage multiplies two accumulated quantities (the reference's mip-gradient aliasing, SURVEY.md
A-14), so per-slab results would not add up to the single-GPU answer.

The sum is `GradExchange`'s device-side peer exchange or, without one and as its fallback, one all-reduce
(`allreduce_sum_`: NCCL on GPUs, gloo in the CPU tests, which run it with the oracle's stages in place of the CUDA ones).
"""
from __future__ import annotations

import math
import os
from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist

from .rawapi import backward_args, forward_args, preprocess_args

TILE = 16


def tile_rows(height: int) -> int:
    return (height + TILE - 1) // TILE


def partition_tile_rows(grid_y: int, world_size: int, weights: Sequence[float] | None = None) -> List[Tuple[int, int]]:
    """Contiguous [begin, end) tile-row slabs, one per rank.

    Without weights rows are split as evenly as possible (earlier ranks take the remainder, e.g. 68 rows over 8
    ranks -> 9,9,9,9,8,8,8,8).  With per-row weights (e.g. instances per tile row from a previous frame) the cut
    points equalise the weight prefix sums; every rank still gets a (possibly empty) contiguous range and the
    ranges tile [0, grid_y) exactly.
    """
    if world_size <= 0:
        raise ValueError("world_size must be positive")
    if weights is None:
        base, rem = divmod(grid_y, world_size)
        out, b = [], 0
        for r in range(world_size):
            e = b + base + (1 if r < rem else 0)
            out.append((b, e))
            b = e
        return out
    if len(weights) != grid_y:
        raise ValueError("need one weight per tile row")
    total = float(sum(weights))
    if total <= 0:
        return partition_tile_rows(grid_y, world_size)
    cuts, acc, r = [0], 0.0, 1
    for y, w in enumerate(weights):
        acc += float(w)
        while r < world_size and acc >= total * r / world_size:
            cuts.append(y + 1)
            r += 1
    while len(cuts) < world_size:
        cuts.append(grid_y)
    cuts.append(grid_y)
    return [(cuts[i], max(cuts[i], cuts[i + 1])) for i in range(world_size)]


def _rank_world(rank, world_size, group):
    """(rank, world size) in `group`: an explicit argument wins; without an initialised process group this is rank 0 of 1."""
    if world_size is None:
        world_size = dist.get_world_size(group) if dist.is_initialized() else 1
    if rank is None:
        rank = dist.get_rank(group) if dist.is_initialized() else 0
    return rank, world_size


def allreduce_sum_(t: torch.Tensor, group=None) -> torch.Tensor:
    """In-place sum over ranks; a no-op outside an initialised process group (single-GPU path)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def broadcast_scene_(scene, src: int = 0, group=None):
    """Make a replicated scene (any object whose tensor attributes are the model / camera state) bit-identical on every rank by
    broadcasting rank `src`'s copy -- what a trainer does with its replicated parameters.  Data-parallel slabs only compose to the
    single-GPU image if every rank rasterizes THE SAME numbers: two processes that each synthesise "the same" scene on their CPUs can
    differ in the last bits (threaded vectorised exp / sigmoid / matmul tails), and a few-ulp difference in one splat is a visible
    few-pixel difference in the gathered image."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return scene
    for k, v in list(vars(scene).items()):
        if isinstance(v, torch.Tensor):
            t = v.contiguous()
            dist.broadcast(t, src=src, group=group)
            setattr(scene, k, t)
    return scene


class GradExchange:
    """The one exchange step of the sharded backward: slab-local accumulator rows -> summed rows on every rank.

    ``peer`` (default on CUDA with NCCL): the library's device-side exchange over peer memory (csrc/rgs_exchange.cu: touched
    rows are reduced into their owner rank with vector reductions through NVLink, the sums are spread to every rank, two
    flag barriers, no host synchronisation; bit-identical rows on all ranks).  torch.distributed is used ONCE, to all-gather
    the 64-byte IPC handles.  ``dense`` (``RGS_GRAD_EXCHANGE=dense``, and the only mode off-GPU or with one rank): stage 1 into
    a fresh tensor + one NCCL / gloo all-reduce of the whole tensor.  Any other mode raises ``ValueError``.

    All ranks must create the object collectively and call ``backward_render`` the same number of times with the same P.
    """

    def __init__(self, capacity_rows: int, row_floats: int, device, group=None, mode: str | None = None):
        self.group, self.device = group, torch.device(device)
        self.rank, self.world = _rank_world(None, None, group)
        mode = mode or os.environ.get("RGS_GRAD_EXCHANGE", "peer")
        if mode not in ("peer", "dense"):
            raise ValueError(f"gradient exchange mode must be 'peer' or 'dense', got {mode!r}")
        if self.world == 1 or self.device.type != "cuda":
            mode = "dense"
        self.mode, self.capacity, self.row_floats, self._ex = mode, int(capacity_rows), int(row_floats), None
        self.window = None
        if mode == "peer":
            from diff_gaussian_rasterization import _C
            idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
            self._ex, handle = _C.exchange_create(self.rank, self.world, self.capacity, self.row_floats, idx)
            mine = handle.to(self.device)
            gathered = [torch.empty_like(mine) for _ in range(self.world)]
            dist.all_gather(gathered, mine, group=group)
            _C.exchange_connect(self._ex, torch.stack(gathered).cpu(), idx)
            self.window = "cuda-ipc"
            dist.barrier(group=group)   # nobody pushes before every rank has mapped every window
            why = self._self_check(_C, idx)
            if why is not None:         # the same verdict on every rank (all-reduced): fall back together
                import warnings
                warnings.warn(f"peer gradient exchange failed its self-check ({why}); using the dense all-reduce")
                self.fallback_reason = why
                self.mode = "dense"

    fallback_reason = None

    def _self_check(self, C, idx):
        """Two synthetic exchange steps with a known answer before the object is trusted: rank r touches every 3rd row starting at
        (r + step) % 3 (+ row 0, touched by all) and fills it with f(step, rank, row); the result must be the sum over the ranks that
        touched the row, bit for bit (small integers: exact in float), on every rank.  Returns None or the reason of the failure."""
        P = min(self.capacity, 4096 + 17)
        dev = torch.device("cuda", idx)
        rows = torch.arange(P, device=dev)
        radii = torch.ones(P, dtype=torch.int32, device=dev)
        radii[5::11] = 0                                         # rows nobody renders are neither pushed nor spread
        ok = True
        try:
            for step in (1, 2):
                expect = torch.zeros(P, self.row_floats, device=dev)
                mine = None
                for r in range(self.world):
                    touched = ((rows % 3) == ((r + step) % 3)) | (rows == 0)   # step 2 leaves some of step 1's rows untouched: they must read zero again
                    touched &= radii > 0
                    val = (touched.float() * (step * 64 + r + 1))[:, None] * (1 + (rows % 7).float())[:, None] * torch.ones(1, self.row_floats, device=dev)
                    expect += val
                    if r == self.rank:
                        mine = (touched, val)
                acc = C.exchange_accumulator(self._ex, P, self.row_floats, idx)
                acc.copy_(mine[1])
                C.exchange_rows(self._ex, mine[0].int(), radii)
                if C.exchange_status(self._ex) != 0:
                    ok = False
                    break
                got = C.exchange_result(self._ex, P, self.row_floats, idx)
                vis = radii > 0
                if not torch.equal(got[vis], expect[vis]) or bool(acc.any()):
                    ok = False
                    break
        except Exception as e:   # noqa: BLE001  (a failing CUDA call: report, fall back)
            ok = False
            why_local = f"{type(e).__name__}: {e}"
        flag = torch.tensor([1 if ok else 0], device=dev, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 1:
            return None
        return "a rank saw a wrong result or a barrier timeout" if ok else locals().get("why_local", "wrong result or barrier timeout on this rank")

    def backward_render(self, C, *stage1_args) -> torch.Tensor:
        """stage 1 (`rasterize_gaussians_backward_render` arguments) + exchange -> summed accumulator rows [P, row_floats]."""
        if self.mode == "peer":
            return C.rasterize_gaussians_backward_render_exchange(self._ex, *stage1_args)
        return allreduce_sum_(C.rasterize_gaussians_backward_render(*stage1_args), self.group)

    def close(self):
        if self._ex is not None:
            from diff_gaussian_rasterization import _C
            if dist.is_initialized():
                dist.barrier(group=self.group)   # peers may still be reading / writing this rank's window
            _C.exchange_destroy(self._ex)
            self._ex = None


class _ShardedRasterize(torch.autograd.Function):
    """Autograd node of the row-sharded rasterizer; same argument / gradient order as the single-GPU
    `_RasterizeGaussians` (reference: diff_gaussian_rasterization/__init__.py:44-169)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, slab, group, exchange=None,
                compact=False, balance=None):
        from diff_gaussian_rasterization import _C
        s = raster_settings
        args = forward_args(s, means3D, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh)
        if balance is not None:   # (rank, world_size, plan): the slab is cut from this frame's tile counts and reported in `plan`
            rank, world_size, plan = balance
            out = _C._slab.rasterize_balanced(*args, world_size, rank, compact)
            cuts, plan["row_stats"] = out[12], out[13]
            plan["slabs"] = [(cuts[r], cuts[r + 1]) for r in range(world_size)]
            slab = plan["slabs"][rank]
            out = out[:12]
        else:
            out = _C.rasterize_gaussians_slab(*args, *slab, compact)
        num_rendered, color, coord, mcoord, alpha, normal, depth, mdepth, radii, geom, binning, img = out
        ctx.s, ctx.slab, ctx.compact, ctx.group, ctx.num_rendered, ctx.exchange = s, slab, compact, group, num_rendered, exchange
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh, geom, binning, img, alpha, opacities)
        return color, radii, coord, mcoord, depth, mdepth, alpha, normal

    @staticmethod
    def backward(ctx, g_color, g_radii, g_coord, g_mcoord, g_depth, g_mdepth, g_alpha, g_normal):
        from diff_gaussian_rasterization import _C
        s = ctx.s
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, normal, radii, sh, geom, binning, img, alpha, opacities = ctx.saved_tensors
        stage1_args = backward_args(s, means3D, radii, colors_precomp, scales, rotations, cov3Ds_precomp,
                                    (g_color, g_coord, g_mcoord, g_depth, g_mdepth, g_alpha, g_normal), normal, sh, geom, ctx.num_rendered,
                                    binning, img, alpha) + (*ctx.slab, ctx.compact, s.image_height)
        # the device-side exchange (or its dense fallback) owned by the caller, else one all-reduce
        acc = (ctx.exchange.backward_render(_C, *stage1_args) if ctx.exchange is not None
               else allreduce_sum_(_C.rasterize_gaussians_backward_render(*stage1_args), ctx.group))
        g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rot = _C.rasterize_gaussians_backward_preprocess(
            *preprocess_args(s, acc, means3D, radii, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, sh, geom))
        return g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rot, g_cov3D, None, None, None, None, None, None


def _gather_rows(mine: torch.Tensor, ranges, n_rows: int, group) -> torch.Tensor:
    """The whole [C, n_rows, ...] map from each rank's rows `ranges[r]` (`mine` holds this rank's): an all-gather of pure copies,
    so every rank holds the bits their owners computed."""
    if len(ranges) == 1:
        return mine
    hmax = max(e - b for b, e in ranges)
    buf = mine.new_zeros(mine.shape[0], hmax, *mine.shape[2:])
    buf[:, :mine.shape[1]] = mine
    parts = [torch.empty_like(buf) for _ in ranges]
    dist.all_gather(parts, buf, group=group)
    out = mine.new_empty(mine.shape[0], n_rows, *mine.shape[2:])
    for (b, e), p in zip(ranges, parts):
        out[:, b:e] = p[:, :e - b]
    return out


class _SlabLayout:
    """How a rank's maps hold its pixel rows [r0, r1) of an H-row image: compact maps ([C, r1 - r0, W]) hold only those rows,
    full-size ones ([C, H, W]) all rows with the slab's filled.  The two coincide when the slab is the whole image."""

    def __init__(self, t, H, r0, r1):   # the layout of map `t`
        self.H, self.r0, self.r1, self.compact = H, r0, r1, t.shape[-2] != H

    @staticmethod
    def check(maps, H, r0, r1, W, together=None):
        """Raise unless every map of `maps` [(name, tensor, channels)] is [channels, H or r1 - r0 rows, W], all in one layout."""
        for name, t, c in maps:
            if t.dim() != 3 or t.shape[0] != c or t.shape[-1] != W or t.shape[-2] not in (H, r1 - r0):
                raise ValueError(f"{name} must be [{c}, {H} or {r1 - r0} rows, {W}] (full-size or the slab's rows), got {tuple(t.shape)}")
        if len({t.shape[-2] for _, t, _ in maps}) != 1:
            raise ValueError(f"{together} must all be full-size or all hold the slab's rows")

    def own(self, t):   # the slab's rows of map `t`, detached
        return t.detach() if self.compact else t.detach()[:, self.r0:self.r1]

    def full(self, rows):   # the slab's rows [C, r1 - r0, W] in a full-size map, zero elsewhere
        out = rows.new_zeros(rows.shape[0], self.H, rows.shape[-1])
        out[:, self.r0:self.r1] = rows
        return out


class _GatherSlabs(torch.autograd.Function):
    """All-gather of the ranks' slab rows into the whole map (pure copies: the gathered map holds exactly the bits each
    rank rendered); identity backward (every rank holds the same full-image loss, and a rank's backward reads only the rows
    of its own slab)."""

    @staticmethod
    def forward(ctx, img, group, pixel_rows, rank):
        if not (dist.is_available() and dist.is_initialized()) or len(pixel_rows) == 1:
            return img.detach().clone()
        return _gather_rows(img.detach()[:, slice(*pixel_rows[rank])], pixel_rows, img.shape[1], group)

    @staticmethod
    def backward(ctx, grad_out):
        return grad_out, None, None, None


class ShardedGaussianRasterizer(torch.nn.Module):
    """`GaussianRasterizer` whose work is split by tile rows over the ranks of a process group.

    Each rank returns full-size maps of which only its slab rows are filled (the rest is zero) or, with ``compact=True``, maps
    that hold only the slab's pixel rows ([C, rows, W]); callers that need the whole image gather the slabs (`gather_image`).  Gradients returned on every rank are the full,
    already-reduced parameter gradients.

    ``balance=True`` cuts the slabs anew in every forward call from that frame's instances per tile row (include/rgs_b200.h's
    partition rule; every rank derives the same partition without communicating).  After a forward, `slabs`, `slab`,
    `pixel_rows()` and `all_pixel_rows()` describe that frame, `row_stats` holds its [2, tile rows] instances and longest tile
    list per row, and `gather_image` uses its partition; the backward of a frame uses the slab chosen at its forward.  Every slab
    holds at least one tile row, so the image needs at least `world_size` tile rows.  Cannot be combined with ``row_weights``.
    """

    def __init__(self, raster_settings, rank: int | None = None, world_size: int | None = None, group=None, row_weights=None,
                 exchange: GradExchange | None = None, compact: bool = False, balance: bool = False):
        super().__init__()
        if balance and row_weights is not None:
            raise ValueError("balance=True cuts the slabs from each frame's tile counts: it cannot be combined with row_weights")
        self.compact = compact     # True: the returned maps are [C, slab rows, W] (per-rank image memory and fill scale with 1/ranks)
        self.raster_settings = raster_settings
        self.group = group
        self.exchange = exchange   # a GradExchange created once by the caller (collective); None: one dense all-reduce per backward
        self.rank, self.world_size = rank, world_size = _rank_world(rank, world_size, group)
        self.balance = bool(balance)
        grid_y = tile_rows(raster_settings.image_height)
        if self.balance and grid_y < world_size:
            raise ValueError(f"balance=True gives every rank at least one tile row: {grid_y} tile rows cannot serve {world_size} ranks")
        self.slabs = partition_tile_rows(grid_y, world_size, row_weights)   # with balance: until the first forward
        self.slab = self.slabs[rank]
        self.row_stats = None

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        from diff_gaussian_rasterization import _inputs
        shs, colors_precomp, scales, rotations, cov3D_precomp = _inputs(shs, colors_precomp, scales, rotations, cov3D_precomp)
        plan = {}
        out = _ShardedRasterize.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                      self.raster_settings, self.slab, self.group, self.exchange, self.compact,
                                      (self.rank, self.world_size, plan) if self.balance else None)
        if self.balance:
            self.slabs, self.row_stats = plan["slabs"], plan["row_stats"]
            self.slab = self.slabs[self.rank]
        return out

    def pixel_rows(self) -> Tuple[int, int]:
        H = self.raster_settings.image_height
        return min(self.slab[0] * TILE, H), min(self.slab[1] * TILE, H)

    def all_pixel_rows(self) -> List[Tuple[int, int]]:
        """Every rank's pixel rows, in rank order: the `all_pixel_rows` argument of the slab losses."""
        H = self.raster_settings.image_height
        return [(min(b * TILE, H), min(e * TILE, H)) for b, e in self.slabs]

    def gather_image(self, img: torch.Tensor) -> torch.Tensor:
        """The whole [C,H,W] map from the ranks' slabs (all-gather of the slab rows; rows outside a rank's slab are zero locally).

        Differentiable: with the whole image on every rank an unchanged full-image loss (train.py:130-165: L1, SSIM,
        normal consistency) can be evaluated redundantly per rank; its gradient flows back unchanged and the sharded
        rasterizer's backward reads only the rows of its own slab, so nothing is counted twice.
        """
        rows = self.all_pixel_rows()
        if self.compact:   # [C, slab rows, W] -> place into a full-size map first (the gather copies slab rows only)
            img = _SlabLayout(img, self.raster_settings.image_height, *rows[self.rank]).full(img)
        return _GatherSlabs.apply(img, self.group, rows, self.rank)


# ---- slab-local image loss with halo rows (SURVEY.md 8f-2, multi-GPU half) ----------------------------------------------------
HALO = 5   # 11x11 SSIM window (utils/loss_utils.py:35: window_size=11, padding 5)


def _exchange_rows(t: torch.Tensor, send_up, send_down, recv_up, recv_down, rank: int, world: int, group, add: bool):
    """Neighbour exchange of row blocks of a [C,H,W] tensor: rows `send_up` go to rank-1, `send_down` to rank+1; what the
    neighbours send lands in rows `recv_up` (from rank-1) / `recv_down` (from rank+1), overwriting or (add=True) accumulating."""
    ops, bufs = [], []
    for peer, srows, rrows in ((rank - 1, send_up, recv_up), (rank + 1, send_down, recv_down)):
        if peer < 0 or peer >= world:
            continue
        if srows[1] > srows[0]:
            ops.append(dist.P2POp(dist.isend, t[:, srows[0]:srows[1]].contiguous(), peer, group=group))
        if rrows[1] > rrows[0]:
            buf = torch.empty_like(t[:, rrows[0]:rrows[1]]).contiguous()
            bufs.append((rrows, buf))
            ops.append(dist.P2POp(dist.irecv, buf, peer, group=group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    for (r0, r1), buf in bufs:
        if add:
            t[:, r0:r1] += buf
        else:
            t[:, r0:r1] = buf


def _exchange_halo(t: torch.Tensor, lo: int, r0: int, r1: int, H: int, halo: int, rank: int, world: int, group, backward: bool = False):
    """The `halo`-row exchange of the rank owning pixel rows [r0, r1) of an H-row image, on `t` holding image rows [lo, lo + t.shape[1]).
    Forward: the slab's first and last min(halo, r1 - r0) rows go up and down (not down when the slab ends at the image's last row:
    the ranks after it hold empty slabs), and the neighbours' rows fill [max(0, r0 - halo), r0) and [r1, min(H, r1 + halo)).
    Backward: the reverse, rows outside [r0, r1) go to their owners and are added into the slab's edge rows.  An empty slab exchanges nothing."""
    if r1 <= r0:
        return
    k = min(halo, r1 - r0)
    edges = ((r0, r0 + k), (r1 - k, r1) if r1 < H else (r1, r1))
    halos = ((max(0, r0 - halo), r0), (r1, min(H, r1 + halo)))
    send, recv = (halos, edges) if backward else (edges, halos)
    _exchange_rows(t, *((b - lo, e - lo) for b, e in send + recv), rank, world, group, add=backward)


def _halo_window(maps, layout: _SlabLayout, halo: int, rank: int, world: int, group):
    """(window, lo): `maps`' rows [lo = max(0, r0 - halo), min(H, r1 + halo)) stacked along channels, the halo rows exchanged."""
    lo = max(0, layout.r0 - halo)
    win = maps[0].new_zeros(sum(m.shape[0] for m in maps), min(layout.H, layout.r1 + halo) - lo, maps[0].shape[-1])
    for part, m in zip(win.split([m.shape[0] for m in maps]), maps):
        part[:, layout.r0 - lo:layout.r1 - lo] = layout.own(m)
    _exchange_halo(win, lo, layout.r0, layout.r1, layout.H, halo, rank, world, group)
    return win, lo


class _SlabSsimL1(torch.autograd.Function):
    """(1 - l) * L1 + l * (1 - SSIM) of the WHOLE image (train.py:163), evaluated slab by slab: a rank counts the SSIM-map and L1
    rows of its own slab; the 11x11 window reaches 5 rows into the neighbours' slabs, so 5 halo rows travel to each neighbour in
    forward and the gradient a rank holds for its neighbours' halo pixels travels back (and is added) in backward.  Two scalars are
    all-reduced; the image itself is never gathered.  `fwd` / `bwd` are the per-slab kernels (CUDA kernels in the product,
    torch expressions in the CPU test): fwd(img, gt, r0, r1, need_grad) -> (sums[2] float64, state), bwd(img, gt, state, w_ssim,
    w_l1, r0, r1) -> d_img [C,H,W] (non-zero in rows [r0-5, r1+5) only)."""

    @staticmethod
    def forward(ctx, image, gt, lambda_dssim, rows, rank, world, group, fwd, bwd):
        r0, r1 = rows
        H = image.shape[-2]
        img = image.detach().clone()
        # my first / last 5 rows are the neighbours' halos; theirs are mine
        _exchange_halo(img, 0, r0, r1, H, HALO, rank, world, group)
        sums, state = fwd(img, gt, r0, r1, ctx.needs_input_grad[0])
        sums = sums.clone()
        if world > 1:
            dist.all_reduce(sums, group=group)
        n = image.numel()
        ctx.save_for_backward(img, gt, *state)
        ctx.meta = (float(lambda_dssim), n, r0, r1, rank, world, group, bwd, H)
        return ((1.0 - lambda_dssim) * sums[1] / n + lambda_dssim * (1.0 - sums[0] / n)).float()

    @staticmethod
    def backward(ctx, grad_out):
        img, gt, *state = ctx.saved_tensors
        lam, n, r0, r1, rank, world, group, bwd, H = ctx.meta
        d = bwd(img, gt, state, -lam / n, (1.0 - lam) / n, r0, r1)
        # rows [r0-5, r0) and [r1, r1+5) hold what MY slab's SSIM values contribute to the neighbours' pixels: send them home
        _exchange_halo(d, 0, r0, r1, H, HALO, rank, world, group, backward=True)
        return _SlabLayout(d, H, r0, r1).full(d[:, r0:r1]) * grad_out, None, None, None, None, None, None, None, None


def _cuda_slab_fwd(img, gt, r0, r1, need_grad):
    from diff_gaussian_rasterization import _C
    sums, dmaps = _C.ssim_l1_forward(img, gt, need_grad, r0, r1)
    return sums, (dmaps,)


def _cuda_slab_bwd(img, gt, state, w_ssim, w_l1, r0, r1):
    from diff_gaussian_rasterization import _C
    return _C.ssim_l1_backward(img, gt, state[0], w_ssim, w_l1, torch.empty(0), r0, r1)


def _check_ssim_rows(pixel_rows, H, world_size):
    """Raise unless this rank's rows suit slab_l1_ssim_loss's 5-row halo exchange: `_check_slab_rows`, and no empty slab at > 1 rank."""
    r0, r1 = _check_slab_rows(pixel_rows, None, H, 0, world_size, HALO, "slab-local SSIM")
    if world_size > 1 and r0 == r1:
        raise ValueError(f"slab-local SSIM needs at least 5 pixel rows on every slab but a non-empty last one; slab [{r0}, {r1}) is empty")
    return r0, r1


def slab_l1_ssim_loss(image: torch.Tensor, gt: torch.Tensor, lambda_dssim: float, pixel_rows: Tuple[int, int], rank: int | None = None,
                      world_size: int | None = None, group=None, kernels=None) -> torch.Tensor:
    """train.py:163's `(1 - l) * l1_loss(image, gt) + l * (1 - ssim(image, gt))` for a row-sharded render: `image` [3,H,W] holds this
    rank's slab rows `pixel_rows` (`ShardedGaussianRasterizer.pixel_rows()`), `gt` the ground truth (at least those rows +- 5).
    Returns the full-image loss (the same value on every rank); its gradient w.r.t. `image` is non-zero in this rank's rows only and
    already contains the neighbours' contributions.  Every slab that does not end at the image's last row must be at least 5 rows
    tall; a non-empty slab that ends there may be shorter (the halo its neighbour above needs ends at the image's edge too), as the
    last tile row of an image whose height is not a multiple of 16 is."""
    rank, world_size = _rank_world(rank, world_size, group)
    rows = _check_ssim_rows(pixel_rows, image.shape[-2], world_size)
    fwd, bwd = kernels if kernels is not None else (_cuda_slab_fwd, _cuda_slab_bwd)
    return _SlabSsimL1.apply(image, gt, float(lambda_dssim), rows, rank, world_size, group, fwd, bwd)


# ---- slab-local normal consistency (train.py:141-156) ------------------------------------------------------------------------
NORMAL_HALO = 2   # a stencil reads its +-1 row neighbours, and a pixel's gradient comes from the stencils +-1 row away


class _SlabNormalConsistency(torch.autograd.Function):
    """train.py:141-156's `(1 - r) * mean(error[0]) + r * mean(error[1])` of the WHOLE image, evaluated slab by slab.  A rank counts
    the error rows of its own slab.  Its kernel also evaluates the stencils one row beyond the slab, whose loss the neighbours count,
    because they read the slab's pixels: every gradient is then complete on the rank that owns the pixel, and backward exchanges
    nothing.  Forward receives 2 rows of both maps and of the normal from each neighbour (one exchange) and all-reduces one fp64
    scalar.  `kernel(normal_win, e_win, m_win, from_depth, inv_fx, inv_fy, cx, cy, w_e, w_m, H, r0, r1)` -> (loss_sum [1] float64,
    d_normal, d_e, d_m on rows [r0, r1)) takes the windows of include/rgs_b200.h's `rgs_normal_consistency_rows`."""

    @staticmethod
    def forward(ctx, normal, map_e, map_m, from_depth, cam, depth_ratio, H, rows, rank, world, group, kernel):
        r0, r1 = rows
        W = normal.shape[-1]
        C = map_e.shape[0]
        layout = _SlabLayout(normal, H, r0, r1)
        n_lo, n_hi = max(0, r0 - 1), min(H, r1 + 1)
        w_e, w_m = (1.0 - depth_ratio) / (H * W), depth_ratio / (H * W)
        if r1 > r0:
            # both maps and the normal in one row window, so that one exchange carries all their halo rows
            win, m_lo = _halo_window([map_e, map_m, normal], layout, NORMAL_HALO, rank, world, group)
            loss, dn, de, dm = kernel(win[2 * C:, n_lo - m_lo:n_hi - m_lo].contiguous(), win[:C].contiguous(), win[C:2 * C].contiguous(), from_depth,
                                      *cam, w_e, w_m, H, r0, r1)
            loss = loss.clone()
        else:
            loss = torch.zeros(1, dtype=torch.float64, device=normal.device)
            dn, de, dm = (normal.new_zeros(c, 0, W) for c in (3, C, C))
        if world > 1:
            dist.all_reduce(loss, group=group)
        ctx.save_for_backward(dn, de, dm)
        ctx.layout = layout
        return loss[0].float()

    @staticmethod
    def backward(ctx, grad_out):
        lay = ctx.layout
        return (*(d * grad_out if lay.compact else lay.full(d * grad_out) for d in ctx.saved_tensors), None, None, None, None, None, None, None, None, None)


def _cuda_normal_rows(normal_win, e_win, m_win, from_depth, inv_fx, inv_fy, cx, cy, w_e, w_m, H, r0, r1):
    from diff_gaussian_rasterization import _C
    return _C._slab.normal_consistency_rows(normal_win, e_win, m_win, from_depth, inv_fx, inv_fy, cx, cy, w_e, w_m, H, r0, r1)


def _check_slab_rows(pixel_rows, all_pixel_rows, H, rank, world_size, halo=NORMAL_HALO, what="slab-local normal consistency"):
    """Raise unless the slab rows suit the `halo`-row exchange.  With `all_pixel_rows` (every rank's rows, e.g.
    `[(min(b * 16, H), min(e * 16, H)) for b, e in rast.slabs]`) every rank checks the whole partition and all raise the same error
    before any collective.  Without it a rank sees only its own rows: a rank whose slab is too short raises, and its neighbours
    then wait in the halo exchange for rows that never come."""
    r0, r1 = int(pixel_rows[0]), int(pixel_rows[1])
    if not 0 <= r0 <= r1 <= H:
        raise ValueError(f"pixel rows [{r0}, {r1}) are not rows of a {H}-row image")
    rows = [(r0, r1)]
    if all_pixel_rows is not None:
        rows = [(int(b), int(e)) for b, e in all_pixel_rows]
        if len(rows) != world_size or rows[rank] != (r0, r1):
            raise ValueError(f"all_pixel_rows must hold one row range per rank ({world_size}) with this rank's pixel_rows at index {rank}")
        if rows[0][0] != 0 or rows[-1][1] != H or any(rows[i][1] != rows[i + 1][0] or rows[i][0] > rows[i][1] for i in range(len(rows) - 1)):
            raise ValueError(f"all_pixel_rows must tile the image's {H} rows in rank order, got {rows}")
    if world_size > 1:
        short = [(b, e) for b, e in rows if e - b < halo and e < H]
        if short:
            raise ValueError(f"{what} needs every slab that does not end at the image's last row to hold at least {halo} pixel "
                             f"rows (a shorter slab breaks the neighbour halo exchange); slabs {short} do not")
    return r0, r1


def _gather_and_check_slab_rows(pixel_rows, H, rank, world_size, group, halo, what, device):
    """Every rank's pixel rows, for a caller that was not given them: at more than one rank all-gathered (one small collective), then
    checked as a whole partition by `_check_slab_rows` on every rank, so that all ranks refuse a bad one together."""
    if world_size == 1:
        return [(int(pixel_rows[0]), int(pixel_rows[1]))]
    parts = [torch.empty(2, dtype=torch.int64, device=device) for _ in range(world_size)]
    dist.all_gather(parts, torch.tensor([int(pixel_rows[0]), int(pixel_rows[1])], dtype=torch.int64, device=device), group=group)
    rows = [tuple(p.tolist()) for p in parts]
    _check_slab_rows(pixel_rows, rows, H, rank, world_size, halo, what)
    return rows


def _slab_normal_loss(normal, map_e, map_m, from_depth, cam, depth_ratio, H, pixel_rows, all_pixel_rows, rank, world_size, group, kernels,
                      map_channels):
    r0, r1 = _check_slab_rows(pixel_rows, all_pixel_rows, H, rank, world_size)
    if kernels is None and not (normal.is_cuda and map_e.is_cuda and map_m.is_cuda):
        raise RuntimeError("slab-local normal consistency needs CUDA tensors: there is no CPU path")
    _SlabLayout.check([("normal", normal, 3), ("expected map", map_e, map_channels), ("median map", map_m, map_channels)], H, r0, r1,
                      normal.shape[-1], "the normal and both maps")
    kernel = kernels if kernels is not None else _cuda_normal_rows
    return _SlabNormalConsistency.apply(normal, map_e, map_m, from_depth, cam, float(depth_ratio), H, (r0, r1), rank, world_size, group, kernel)


def _image_height(t, pixel_rows, image_height, world_size):
    """The image's row count: `image_height`, else that of full-size maps.  Maps with the slab's row count are taken for compact
    ones when there are several ranks, and then the height cannot be read from them."""
    if image_height is not None:
        return int(image_height)
    if world_size > 1 and t.shape[-2] == pixel_rows[1] - pixel_rows[0]:
        raise ValueError("maps that hold only the slab's rows need image_height")
    return int(t.shape[-2])


def slab_depth_normal_consistency_loss(view, normal: torch.Tensor, expected_depth: torch.Tensor, median_depth: torch.Tensor,
                                       pixel_rows: Tuple[int, int], depth_ratio: float = 0.6, image_height: int | None = None,
                                       all_pixel_rows=None, rank: int | None = None, world_size: int | None = None, group=None,
                                       kernels=None) -> torch.Tensor:
    """`losses.depth_normal_consistency_loss` (train.py:141-156 with require_depth) for a row-sharded render.  The maps are
    `ShardedGaussianRasterizer`'s: compact ([3 or 1, slab rows, W]) or full-size with this rank's slab rows `pixel_rows` filled.
    `view` needs FoVx and FoVy; the image height is `image_height`, else `view.image_height`, else the maps' when they are
    full-size.  Returns the whole image's loss, the same value on every rank; its gradient lands in this rank's rows only and is
    complete there.  Every slab that does not end at the image's last row must hold at least 2 rows.  Pass `all_pixel_rows`, every
    rank's row range, so that every rank refuses a partition that breaks this rule; without it only the rank with the short slab
    raises and its neighbours block in the halo exchange."""
    if image_height is None:
        image_height = getattr(view, "image_height", None)
    rank, world_size = _rank_world(rank, world_size, group)
    H = _image_height(normal, pixel_rows, image_height, world_size)
    W = normal.shape[-1]
    fx = W / (2 * math.tan(view.FoVx / 2.))
    fy = H / (2 * math.tan(view.FoVy / 2.))
    # entries of intrins_inv (utils/graphics_utils.py:101-105), as losses.depth_normal_consistency_loss passes them
    cam = (1 / fx, 1 / fy, -W / (2 * fx), -H / (2 * fy))
    return _slab_normal_loss(normal, expected_depth, median_depth, True, cam, depth_ratio, H, pixel_rows, all_pixel_rows, rank, world_size, group,
                             kernels, 1)


def slab_point_normal_consistency_loss(normal: torch.Tensor, expected_coord: torch.Tensor, median_coord: torch.Tensor, pixel_rows: Tuple[int, int],
                                       depth_ratio: float = 0.6, image_height: int | None = None, all_pixel_rows=None, rank: int | None = None,
                                       world_size: int | None = None, group=None, kernels=None) -> torch.Tensor:
    """`losses.point_normal_consistency_loss` (train.py:141-156 with require_coord) for a row-sharded render; the maps as in
    `slab_depth_normal_consistency_loss`, and so is `all_pixel_rows`.  Compact maps need `image_height`."""
    rank, world_size = _rank_world(rank, world_size, group)
    H = _image_height(normal, pixel_rows, image_height, world_size)
    return _slab_normal_loss(normal, expected_coord, median_coord, False, (0.0, 0.0, 0.0, 0.0), depth_ratio, H, pixel_rows, all_pixel_rows, rank,
                             world_size, group, kernels, 3)


# ---- slab-local decoupled-appearance L1 (train.py:37-58) ---------------------------------------------------------------------
APPEARANCE_HALO = 4   # image rows either side of a slab whose loss derivative its d_up4 rows need (include/rgs_b200.h)


def _sum_in_rank_order(mine: torch.Tensor, world: int, group) -> torch.Tensor:
    """The fp64 per-rank values added in rank order (the same bits on every rank, whatever the collective's own order)."""
    if world == 1:
        return mine
    parts = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine, group=group)
    total = parts[0]
    for p in parts[1:]:
        total = total + p
    return total


class _SlabAppearanceL1(torch.autograd.Function):
    """train.py:37-58's `L1_loss_appearance` of the WHOLE image, evaluated slab by slab (include/rgs_b200.h's
    `rgs_appearance_*_rows`).  Forward: 4 image rows to and from each neighbour, the owned low-resolution rows all-gathered, the
    head replicated on every rank (the fused head kernels when `kernels` has them, else the module's layers), the tail on the slab, and the per-rank fp64 loss sums all-gathered and added in rank order.
    Backward: the owned rows of d(up4) all-gathered, so that the head's backward, d(down) and the embedding gradient are the
    single-GPU call's; the per-rank fp64 rows of conv2 / conv3's weight gradients added in rank order.  The image is never gathered.
    `kernels` supplies the four row stages and the head (the CUDA ones), or the row stages alone (fp64 stand-ins in the CPU test)."""

    @staticmethod
    def forward(ctx, image, gt, emb, net, slab, kernels, *params):
        H0, rows, rank, world, group = slab
        from diff_gaussian_rasterization import _C
        from .appearance import _head, _head_input
        r0, r1 = rows[rank]
        W0 = gt.shape[-1]
        layout = _SlabLayout(image, H0, r0, r1)
        H, W = H0 // 32 * 32, W0 // 32 * 32
        wins = [_C._slab.appearance_row_windows(H0, W0, b, e) for b, e in rows]
        win, lo = _halo_window([image], layout, APPEARANCE_HALO, rank, world, group)
        gt_win = gt.detach()[:, lo:lo + win.shape[1]].contiguous()
        down = _gather_rows(kernels.downsample_rows(win, lo, H0, r0, r1), [(w[2], w[3]) for w in wins], H // 32, group)
        if hasattr(kernels, "head_forward"):   # the fused head (csrc/rgs_appearance_head.cu)
            e, head = emb.detach(), [p.detach() for p in params[:-4]]
            head_act, up4 = kernels.head_forward(down, e, head)
            ctx.head = (up4, down, e, head, head_act)
        else:                                  # the module's layers, for row stages that bring no head
            with torch.enable_grad():
                d_leaf = down.detach().requires_grad_(True)
                e_leaf = emb.detach().requires_grad_(True)
                up4 = _head(net, _head_input(d_leaf, e_leaf))
            ctx.head = (up4, d_leaf, e_leaf, params[:-4], None)
        w2, b2, w3, b3 = (p.detach() for p in (net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias))
        loss_sum, act = kernels.l1_forward_rows(win, gt_win, lo, H0, r0, r1, up4.detach(), w2, b2, w3, b3)
        total = _sum_in_rank_order(loss_sum.clone(), world, group)
        ctx.meta = (H0, lo, r0, r1, layout, [(w[4], w[5]) for w in wins], world, group, kernels)
        ctx.save_for_backward(win, gt_win, act, w2, b2, w3, b3)
        return (total[0] / (3.0 * H * W)).to(gt.dtype)   # float32 on the GPU, as L1_loss_appearance returns it

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        win, gt_win, act, w2, b2, w3, b3 = ctx.saved_tensors
        up4, down, emb, head_params, head_act = ctx.head
        H0, lo, r0, r1, layout, u_rows, world, group, kernels = ctx.meta
        d_img, d_up4, grad_row = kernels.l1_backward_rows(win, gt_win, lo, H0, r0, r1, up4.detach(), act, w2, b2, w3, b3,
                                                          grad_out.float().reshape(1))
        d_up4 = _gather_rows(d_up4, u_rows, up4.shape[-2], group).reshape(up4.shape)
        if head_act is not None:
            grads = kernels.head_backward(down, emb, head_params, head_act, up4, d_up4)
        else:
            grads = torch.autograd.grad(up4, [down, emb, *head_params], d_up4)
        g = _sum_in_rank_order(grad_row.clone(), world, group).to(w2.dtype)
        d_w2, d_b2, d_w3, d_b3 = g[:2304].view(w2.shape), g[2304:2320].view(b2.shape), g[2320:2752].view(w3.shape), g[2752:].view(b3.shape)
        kernels.downsample_backward_rows(grads[0], d_img, H0, r0, r1)
        ctx.head = None
        return (d_img if layout.compact else layout.full(d_img), None, grads[1], None, None, None, *grads[2:], d_w2, d_b2, d_w3, d_b3)


class _CudaAppearanceRows:
    """The CUDA row stages (`_C._slab.appearance_*_rows`) and the fused head (`_C._appearance_head`)."""

    @staticmethod
    def downsample_rows(win, lo, H0, r0, r1):
        from diff_gaussian_rasterization import _C
        return _C._slab.appearance_downsample_rows(win, lo, H0, r0, r1)

    @staticmethod
    def l1_forward_rows(win, gt_win, lo, H0, r0, r1, up4, w2, b2, w3, b3):
        from diff_gaussian_rasterization import _C
        return _C._slab.appearance_l1_forward_rows(win, gt_win, lo, H0, r0, r1, up4, w2, b2, w3, b3)

    @staticmethod
    def l1_backward_rows(win, gt_win, lo, H0, r0, r1, up4, act, w2, b2, w3, b3, upstream):
        from diff_gaussian_rasterization import _C
        return _C._slab.appearance_l1_backward_rows(win, gt_win, lo, H0, r0, r1, up4, act, w2, b2, w3, b3, upstream)

    @staticmethod
    def downsample_backward_rows(d_down, d_img, H0, r0, r1):
        from diff_gaussian_rasterization import _C
        _C._slab.appearance_downsample_backward_rows(d_down, d_img, H0, r0, r1)

    @staticmethod
    def head_forward(down, emb, head_params):
        from diff_gaussian_rasterization import _C
        return _C._appearance_head.forward(down, emb, head_params)

    @staticmethod
    def head_backward(down, emb, head_params, head_act, up4, d_up4):
        from diff_gaussian_rasterization import _C
        return _C._appearance_head.backward(down, emb, head_params, head_act, up4, d_up4)


def slab_L1_loss_appearance(image: torch.Tensor, gt_image: torch.Tensor, gaussians, view_idx, pixel_rows: Tuple[int, int], all_pixel_rows=None,
                            image_height: int | None = None, rank: int | None = None, world_size: int | None = None, group=None, kernels=None,
                            return_transformed_image: bool = False) -> torch.Tensor:
    """`appearance.L1_loss_appearance` (train.py:37-58, `--use_decoupled_appearance`) for a row-sharded render.  `image` is
    `ShardedGaussianRasterizer`'s colour: compact ([3, slab rows, W]) or full-size with this rank's slab rows `pixel_rows` filled;
    `gt_image` is the whole ground truth [3, H, W], as train.py holds it (it also gives the image height; `image_height`, when
    given, must agree).  Returns the whole image's loss, the same value on every rank.  Its gradient w.r.t. `image` lies in this
    rank's rows and is complete there; the network's parameter gradients and the embedding row's are the same bits on every rank.
    Only conv2 / conv3's weight gradients and the loss are summed in another order than the single-GPU call's (fp64 per rank, then
    over the ranks in rank order); at one rank every result is that call's, bit for bit.  With the built-in CUDA stages
    (`kernels=None`) the head runs in the project's kernels on every rank, so its gradients are the same bits on every rank and
    in every call, whatever torch's cuDNN and TF32 settings.  A `kernels` object without `head_forward` / `head_backward` runs the
    head as the module's own layers instead (the CPU test's fp64 stand-ins), and that guarantee does not hold for it.

    Every slab that does not end at the image's last row must hold at least 4 rows (the halo).  With `all_pixel_rows`, every rank's
    row range, every rank refuses a bad partition before any collective; without it the ranks first all-gather their row ranges
    (one small collective) and then all refuse a bad partition together.  The checks of a rank's own arguments (the network, the
    image's shape, the embedding row, CUDA tensors) run before that gather: a rank whose own arguments are wrong raises alone, and without
    `all_pixel_rows` its peers then wait in the gather.  `return_transformed_image` has no slab form."""
    if return_transformed_image:
        raise ValueError("slab_L1_loss_appearance has no transformed-image form: gather the image and call appearance.L1_loss_appearance")
    from .appearance import _check_network, _embedding, _head_params
    net = gaussians.appearance_network
    _check_network(net)
    emb = _embedding(gaussians, view_idx)
    if gt_image.requires_grad:
        raise ValueError("slab_L1_loss_appearance differentiates w.r.t. the rendered image, not the ground truth")
    if gt_image.dim() != 3 or gt_image.shape[0] != 3 or gt_image.shape[1] < 32 or gt_image.shape[2] < 32:
        raise ValueError(f"slab_L1_loss_appearance needs a [3, H, W] ground truth with H, W >= 32, got {tuple(gt_image.shape)}")
    H0, W0 = gt_image.shape[1:]
    if image_height is not None and int(image_height) != H0:
        raise ValueError(f"image_height {image_height} is not the ground truth's {H0} rows")
    rank, world_size = _rank_world(rank, world_size, group)
    what = "the slab-local appearance loss"
    # without every rank's rows, the slab lengths are checked after the rows are gathered, so that all ranks raise together
    r0, r1 = _check_slab_rows(pixel_rows, all_pixel_rows, H0, rank, world_size if all_pixel_rows is not None else 1, APPEARANCE_HALO, what)
    _SlabLayout.check([("image", image, 3)], H0, r0, r1, W0)
    if kernels is None and not (image.is_cuda and gt_image.is_cuda):
        raise RuntimeError("slab_L1_loss_appearance needs CUDA tensors: there is no CPU path")
    rows = ([(int(b), int(e)) for b, e in all_pixel_rows] if all_pixel_rows is not None
            else _gather_and_check_slab_rows(pixel_rows, H0, rank, world_size, group, APPEARANCE_HALO, what, image.device))
    params = _head_params(net) + [net.conv2.weight, net.conv2.bias, net.conv3.weight, net.conv3.bias]
    if len(params) != len(list(net.parameters())):
        raise ValueError("appearance network: parameters outside conv1, up1..up4, conv2 and conv3 are not supported")
    return _SlabAppearanceL1.apply(image, gt_image, emb, net, (H0, rows, rank, world_size, group), kernels or _CudaAppearanceRows, *params)
