"""Balanced row sharding (`ShardedGaussianRasterizer(balance=True)`, include/rgs_b200.h's `rgs_forward_balanced`) on one GPU.

  * the per-row instance counts and longest lists are those of a whole-image call's tile ranges;
  * every rank's balanced call leaves exactly the state a fixed-slab call over the same rows leaves: maps, radii, num_rendered,
    sorted lists and per-tile state bit for bit; backward-preprocess of the same accumulator bit for bit; stage 1 (a float-atomic
    sum) within the run-to-run bars;
  * the slabs stitch to the whole-image render bit for bit, and the skewed scene's largest slab weight meets the rule's bounds;
  * 2, 3 and 4 ranks as processes on one GPU through one sharded training step with the whole loss;
  * the entry point on poisoned memory and on a late-ready side stream.
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_gpu_stale_memory import Case, _step, check_case, poisoned_allocator  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu

DEV = "cuda"
IMAGES = ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth")


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def uniform_scene():
    from rade_gs_b200 import scenes
    return scenes.make_scene(40000, 640, 400, 500.0, -3.8, seed=21, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.2, 0.1, 0.3))


def skewed_scene(W=640, H=400):
    """Dense splats in the image's lower third, one in twelve of the rest above it."""
    from rade_gs_b200 import scenes
    sc = scenes.make_scene(120000, W, H, 500.0, -3.8, seed=23, view=scenes.look_at_view((0.1, -0.1, -0.2), (0.0, 0.0, 6.0)), bg=(0.1, 0.2, 0.3))
    hom = torch.cat([sc.means3D, torch.ones(sc.means3D.shape[0], 1)], 1) @ sc.projmatrix
    py = ((hom[:, 1] / (hom[:, 3] + 1e-7) + 1.0) * sc.height - 1.0) * 0.5
    keep = (py >= 2 * sc.height / 3) | (torch.arange(py.shape[0]) % 12 == 0)
    kw = {k: (v[keep] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == keep.shape[0] else v) for k, v in vars(sc).items()}
    return scenes.Scene(**kw)


def skewed_tail_scene():
    """The skewed scene at 979x546 (a Tanks and Temples recipe's size): the last tile row holds 2 pixel rows."""
    return skewed_scene(979, 546)


SCENES = {"uniform": uniform_scene, "skewed": skewed_scene, "skewed_979x546": skewed_tail_scene}


def _call(coord, depth, ks):
    from rade_gs_b200 import rawapi
    return dict(require_coord=coord, require_depth=depth, kernel_size=ks, sh_degree=3, scale_modifier=1.0, debug=False, tile_rows=None, compact=False,
                shs=None, cols=rawapi._absent(), scales=None, rots=None, cov=rawapi._absent())


def balanced(C, sc, world, rank, coord=False, depth=True, ks=0.1, compact=True):
    """The balanced forward as a `rawapi.forward`-style dict (so that rawapi's backward stages take it), + cuts and row stats."""
    from rade_gs_b200 import rawapi
    c = _call(coord, depth, ks)
    c.update(shs=sc.shs, scales=sc.scales, rots=sc.rotations, compact=compact)
    out = C._slab.rasterize_balanced(*rawapi._forward_args(sc, c), world, rank, compact)
    cuts, stats = list(out[12]), out[13]
    c["tile_rows"] = (cuts[rank], cuts[rank + 1])
    res = dict(zip(rawapi.FWD_KEYS, out[:12]))
    res["_call"] = c
    return res, cuts, stats


def _tile_state(f, sc):
    """The per-tile and per-splat state a balanced call rewrites, as laid out by rgs_api.cu's carve_img / carve_geom."""
    from rade_gs_b200 import rawapi
    P = sc.means3D.shape[0]
    tiles = ((sc.width + 15) // 16) * ((sc.height + 15) // 16)
    g = rawapi._Cursor(f["geom"])
    g.take(P * (24 if f["_call"]["require_coord"] else 16), torch.float32, 4)
    g.take(P, torch.float32, 4)
    touched = g.take(P, torch.int32, 4)
    i = rawapi._Cursor(f["img"])
    ranges = i.take(tiles * 2, torch.int32, 4)
    count = i.take(tiles, torch.int32, 4)
    totals = i.take(2, torch.int32, 4)
    chunk = i.take(tiles, torch.int32, 4)
    R = int(f["num_rendered"])
    b = rawapi._Cursor(f["binning"])
    return dict(tiles_touched=touched, ranges=ranges, tile_count=count, totals=totals, chunk_base=chunk, point_list=b.take(R, torch.int32, 4),
                keys=b.take(R, torch.int64, 8))


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _row_weights(stats, grid_x):
    return (stats[0].to(torch.int64) + _C()._slab.BALANCE_TILE_COST * grid_x).tolist()


@pytest.fixture(scope="module")
def scenes_on_gpu():
    return {k: v().to(DEV) for k, v in SCENES.items()}


@pytest.mark.parametrize("name", list(SCENES))
def test_row_stats_are_the_whole_image_tile_ranges(name, scenes_on_gpu):
    from rade_gs_b200 import rawapi
    C, sc = _C(), scenes_on_gpu[name]
    _, _, stats = balanced(C, sc, 1, 0)
    whole = rawapi.forward(C, sc, False, True, kernel_size=0.1)
    gx, gy = (sc.width + 15) // 16, (sc.height + 15) // 16
    r = rawapi.ours_views(whole, sc)["ranges"].long()
    n = (r[:, 1] - r[:, 0]).view(gy, gx).cpu()
    assert torch.equal(stats[0], n.sum(1)) and torch.equal(stats[1], n.max(1).values)
    assert int(stats[0].sum()) == whole["num_rendered"]


@pytest.mark.parametrize("compact", [True, False], ids=["compact", "full"])
@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_balanced_slab_is_the_fixed_slab_call(world, name, compact, scenes_on_gpu):
    import tolerances as tol
    from rade_gs_b200 import multigpu, rawapi, scenes
    C, sc = _C(), scenes_on_gpu[name]
    H, gx = sc.height, (sc.width + 15) // 16
    g = scenes.make_upstream_grads(H, sc.width, seed=9, device=DEV)
    whole = rawapi.forward(C, sc, False, True, kernel_size=0.1)
    stitched = {k: [] for k in IMAGES}
    partitions = set()
    for rank in range(world):
        fb, cuts, stats = balanced(C, sc, world, rank, compact=compact)
        partitions.add(tuple(cuts))
        assert cuts == C._slab.balance_partition(stats[0].tolist(), gx, world)
        rows = (cuts[rank], cuts[rank + 1])
        ff = rawapi.forward(C, sc, False, True, kernel_size=0.1, tile_rows=rows, compact=compact)
        assert fb["num_rendered"] == ff["num_rendered"], (rank, fb["num_rendered"], ff["num_rendered"])
        for k in IMAGES + ("radii",):
            assert torch.equal(_bits(fb[k]), _bits(ff[k])), (rank, k)
        sb, sf = _tile_state(fb, sc), _tile_state(ff, sc)
        for k in sb:
            assert torch.equal(sb[k], sf[k]), (rank, k)
        r0, r1 = min(rows[0] * 16, H), min(rows[1] * 16, H)
        gr = {k: v[:, r0:r1].contiguous() for k, v in g.items()} if compact else g
        acc_b, acc_f = rawapi.backward_render(C, sc, fb, gr), rawapi.backward_render(C, sc, ff, gr)
        zb, zf = (acc_b == 0).all(1), (acc_f == 0).all(1)
        assert torch.equal(zb, zf), rank
        tol.grad_close_gpu(acc_b.double().cpu().numpy(), acc_f.double().cpu().numpy(), f"rank {rank} stage 1")   # a float-atomic sum
        gb, gf = rawapi.backward_preprocess(C, sc, fb, acc_f), rawapi.backward_preprocess(C, sc, ff, acc_f)
        for k in gb:
            assert torch.equal(_bits(gb[k]), _bits(gf[k])), (rank, k)
        for k in IMAGES:
            stitched[k].append(fb[k] if compact else fb[k][:, r0:r1])
    assert len(partitions) == 1, "every rank derives the same partition"
    for k in IMAGES:
        assert torch.equal(_bits(torch.cat(stitched[k], 1)), _bits(whole[k])), k
    if name.startswith("skewed"):
        cuts = list(partitions.pop())
        w = _row_weights(stats, gx)
        largest = max(sum(w[cuts[r]:cuts[r + 1]]) for r in range(world))
        equal = multigpu.partition_tile_rows(len(w), world)
        assert largest <= -(-sum(w) // world) + max(w)
        assert largest <= max(sum(w[b:e]) for b, e in equal)


def test_more_ranks_than_tile_rows_raises(scenes_on_gpu):
    sc = scenes_on_gpu["uniform"]
    with pytest.raises(RuntimeError, match="fewer tile rows than ranks"):
        balanced(_C(), sc, (sc.height + 15) // 16 + 1, 0)


# ---- poisoned memory and a late-ready side stream -------------------------------------------------------------------------

def _balanced_case():
    from rade_gs_b200 import rawapi, scenes
    C = _C()
    sc = skewed_scene().to(DEV)
    g = scenes.make_upstream_grads(sc.height, sc.width, seed=19, device=DEV)
    world = 3
    accs = []
    for rank in range(world):
        f, cuts, _ = balanced(C, sc, world, rank)
        r0, r1 = min(cuts[rank] * 16, sc.height), min(cuts[rank + 1] * 16, sc.height)
        accs.append(rawapi.backward_render(C, sc, f, {k: v[:, r0:r1].contiguous() for k, v in g.items()}))

    def run(x):
        out = {}
        for rank in range(world):
            f, cuts, stats = balanced(C, x["sc"], world, rank)
            _step()
            out.update({f"r{rank}.{k}": f[k] for k in IMAGES + ("radii", "num_rendered")})
            out.update({f"r{rank}.{k}": v for k, v in _tile_state(f, x["sc"]).items() if k != "tile_count"})
            out[f"r{rank}.cuts"] = tuple(cuts)
            out[f"r{rank}.stats"] = stats
            r0, r1 = min(cuts[rank] * 16, x["sc"].height), min(cuts[rank + 1] * 16, x["sc"].height)
            out[f"r{rank}.acc"] = rawapi.backward_render(C, x["sc"], f, {k: v[:, r0:r1].contiguous() for k, v in x["g"].items()})
            out.update({f"r{rank}.stage2.{k}": v for k, v in rawapi.backward_preprocess(C, x["sc"], f, x["accs"][rank]).items()})
        return out
    return Case({"sc": sc, "g": g, "accs": accs}, run, {f"r{r}.acc": ("acc",) for r in range(world)})


def test_balanced_forward_on_poisoned_memory_and_a_side_stream(poisoned_allocator):
    check_case(_balanced_case(), poisoned_allocator)


# ---- 2, 3 and 4 ranks as processes on one GPU: one sharded training step with the whole loss ------------------------------

JOIN_TIMEOUT_S = 900


def _rank_main(rank, world, store, outdir, scene):
    for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import traceback

    import torch.distributed as dist
    dist.init_process_group("gloo", store=dist.FileStore(store, world), rank=rank, world_size=world)
    try:
        torch.save(_step_job(rank, world, scene), os.path.join(outdir, f"rank{rank}.pt"))
    except BaseException:   # noqa: BLE001  (reported to the parent, which fails the test)
        with open(os.path.join(outdir, f"error{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
    finally:
        dist.destroy_process_group()


def _step_job(rank, world, scene):
    """One training step of the DTU / TNT recipe (L1 + SSIM, depth-normal consistency, decoupled appearance) with balanced slabs,
    and the single-GPU step in the same process.  The ranks share cuda:0 and talk over gloo: the halo rows of the slab losses
    travel through host memory (gloo's point-to-point calls take CPU tensors), everything else as in a multi-GPU run."""
    from types import SimpleNamespace

    import torch.distributed as dist

    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import losses, multigpu
    from rade_gs_b200.appearance import L1_loss_appearance
    from test_gpu_appearance import _Net
    from test_gpu_slab_appearance import _recipe_inputs

    exchange_on_device = multigpu._exchange_rows

    def exchange_through_host(t, *args, **kw):
        h = t.cpu()
        exchange_on_device(h, *args, **kw)
        t.copy_(h)

    multigpu._exchange_rows = exchange_through_host
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sc = SCENES[scene]().to(dev)
    sc = multigpu.broadcast_scene_(sc)
    H, W = sc.height, sc.width
    st = dgr.GaussianRasterizationSettings(H, W, sc.tanfovx, sc.tanfovy, 0.1, sc.bg, 1.0, sc.viewmatrix, sc.projmatrix, 3, sc.campos, False, True,
                                           False, False)
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
    res = {}

    def step(sharded):
        lv = {k: getattr(sc, k).clone().requires_grad_(True) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        m2 = torch.zeros_like(lv["means3D"], requires_grad=True)
        net = _Net().to(dev)
        net.load_state_dict(net0.state_dict())
        table = torch.nn.Parameter(table0.clone())
        g = SimpleNamespace(appearance_network=net, get_apperance_embedding=lambda i: table[i])
        rast = multigpu.ShardedGaussianRasterizer(st, compact=True, balance=True) if sharded else dgr.GaussianRasterizer(st)
        color, _, _, _, dep, mdep, _, normal = rast(lv["means3D"], m2, lv["opacities"], shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"])
        if sharded:   # INTEGRATION.md section 3, the balanced step
            rows, everyone = rast.pixel_rows(), rast.all_pixel_rows()
            res["slabs"] = rast.slabs
            full = color.new_zeros(3, H, W)
            full[:, rows[0]:rows[1]] = color
            l1 = multigpu.slab_L1_loss_appearance(color, gt, g, uid, rows, all_pixel_rows=everyone)
            ssim_term = multigpu.slab_l1_ssim_loss(full, gt, 1.0, rows)
            nc = multigpu.slab_depth_normal_consistency_loss(view, normal, dep, mdep, rows, all_pixel_rows=everyone)
        else:
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
    mine = torch.tensor([c for s in res["slabs"] for c in s], dtype=torch.int64)
    parts = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine)
    res["partitions"] = [p.tolist() for p in parts]
    res["tile_rows"] = multigpu.tile_rows(H)
    res["loss"] = (ls, l1)
    res["grads"] = {}
    for k in gs:
        ref = gs[k].contiguous().clone()
        dist.broadcast(ref, src=0)
        res["grads"][k] = (gs[k].double().cpu().numpy(), g1[k].double().cpu().numpy(), int((_bits(gs[k]) != _bits(ref)).sum()))
    return res


@pytest.mark.parametrize("scene", ["skewed", "skewed_979x546"])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_balanced_training_step_at_several_ranks_on_one_gpu(world, scene, tmp_path):
    """Every rank derives the same partition, every gradient has the same bits on every rank, and each is within the sharded-step
    bars (tests/test_gpu_slab_appearance.py) of the single-GPU step."""
    import tolerances as tol
    import torch.multiprocessing as mp
    from rade_gs_b200.multigpu import partition_tile_rows
    ctx = mp.get_context("spawn")
    store = str(tmp_path / "store")
    procs = [ctx.Process(target=_rank_main, args=(r, world, store, str(tmp_path), scene)) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + JOIN_TIMEOUT_S
    try:
        for p in procs:
            p.join(max(1.0, deadline - time.monotonic()))
    finally:
        hung = [r for r, p in enumerate(procs) if p.is_alive()]
        for p in procs:
            if p.is_alive():
                p.terminate()
        for p in procs:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    errors = {r: (tmp_path / f"error{r}.txt").read_text() for r in range(world) if (tmp_path / f"error{r}.txt").exists()}
    assert not errors, "\n".join(f"rank {r}:\n{e}" for r, e in errors.items())
    assert not hung, f"ranks {hung} did not finish within {JOIN_TIMEOUT_S} s"
    per_rank = [torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in range(world)]
    for rank, res in enumerate(per_rank):
        assert all(p == res["partitions"][0] for p in res["partitions"]), res["partitions"]
        ls, l1 = res["loss"]
        assert abs(ls - l1) <= 1e-5 * max(1.0, abs(l1)), (rank, ls, l1)
        assert {"embedding", "net.conv1.weight", "means3D", "shs"} <= set(res["grads"])
        for k, (got, ref, differ) in res["grads"].items():
            assert differ == 0, (rank, k, differ)
            tol.grad_close_gpu(got, ref, f"rank {rank} {k}")
    if scene == "skewed":
        equal = [c for b, e in partition_tile_rows(per_rank[0]["tile_rows"], world) for c in (b, e)]
        assert per_rank[0]["partitions"][0] != equal, "the skewed scene moves the cuts off the equal partition"
