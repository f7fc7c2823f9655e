"""The peer gradient exchange (csrc/rgs_exchange.cu) at 2, 3 and 4 ranks on ONE GPU.

CUDA IPC works between processes on the same device, so the ranks are processes on cuda:0, each with its own context; the
contexts take turns on the GPU, so one rank's spinning barrier gives way to the others' pushes and flags.  The ranks talk
over gloo (a FileStore in the test's directory) on CPU tensors only: the IPC handles, ok flags and results.

  A. the bare step (`exchange_accumulator` / `exchange_rows` / `exchange_result`) on rows aimed at its edges, every summed
     element checked bit for bit against the admissible set of tests/exchange_model.py;
  B. stage 1 through the exchange on a real scene, against the whole-image backward of the same process;
  C. `GradExchange(mode="peer")` under gloo: its self-check and one stage 1 through it.
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

import exchange_model as em
from conftest import ROOT

pytestmark = pytest.mark.gpu

JOIN_TIMEOUT_S = 900

# ---- process harness ----------------------------------------------------------------------------------------------------


def _rank_main(rank, world, store, outdir, job, params):
    """One rank: gloo over a FileStore, CUDA on device 0; `job` writes `rank{r}.pt` (or `skip{r}.txt` / `error{r}.txt`)."""
    for p in (os.path.join(ROOT, "rade-gs_b200"), os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    import traceback

    import torch.distributed as dist
    dist.init_process_group("gloo", store=dist.FileStore(store, world), rank=rank, world_size=world)
    try:
        out = globals()[job](rank, world, params)
        if isinstance(out, str):
            with open(os.path.join(outdir, f"skip{rank}.txt"), "w") as f:
                f.write(out)
        else:
            torch.save(out, os.path.join(outdir, f"rank{rank}.pt"))
    except BaseException:   # noqa: BLE001  (reported to the parent, which fails the test)
        with open(os.path.join(outdir, f"error{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
    finally:
        dist.destroy_process_group()


def _spawn(world, job, params, tmp_path):
    """Runs `job` on `world` ranks; every child is joined or terminated before this returns.  -> per-rank results."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    store = str(tmp_path / "store")
    procs = [ctx.Process(target=_rank_main, args=(r, world, store, str(tmp_path), job, params)) for r in range(world)]
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
    skips = [(tmp_path / f"skip{r}.txt").read_text() for r in range(world) if (tmp_path / f"skip{r}.txt").exists()]
    if skips:
        pytest.skip(f"no peer exchange between processes on this GPU: {skips[0]}")
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in range(world)]


def _connect(C, rank, world, capacity, row_floats):
    """Creates and connects this rank's exchange object.  Any rank's failure (e.g. a GPU in exclusive-process mode, where a
    second process gets no context) stops all ranks before an exchange kernel runs: -> (handle, None) or (None, reason)."""
    import torch.distributed as dist

    def agree(why):
        flag = torch.tensor([0 if why else 1], dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        return why or (None if int(flag) == 1 else "another rank failed")

    ex, handle, why = None, None, None
    try:
        torch.cuda.set_device(0)
        torch.zeros(1, device="cuda")
        ex, handle = C.exchange_create(rank, world, capacity, row_floats, 0)
    except Exception as e:   # noqa: BLE001
        why = f"rank {rank}: {type(e).__name__}: {e}"
    why = agree(why)
    if why is None:
        gathered = [torch.empty_like(handle) for _ in range(world)]
        dist.all_gather(gathered, handle)
        try:
            C.exchange_connect(ex, torch.stack(gathered), 0)
        except Exception as e:   # noqa: BLE001
            why = f"rank {rank}: {type(e).__name__}: {e}"
        why = agree(why)
    if why is not None:
        if ex is not None:
            C.exchange_destroy(ex)
        return None, why
    dist.barrier()   # nobody pushes before every rank has mapped every window
    return ex, None


def _close(C, ex):
    import torch.distributed as dist
    dist.barrier()   # peers may still be reading / writing this rank's window
    C.exchange_destroy(ex)


def _status(C, ex, what):
    rc = C.exchange_status(ex)
    assert rc == 0, f"{what}: an exchange barrier gave up waiting for rank {rc - 1}"


# ---- A. the bare step ---------------------------------------------------------------------------------------------------

CAPACITY = 3000
TINY = np.float32(2.0 ** -126)
NAN = em.f32(em.CANONICAL_NAN)
FAMILIES = ("random", "touched_zero", "cancel", "on_off", "neg_zero", "nan_inf", "subnormal")


def _p_sequence(world):
    """P of each step on one exchange object: the capacity (twice: the same P keeps the rows), P - 1, the capacity again,
    rows_per_rank 255 / 256 / 257 (the kernels' 256-thread grids), P not divisible by the world, P < world, P = 0, and the
    capacity after P = 0."""
    c = CAPACITY
    return [c, c, c - 1, c - 1, c, 255 * world, 256 * world, 256 * world, 256 * world + 1, 700 * world + world - 1,
            max(world - 1, 1), 0, c]


def _step_rows(world, row_floats, step, P):
    """What every rank's accumulator holds before `step`, and which rows its slab touched: rows [W, P, F], touched [W, P].
    Each row belongs to one family, fixed per row index (so rows keep their family while P stays); ranks write only the rows
    they touch."""
    W, F, Q = world, row_floats, row_floats // 4
    fam = np.random.default_rng([world, F]).integers(0, len(FAMILIES), CAPACITY)[:P]
    rng = np.random.default_rng([world, F, step])
    rows = np.zeros((W, P, F), np.float32)
    touched = np.zeros((W, P), bool)
    even = step % 2 == 0

    def rand(*shape):
        return (rng.standard_normal(shape) * 10.0 ** rng.uniform(-3, 3, shape)).astype(np.float32)

    m = fam == 0   # random rows, a share of zero quarters and zero rows, touched by a random subset of the ranks
    n = int(m.sum())
    v = rand(W, n, F)
    v *= np.repeat(rng.random((W, n, Q)) > 0.3, 4, axis=-1)
    v *= (rng.random((W, n, 1)) > 0.1)
    rows[:, m], touched[:, m] = v, rng.random((W, n)) < 0.6
    m = fam == 1   # touched, zero
    touched[:, m] = True
    m = fam == 2   # contributions that cancel: exactly (small multiples of powers of two), or through rounding (1e8 + x - 1e8)
    n = int(m.sum())
    ints = (rng.integers(-64, 64, (W, n, F)) * 2.0 ** rng.integers(-10, 10, (1, n, F))).astype(np.float32)
    ints[-1] = -ints[:-1].sum(0)
    big = np.where(rng.random((W, n, F)) < 0.5, 1e8, -1e8).astype(np.float32)
    big[1::2] = (rng.standard_normal((len(range(1, W, 2)), n, F)) * 4).astype(np.float32)
    if W % 2 == 0:
        big[0::2] = np.where(np.arange(W // 2)[:, None, None] % 2 == 0, 1e8, -1e8).astype(np.float32)
    rows[:, m] = np.where(rng.random((1, n, F)) < 0.5, ints, big)
    touched[:, m] = True
    m = fam == 3   # non-zero in one step, untouched in the next
    n = int(m.sum())
    rows[:, m], touched[:, m] = (rand(W, n, F), True) if even else (0, False)
    m = fam == 4   # -0.0 quarters: some all -0.0 (not pushed), some -0.0 beside a value
    n = int(m.sum())
    v = np.full((W, n, F), -0.0, np.float32)
    keep = rng.random((W, n, F)) < 0.15
    v[keep] = rand(int(keep.sum()))
    rows[:, m], touched[:, m] = v, True
    m = fam == 5   # NaN, +Inf, -Inf (Inf on one rank and -Inf on another), beside finite values
    n = int(m.sum())
    v = rand(W, n, F)
    pick = rng.integers(0, 8, (W, n, F))
    v[pick == 0] = NAN
    v[pick == 1] = np.inf
    v[pick == 2] = -np.inf
    v[pick == 3] = 0.0
    rows[:, m], touched[:, m] = v, rng.random((W, n)) < 0.8
    m = fam == 6   # subnormals; pairs of normals whose sum is a subnormal (flushed: -0.0 results in an otherwise zero quarter);
    n = int(m.sum())  # on odd steps half of them untouched and half pushed as (-0.0, value) quarters
    if even:
        v = np.zeros((W, n, F), np.float32)
        sub = (rng.integers(1, 1 << 23, (W, n, F)).astype(np.uint32)) | (rng.integers(0, 2, (W, n, F)).astype(np.uint32) << 31)
        v[:] = np.where(rng.random((W, n, F)) < 0.3, sub.view(np.float32), 0)
        pair = rng.random((n, F)) < 0.3
        v[0] = np.where(pair, -1.5 * TINY, v[0])
        v[1] = np.where(pair, TINY, v[1])
        if W > 2:
            v[2:] = np.where(pair, 0, v[2:])
        rows[:, m], touched[:, m] = v, True
    else:
        idx = np.nonzero(m)[0]
        on = idx[idx % 2 == 1]
        v = np.full((W, len(on), F), -0.0, np.float32)
        v[:, :, 1::4] = rand(W, len(on), Q)
        rows[:, on], touched[:, on] = v, True
    rows[~touched] = 0
    return rows, touched.astype(np.int32)


def _flushed_zero_p_sequence(world):
    return [600, 600, 600, 600, 599]


def _flushed_zero_rows(world, row_floats, step, P):
    """The case that showed the spread pass taking a -0.0 sum for an empty row: -1.5 * 2^-126 + 2^-126 is a subnormal, which
    red.add.f32 flushes to -0.0.  That -0.0 was neither cleared from the owner's `sum` nor marked for the rewrite, so the
    next step read -0.0 where nobody pushed, and -0.0 + -0.0 where a quarter pushed -0.0 beside a value, both for +0.0.
    Steps: the flushed sums; nothing pushed; (-0.0, v, -0.0, -0.0) quarters pushed by rank 0; the flushed sums; P - 1."""
    W, F = world, row_floats
    rows = np.zeros((W, P, F), np.float32)
    touched = np.ones((W, P), np.int32)
    if step in (0, 3):
        rows[0, :, 0::4], rows[1, :, 0::4] = -1.5 * TINY, TINY
    elif step == 1:
        touched[:] = 0
    else:
        rows[0] = -0.0
        rows[0, :, 1::4] = np.arange(1, P * F // 4 + 1, dtype=np.float32).reshape(P, F // 4)
    return rows, touched


CASES = {"families": (_p_sequence, _step_rows), "flushed_zero": (_flushed_zero_p_sequence, _flushed_zero_rows)}


def _bare_job(rank, world, params):
    from diff_gaussian_rasterization import _C as C
    F = params["row_floats"]
    p_sequence, step_rows = CASES[params["case"]]
    ex, why = _connect(C, rank, world, CAPACITY, F)
    if why is not None:
        return why
    out = []
    try:
        for step, P in enumerate(p_sequence(world)):
            rows, touched = step_rows(world, F, step, P)
            acc = C.exchange_accumulator(ex, P, F, 0)
            acc.copy_(torch.from_numpy(rows[rank]))
            C.exchange_rows(ex, torch.from_numpy(touched[rank]).cuda(), torch.ones(P, dtype=torch.int32, device="cuda"))
            _status(C, ex, f"step {step} (P {P})")
            out.append({"result": C.exchange_result(ex, P, F, 0).cpu().numpy().copy(), "acc": acc.cpu().numpy().copy()})
    finally:
        _close(C, ex)
    return out


def _check_bare(world, row_floats, case, tmp_path):
    """Runs a case's steps on `world` ranks and checks every step against the model.  -> (elements with more than one
    admissible value, how many of them took the rank-order sum)."""
    p_sequence, step_rows = CASES[case]
    per_rank = _spawn(world, "_bare_job", {"row_floats": row_floats, "case": case}, tmp_path)
    multi, rank_order = 0, 0
    for step, P in enumerate(p_sequence(world)):
        rows, touched = step_rows(world, row_floats, step, P)
        adm = em.admissible(rows, touched)
        fam = np.random.default_rng([world, row_floats]).integers(0, len(FAMILIES), CAPACITY)[:P]
        res0 = per_rank[0][step]["result"]
        for r in range(world):
            got = per_rank[r][step]
            assert np.array_equal(em.bits(got["result"]), em.bits(res0)), \
                f"step {step} (P {P}): rank {r}'s summed rows differ in their bits from rank 0's"
            ok = em.check_result(got["result"], adm)
            if not ok.all():
                i, j = np.argwhere(~ok)[0]
                raise AssertionError(
                    f"step {step} (P {P}, rows_per_rank {-(-P // world)}): rank {r}: {int((~ok).sum())} elements outside their admissible "
                    f"set; first row {i} ({FAMILIES[fam[i]] if case == "families" else case}) element {j}: got {got['result'][i, j]!r} (0x{int(em.bits(got['result'][i, j])):08x}), "
                    f"admissible {sorted(set('0x%08x' % b for b in adm[:, i, j]))}, contributions {rows[:, i, j].tolist()} touched {touched[:, i].tolist()}")
            want = em.accumulator_after(rows[r], touched[r])
            pushed = np.repeat(em.pushed_quarters(rows[r], touched[r]), 4, axis=-1)
            assert (got["acc"] == 0).all() and (em.bits(got["acc"])[pushed] == 0).all() and (em.bits(got["acc"]) == em.bits(want)).all(), \
                f"step {step} (P {P}): rank {r}'s accumulator is not cleared: {int((got['acc'] != 0).sum())} non-zero elements"
        mult = em.multi_admissible(adm)
        multi += int(mult.sum())
        rank_order += int((adm[0][mult] == em.bits(res0)[mult]).sum())
    return multi, rank_order


@pytest.mark.parametrize("row_floats", [16, 32])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_bare_step_is_an_admissible_sum(world, row_floats, tmp_path):
    """Thirteen steps on one exchange object (tests/exchange_model.py): every summed element admissible, bit for bit, and the
    same on every rank; every accumulator cleared."""
    t0 = time.monotonic()
    multi, rank_order = _check_bare(world, row_floats, "families", tmp_path)
    print(f"\n[exchange] world {world} row_floats {row_floats}: {multi} elements with more than one admissible value; "
          f"{rank_order} took the rank-order sum, {multi - rank_order} another order ({time.monotonic() - t0:.1f} s)")


@pytest.mark.parametrize("world", [2, 3])
def test_flushed_negative_zero_sum_reads_positive_zero_next_step(world, tmp_path):
    _check_bare(world, 16, "flushed_zero", tmp_path)


# ---- B. stage 1 through the exchange, C. GradExchange under gloo ---------------------------------------------------------

VARIANTS = {"coord_depth": (True, True, 0.1), "depth": (False, True, 0.0), "coord": (True, False, 0.0), "plain": (False, False, 0.1)}
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")


def _scene_file(tmp_path):
    """The multi-GPU tests' scene (60 000 splats, 640 x 400), built once here: processes that build "the same" scene on their
    own CPUs can differ in the last bits."""
    from rade_gs_b200 import scenes
    sc = scenes.make_scene(60000, 640, 400, 500.0, -3.8, seed=21, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.2, 0.1, 0.3))
    path = str(tmp_path / "scene.pt")
    torch.save(sc, path)
    return path


def _slabs(C, rawapi, multigpu, sc, coord, depth, ks, world, weighted):
    grid_y = multigpu.tile_rows(sc.height)
    if not weighted:
        return multigpu.partition_tile_rows(grid_y, world)
    f = rawapi.forward(C, sc, coord, depth, kernel_size=ks)   # weight = rendered alpha per tile row: slabs of unequal height
    w = f["alpha"][0].sum(1)
    w = torch.nn.functional.pad(w, (0, grid_y * 16 - sc.height)).view(grid_y, 16).sum(1)
    return multigpu.partition_tile_rows(grid_y, world, w.tolist())


def _digest(t):
    import hashlib
    return hashlib.sha1(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def _tiles_touched(rawapi, f, sc):
    """The per-splat tile counts of a (slab) forward: the third array of the geometry buffer (rgs_api.cu carve_geom)."""
    P, RF = sc.means3D.shape[0], 24 if f["_call"]["require_coord"] else 16
    g = rawapi._Cursor(f["geom"])
    g.take(P * RF, torch.float32, 4)
    g.take(P, torch.float32, 4)
    return g.take(P, torch.int32, 4)


def _stage1_job(rank, world, params):
    """Per variant, partition and map layout, three steps of slab forward -> stage 1 through the exchange -> backward-preprocess.
    Every rank returns digests of its rows and gradients; rank 0 and the last rank also check them against the whole-image
    backward of their own process (the results themselves are too large to ship)."""
    import torch.distributed as dist
    from diff_gaussian_rasterization import _C as C
    from rade_gs_b200 import multigpu, rawapi, scenes
    from rade_gs_b200.multigpu import GradExchange
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    sc0 = torch.load(params["scene"], weights_only=False).to(dev)
    P0 = sc0.means3D.shape[0]
    checks = rank == 0 or rank == world - 1
    out = {}
    for name, (coord, depth, ks) in VARIANTS.items():
        GS = C.grad_stride(coord, depth)
        ex, why = _connect(C, rank, world, P0, GS)
        if why is not None:
            return why
        try:
            for weighted in (False, True):
                slabs = _slabs(C, rawapi, multigpu, sc0, coord, depth, ks, world, weighted)
                b, e = slabs[rank]
                for compact in (False, True):
                    # three steps on one exchange object: new upstream gradients, then P - 1234 (rows re-associated)
                    for step, (seed, n) in enumerate(((5, P0), (6, P0), (7, P0 - 1234))):
                        what = f"world {world} {name} {'weighted' if weighted else 'equal'} slabs {slabs} {'compact' if compact else 'full-size'} step {step}"
                        sc = scenes.Scene(**{k: (v[:n] if k in ("means3D", "scales", "rotations", "opacities", "shs") else v)
                                             for k, v in sc0.__dict__.items()})
                        g = scenes.make_upstream_grads(sc.height, sc.width, seed=seed, device=dev)
                        f = rawapi.forward(C, sc, coord, depth, kernel_size=ks, tile_rows=(b, e), compact=compact)
                        gs = {k: v[:, min(b * 16, sc.height):min(e * 16, sc.height)] for k, v in g.items()} if compact else g
                        rows = C.rasterize_gaussians_backward_render_exchange(ex, *rawapi._backward_args(sc, f, gs), b, e, compact, sc.height)
                        _status(C, ex, what)
                        rows = rows.clone()
                        grads = rawapi.backward_preprocess(C, sc, f, rows)
                        touched = (_tiles_touched(rawapi, f, sc) != 0).int().cpu()
                        dist.all_reduce(touched, op=dist.ReduceOp.MAX)       # touched by some rank's slab
                        rec = {"rows": _digest(rows), **{"g_" + k: _digest(v) for k, v in grads.items()}, "error": None}
                        if checks:
                            try:
                                fw = rawapi.forward(C, sc, coord, depth, kernel_size=ks)
                                quiet = ((fw["radii"] == 0) | (touched == 0).to(dev))
                                assert int(quiet.sum()) > 0, "no quiet rows to check"
                                assert (rows[quiet].view(torch.int32) == 0).all(), \
                                    f"{what}: {int((rows[quiet] != 0).any(1).sum())} rows of unrendered or untouched Gaussians are not +0.0"
                                whole = [rawapi.backward_render(C, sc, fw, g).cpu() for _ in range(2)]
                                _close_to_whole(rows.cpu().numpy(), whole[0].numpy(), whole[1].numpy(), f"{what}: summed rows (rank {rank})")
                                ref = [rawapi.backward(C, sc, fw, g) for _ in range(2)]
                                for k in GRAD_KEYS:
                                    _close_to_whole(grads[k].cpu().numpy(), ref[0][k].cpu().numpy(), ref[1][k].cpu().numpy(), f"{what}: {k} (rank {rank})")
                                if (name, weighted, compact, step) == ("coord_depth", False, False, 0):
                                    out["whole"] = [w.numpy() for w in whole]
                            except AssertionError as err:
                                rec["error"] = str(err)
                        out[(name, weighted, compact, step)] = rec
        finally:
            _close(C, ex)
    # C. GradExchange(mode="peer") under gloo: its self-check, then one stage 1 through it (first variant, equal slabs)
    coord, depth, ks = VARIANTS["coord_depth"]
    gx = GradExchange(P0, C.grad_stride(coord, depth), dev, mode="peer")
    try:
        out["gx_mode"], out["gx_fallback"] = gx.mode, gx.fallback_reason
        b, e = multigpu.partition_tile_rows(multigpu.tile_rows(sc0.height), world)[rank]
        g = scenes.make_upstream_grads(sc0.height, sc0.width, seed=5, device=dev)
        f = rawapi.forward(C, sc0, coord, depth, kernel_size=ks, tile_rows=(b, e))
        rows = gx.backward_render(C, *rawapi._backward_args(sc0, f, g), b, e, False, sc0.height)
        if gx.mode == "peer":
            _status(C, gx._ex, "GradExchange")
        out["gx_digest"] = _digest(rows)
        if checks:
            out["gx_rows"] = rows.cpu().numpy()
    finally:
        gx.close()
    return out


def _close_to_whole(got, w1, w2, name):
    """Within tolerances.grad_close_gpu of the whole-image run, widened by 4x the spread of two whole-image runs."""
    import tolerances as tol
    w1, w2, got = (np.asarray(x, np.float64) for x in (w1, w2, got))
    noise_rel = tol.rel_l2(w1, w2)
    noise_max = float(np.abs(w1 - w2).max()) if w1.size else 0.0
    scale = float(np.abs(w1).max()) if w1.size else 1.0
    tol.grad_close_gpu(got, w1, name, rel=tol.GRAD_REL_L2_GPU + tol.GRAD_NOISE_FACTOR * noise_rel,
                       elem=tol.GRAD_ELEM_GPU + tol.GRAD_NOISE_FACTOR * noise_max / (scale + 1e-30))


@pytest.mark.parametrize("world", [2, 3, 4])
def test_stage1_through_the_exchange(world, tmp_path):
    """Slab forward + stage 1 through the exchange + backward-preprocess on every rank: rows and the eight gradients are the
    same bits on every rank, rows nobody pushed are +0.0, and the sums match the whole-image backward."""
    t0 = time.monotonic()
    per_rank = _spawn(world, "_stage1_job", {"scene": _scene_file(tmp_path)}, tmp_path)
    keys = [k for k in per_rank[0] if isinstance(k, tuple)]
    assert len(keys) == len(VARIANTS) * 12
    for key in keys:
        for r in range(world):
            rec = per_rank[r][key]
            assert rec["error"] is None, rec["error"]
            for k in ["rows"] + ["g_" + k for k in GRAD_KEYS]:
                assert rec[k] == per_rank[0][key][k], f"world {world} {key}: rank {r}'s {k} differ in their bits from rank 0's"
    # C: GradExchange(mode="peer") under gloo keeps the peer mode through its self-check and sums the same rows
    for r in range(world):
        assert per_rank[r]["gx_mode"] == "peer" and per_rank[r]["gx_fallback"] is None, (r, per_rank[r]["gx_fallback"])
        assert per_rank[r]["gx_digest"] == per_rank[0]["gx_digest"], f"GradExchange: rank {r}'s rows differ in their bits from rank 0's"
    w1, w2 = per_rank[0]["whole"]
    _close_to_whole(per_rank[0]["gx_rows"], w1, w2, f"world {world}: GradExchange rows")
    print(f"\n[exchange] world {world}: {len(keys)} stage-1 steps through the exchange and one through GradExchange "
          f"({time.monotonic() - t0:.1f} s)")
