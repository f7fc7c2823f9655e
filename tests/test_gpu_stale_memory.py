"""Stale memory and foreign streams: every `_C` entry point, run on memory pre-filled with a byte pattern and on a late-ready
side stream, gives what a clean run gives.

Two contracts the fresh-process, default-stream tests cannot see:
  * outputs are `empty()`-allocated and scratch is carved from uncleared buffers, so the kernels must write every element they
    return and read only words they wrote.  Inside a training loop those bytes hold the previous iteration's data;
  * work is queued on torch's CURRENT stream.  A launch, copy, memset or CUB call that fell back to the legacy stream would race
    a caller's torch side stream, which does not synchronise with stream 0.

Each case runs once clean (the reference), then once per byte pattern (0x00, 0x3B, 0x7F, 0xFF: 0xFF makes floats NaN and
integers -1) with `_C.set_poison(pattern)` (glue outputs and resize-callback scratch) and torch's caching allocator pre-filled
with the pattern (everything torch.empty hands out, the Python wrappers' buffers included), synchronising after every call.
Then once more on a new torch stream that first spins for about 100 ms and only then clones the inputs into pre-poisoned
memory: work enqueued anywhere else reads the pattern or races the clone.

Every deterministic output must be bit-identical to the reference (compared through an integer view: NaN == NaN).  The outputs
that depend on float-atomic order are the backward-render accumulator, the combined backward and the double sums of the SSIM
and normal losses.  For those: no non-finite value where the reference is finite, the same set of exactly-zero accumulator rows,
every gradient row whose reference accumulator row is zero exactly zero, and the rest within tolerances.grad_close_gpu of the
reference widened by 4x the larger spread of two further clean runs (the convention of tolerances.py); the double sums within
1e-9 relative.

The case table must name every entry of test_glue_host.ENTRIES and every `_C._densify` stage; a host test checks that.
Measured: the file's 116 cases take 90 s on one H100 80GB HBM3 (700 W power limit)."""
from __future__ import annotations

import copy

import numpy as np
import pytest
import torch

import tolerances as tol

DEV = "cuda"
PATTERNS = (0x00, 0x3B, 0x7F, 0xFF)
LARGE_BLOCK = 2 << 30          # one large-pool block (bytes)
SMALL_BLOCK, SMALL_TOTAL = 512 << 10, 64 << 20   # small-pool blocks (< 1 MiB each), 64 MiB of them
SMALL_LIMIT = 1 << 20          # the caching allocator's largest small-pool request
SPIN_CYCLES = 200_000_000      # about 100 ms at the H100's 1.98 GHz boost clock
DENSIFY_STAGES = {"select", "plan", "gather", "reset_opacity"}
E = torch.Tensor([])           # the rasterizer's "absent" convention


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


# ---- the pre-poisoned allocator ---------------------------------------------------------------------------------------

def _free_blocks():
    """(size, small pool?) of every cached free block the current stream can be handed."""
    stream = torch.cuda.current_stream().cuda_stream
    return [(b["size"], seg["segment_type"] == "small") for seg in torch.cuda.memory_snapshot() if seg["stream"] == stream
            for b in seg["blocks"] if b["state"] == "inactive"]


def _prefill(byte):
    """Leave torch's caching allocator, for the current stream, holding only blocks filled with `byte`, freed without empty_cache,
    so that torch.empty hands them out again: the free remainders of segments that live tensors keep (otherwise a best-fit request
    lands in one of those and sees whatever it held), one large-pool block and 64 MiB of small-pool blocks.  Checks that it does."""
    torch.cuda.empty_cache()
    held = []
    for _ in range(4):
        free = _free_blocks()
        if not free:
            break
        for size, small in sorted(free):
            while size > 0:       # a small-pool remainder serves requests of at most 1 MiB: take it in such pieces
                k = min(size, SMALL_LIMIT) if small else size
                held.append(torch.empty(k, dtype=torch.uint8, device=DEV).fill_(byte))
                size -= k
    held.append(torch.empty(LARGE_BLOCK, dtype=torch.uint8, device=DEV).fill_(byte))
    held += [torch.empty(SMALL_BLOCK, dtype=torch.uint8, device=DEV).fill_(byte) for _ in range(SMALL_TOTAL // SMALL_BLOCK)]
    del held
    for n in (1000, 4 << 20):      # one small-pool and one large-pool request
        t = torch.empty(n, dtype=torch.uint8, device=DEV)
        assert bool((t == byte).all()), f"torch.empty({n} bytes) did not come back filled with 0x{byte:02X}: the allocator pre-fill checks nothing"


@pytest.fixture
def poisoned_allocator():
    yield _prefill
    torch.cuda.empty_cache()


# ---- running a case ---------------------------------------------------------------------------------------------------

_SYNC = [True]


def _step():
    """After each entry point: synchronise, so that a fault is raised at the call that made it (not on the side stream, where
    that would end the race the run is there to provoke)."""
    if _SYNC[0]:
        torch.cuda.current_stream().synchronize()


def _clone(x):
    if torch.is_tensor(x):
        return x.clone() if x.is_cuda else x
    if isinstance(x, dict):
        return {k: _clone(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_clone(v) for v in x)
    if hasattr(x, "__dict__") and any(torch.is_tensor(v) for v in vars(x).values()):
        y = copy.copy(x)
        for k, v in vars(x).items():
            setattr(y, k, _clone(v))
        return y
    return x


class Case:
    """`inputs`: tensors (cloned per run) and anything else; `run(inputs)` -> {name: tensor or number}; `loose`: {name: kind} for
    the outputs that depend on float-atomic order: ("acc",), ("grad", accumulator name) or ("sum",)."""

    def __init__(self, inputs, run, loose=None, close=None):
        self.inputs, self.run, self.loose, self.close = inputs, run, loose or {}, close


def _int_view(t):
    t = t.detach().contiguous()
    if t.dtype == torch.bool:
        return t.view(torch.uint8)
    if t.is_floating_point():
        return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t


def _exact(name, got, ref):
    if not torch.is_tensor(ref):
        assert got == ref, f"{name}: {got} != {ref}"
        return
    assert got.shape == ref.shape and got.dtype == ref.dtype, f"{name}: {tuple(got.shape)} {got.dtype} != {tuple(ref.shape)} {ref.dtype}"
    bad = (_int_view(got) != _int_view(ref)).reshape(-1)
    n = int(bad.sum())
    if n:
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{name}: {n} of {ref.numel()} elements differ, first at flat index {i}: {got.reshape(-1)[i].item()} "
                             f"vs {ref.reshape(-1)[i].item()}")


def _np(t):
    return t.detach().double().cpu().numpy()


def _rows_zero(a):
    return (a.reshape(a.shape[0], -1) == 0).all(axis=1) if a.size else np.zeros(a.shape[0], bool)


def _loose(name, kind, got, ref, ref_all, spread):
    g, r = _np(got), _np(ref)
    assert g.shape == r.shape, f"{name}: shape {g.shape} != {r.shape}"
    lost = ~np.isfinite(g) & np.isfinite(r)
    assert not lost.any(), f"{name}: {int(lost.sum())} non-finite elements where the clean run is finite"
    if kind[0] == "sum":
        f = np.isfinite(r)
        assert np.array_equal(np.isfinite(g), f) and np.allclose(g[f], r[f], rtol=1e-9, atol=0), f"{name}: {g} vs {r}"
        return
    if kind[0] == "acc":
        zr, zg = _rows_zero(r), _rows_zero(g)
        assert np.array_equal(zr, zg), f"{name}: {int((zr != zg).sum())} rows differ in being exactly zero"
    else:
        zero = _rows_zero(_np(ref_all[kind[1]]))
        rows = g.reshape(g.shape[0], -1)[zero]
        assert not rows.any(), f"{name}: {int((rows != 0).any(axis=1).sum())} rows with a zero accumulator row are not zero"
    rel, elem = spread
    tol.grad_close_gpu(g, r, name, rel=tol.GRAD_REL_L2_GPU + tol.GRAD_NOISE_FACTOR * rel, elem=tol.GRAD_ELEM_GPU + tol.GRAD_NOISE_FACTOR * elem)


def _spread(a, b):
    """(relative L2, largest |difference| over the largest |value|) between two clean runs."""
    a, b = _np(a), _np(b)
    if not a.size:
        return 0.0, 0.0
    a, b = np.nan_to_num(a), np.nan_to_num(b)
    return tol.rel_l2(a, b), float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _compare(tag, got, ref, case, spreads):
    assert sorted(got) == sorted(ref), f"{tag}: outputs {sorted(got)} != {sorted(ref)}"
    for k in ref:
        if k in case.loose:
            _loose(f"{tag} {k}", case.loose[k], got[k], ref[k], ref, spreads[k])
        else:
            _exact(f"{tag} {k}", got[k], ref[k])


def _outputs(case, inputs):
    return {k: _clone(v) for k, v in case.run(inputs).items()}


def check_case(case, prefill):
    C = _C()
    try:
        C.set_poison(-1)
        _SYNC[0] = True
        ref = _outputs(case, _clone(case.inputs))
        torch.cuda.synchronize()
        spreads = {k: (0.0, 0.0) for k in case.loose}
        for _ in range(2 if case.loose else 0):      # the run-to-run spread of the float-atomic outputs: the largest of two draws
            again = _outputs(case, _clone(case.inputs))
            torch.cuda.synchronize()
            spreads = {k: tuple(map(max, spreads[k], _spread(again[k], ref[k]))) for k in case.loose}
        for pat in PATTERNS:
            C.set_poison(pat)
            prefill(pat)
            got = _outputs(case, _clone(case.inputs))
            torch.cuda.synchronize()
            _compare(f"poison 0x{pat:02X}:", got, ref, case, spreads)
        # the side stream: spin, then clone the inputs into pre-poisoned memory, run, clone the outputs, all on that stream
        C.set_poison(0xFF)
        _SYNC[0] = False
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            prefill(0xFF)
            torch.cuda._sleep(SPIN_CYCLES)
            got = _outputs(case, _clone(case.inputs))
        side.synchronize()
        torch.cuda.synchronize()
        _compare("side stream:", got, ref, case, spreads)
    finally:
        _SYNC[0] = True
        C.set_poison(-1)
        if case.close is not None:
            case.close()


# ---- the rasterizer ---------------------------------------------------------------------------------------------------

IMAGES = ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth")
VARIANTS = {"none": (False, False), "depth": (False, True), "coord": (True, False), "both": (True, True)}


def _upstream(sc, seed=17):
    from rade_gs_b200 import scenes
    return scenes.make_upstream_grads(sc.height, sc.width, seed=seed, device=DEV)


def _binning(f):
    from rade_gs_b200 import rawapi
    cur = rawapi._Cursor(f["binning"])
    R = int(f["num_rendered"])
    return cur.take(R, torch.int32, 4), cur.take(R, torch.int64, 8)


def _forward_outputs(f, sc, prefix="", whole=True):
    """The maps, radii and num_rendered; the meaningful views of the byte buffers (not their raw bytes)."""
    from rade_gs_b200 import rawapi
    out = {prefix + k: f[k] for k in IMAGES + ("radii", "num_rendered")}
    if whole:
        v = rawapi.ours_views(f, sc)
        for k in ("point_list", "keys", "ranges", "n_contrib"):
            out[prefix + k] = v[k]
    else:
        out[prefix + "point_list"], out[prefix + "keys"] = _binning(f)
    return out


def _scene(make):
    sc = make()
    return sc.to(DEV)


def raster_whole(make, coord, depth, ks):
    """forward -> backward_render -> backward_preprocess fed the clean accumulator -> the combined backward."""
    def build():
        from rade_gs_b200 import rawapi
        C = _C()
        sc = _scene(make)
        g = _upstream(sc)
        f = rawapi.forward(C, sc, coord, depth, kernel_size=ks)
        acc = rawapi.backward_render(C, sc, f, g)

        def run(x):
            sc, g = x["sc"], x["g"]
            f = rawapi.forward(C, sc, coord, depth, kernel_size=ks)
            _step()
            out = _forward_outputs(f, sc)
            out["acc"] = rawapi.backward_render(C, sc, f, g)
            _step()
            out.update({"stage2." + k: v for k, v in rawapi.backward_preprocess(C, sc, f, x["acc"]).items()})
            _step()
            out.update({"bwd." + k: v for k, v in rawapi.backward(C, sc, f, g).items()})
            _step()
            return out
        loose = {"acc": ("acc",)}
        loose.update({"bwd." + k: ("grad", "acc") for k in rawapi.BWD_KEYS})
        return Case({"sc": sc, "g": g, "acc": acc}, run, loose)
    return build


def raster_slabs(make, coord, depth, ks, K, compact):
    """K tile-row slabs: the slab forward and its backward_render, with full-height or compact maps."""
    def build():
        from rade_gs_b200 import multigpu, rawapi
        C = _C()
        sc = _scene(make)
        g = _upstream(sc)
        slabs = multigpu.partition_tile_rows((sc.height + 15) // 16, K)
        gs = [{k: v[:, b * 16: min(e * 16, sc.height)].contiguous() for k, v in g.items()} if compact else g for b, e in slabs]

        def run(x):
            out = {}
            for i, (b, e) in enumerate(slabs):
                f = rawapi.forward(C, x["sc"], coord, depth, kernel_size=ks, tile_rows=(b, e), compact=compact)
                _step()
                out.update(_forward_outputs(f, x["sc"], f"slab{i}.", whole=False))
                out[f"slab{i}.acc"] = rawapi.backward_render(C, x["sc"], f, x["gs"][i])
                _step()
            return out
        return Case({"sc": sc, "gs": gs}, run, {f"slab{i}.acc": ("acc",) for i in range(len(slabs))})
    return build


def _call(coord, depth, ks, sc):
    return dict(require_coord=coord, require_depth=depth, kernel_size=ks, sh_degree=3, scale_modifier=1.0, debug=False, tile_rows=None, compact=False,
                shs=sc.shs, cols=E, scales=sc.scales, rots=sc.rotations, cov=E)


def raster_split_sh(make, coord, depth, ks):
    """rasterize_gaussians_split_sh and rasterize_gaussians_backward_split_sh: features_dc and features_rest as two tensors."""
    def build():
        from rade_gs_b200 import rawapi
        C = _C()
        sc = _scene(make)
        g = _upstream(sc)
        keys = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh_dc", "sh_rest", "scales", "rotations")

        def run(x):
            sc, g = x["sc"], x["g"]
            dc, rest = sc.shs[:, :1].contiguous(), sc.shs[:, 1:].contiguous()
            c = _call(coord, depth, ks, sc)
            a = rawapi._forward_args(sc, c)
            f = dict(zip(rawapi.FWD_KEYS, C.rasterize_gaussians_split_sh(*a[:15], dc, rest, *a[16:])))
            f["_call"] = c
            _step()
            out = _forward_outputs(f, sc)
            out["acc"] = rawapi.backward_render(C, sc, f, g)
            _step()
            b = rawapi._backward_args(sc, f, g)
            out.update({"bwd." + k: v for k, v in zip(keys, C.rasterize_gaussians_backward_split_sh(*b[:21], dc, rest, *b[22:]))})
            _step()
            return out
        loose = {"acc": ("acc",)}
        loose.update({"bwd." + k: ("grad", "acc") for k in keys})
        return Case({"sc": sc, "g": g}, run, loose)
    return build


def raster_exchange(make, coord, depth, ks):
    """The device-side exchange at world 1 in one process: its bare step (exchange_rows) and stage 1 through it.  Only the rows
    of rendered Gaussians (radii > 0) are defined in the result; the others are neither pushed nor spread."""
    def build():
        from rade_gs_b200 import rawapi
        C = _C()
        sc = _scene(make)
        g = _upstream(sc)
        P, GS = sc.means3D.shape[0], C.grad_stride(coord, depth)
        idx = torch.cuda.current_device()
        ex, handle = C.exchange_create(0, 1, P, GS, idx)
        C.exchange_connect(ex, handle[None], idx)
        gen = torch.Generator().manual_seed(3)
        rows = (torch.randn(P, GS, generator=gen) * (torch.rand(P, 1, generator=gen) < 0.7)).to(DEV)
        touched = (rows != 0).any(1).int()
        radii = torch.where(torch.arange(P, device=DEV) % 11 == 5, 0, 1).int()

        def run(x):
            sc, g = x["sc"], x["g"]
            out = {}
            acc = C.exchange_accumulator(ex, P, GS, idx)
            acc.copy_(x["rows"])
            C.exchange_rows(ex, x["touched"], x["radii"])
            _step()
            out["rows.status"] = C.exchange_status(ex)
            vis = x["radii"] > 0
            out["rows.result"] = C.exchange_result(ex, P, GS, idx)[vis].clone()
            out["rows.accumulator"] = acc.clone()
            f = rawapi.forward(C, sc, coord, depth, kernel_size=ks)
            _step()
            out["radii"] = f["radii"]
            a = rawapi._backward_args(sc, f, g)
            res = C.rasterize_gaussians_backward_render_exchange(ex, *a, 0, -1, False, sc.height)
            _step()
            out["status"] = C.exchange_status(ex)
            out["acc"] = res[f["radii"] > 0].clone()
            return out
        return Case({"sc": sc, "g": g, "rows": rows, "touched": touched, "radii": radii}, run, {"acc": ("acc",)}, close=lambda: C.exchange_destroy(ex))
    return build


def mark_visible_case():
    from rade_gs_b200 import scenes
    sc = scenes.make_scene(5000, 160, 120, 140.0, -3.0, seed=5, view=scenes.look_at_view((0.3, 0.1, -0.5), (0.0, 0.0, 6.0))).to(DEV)
    return Case({"m": sc.means3D, "v": sc.viewmatrix, "p": sc.projmatrix}, lambda x: {"present": _C().mark_visible(x["m"], x["v"], x["p"])})


def integrate_case(fam):
    def build():
        import integrate_scenes as isc
        C = _C()
        case = isc.FAMILIES[fam]()
        sc = case.sc.to(DEV)
        M = (case.deg + 1) ** 2
        cols = case.colors_precomp.to(DEV) if case.colors_precomp is not None else E

        def run(x):
            sc = x["sc"]
            shs = E if x["cols"].numel() else sc.shs[:, :M].contiguous()
            r = C.integrate_gaussians_to_points(sc.bg, x["pts"], sc.means3D, x["cols"], sc.opacities, sc.scales, sc.rotations, 1.0, E, E, sc.viewmatrix,
                                                sc.projmatrix, sc.tanfovx, sc.tanfovy, 0.0, E, sc.height, sc.width, shs, case.deg, sc.campos, False, False)
            _step()
            out = dict(zip(("num_rendered", "color", "alpha_integrated", "color_integrated", "point_coordinate", "sdf", "radii"), r[:7]))
            f = dict(num_rendered=r[0], geom=r[7], binning=r[8], img=r[9], _call=dict(require_coord=False, require_depth=True))
            from rade_gs_b200 import rawapi
            v = rawapi.ours_views(f, sc)
            out.update({k: v[k] for k in ("point_list", "keys", "ranges")})    # integrate keeps no n_contrib in the image buffer
            return out
        return Case({"sc": sc, "pts": case.points.to(DEV), "cols": cols}, run)
    return build


# ---- per-Gaussian stages, losses and appearance ------------------------------------------------------------------------

def activation_case(P):
    def build():
        import activation_f64 as af
        C = _C()
        fam = af.families(seed=11)
        cols = [torch.cat([fam[k][i] for k in sorted(fam)]) for i in range(4)]
        n = cols[0].shape[0]
        idx = torch.randperm(max(P, n), generator=torch.Generator().manual_seed(P)) % n
        raw = [c[idx[:P]].contiguous().to(DEV) for c in cols]
        up = [u.to(DEV) for u in af.upstream(P, P)]
        gen = torch.Generator().manual_seed(P + 1)
        m2d = torch.randn(P, 3, generator=gen).to(DEV)
        radii = torch.randint(-1, 40, (P,), generator=gen).int().to(DEV)
        stats = [torch.rand(P, 1, generator=gen).to(DEV) for _ in range(4)] + [torch.randint(0, 30, (P,), generator=gen).float().to(DEV)]

        def run(x):
            out = dict(zip(("scales", "opacity", "rotations"), C.activate_forward(*x["raw"])))
            _step()
            out.update(zip(("d_raw_scaling", "d_raw_opacity", "d_raw_rotation"), C.activate_backward(*x["raw"], *x["up"])))
            _step()
            st = x["stats"]
            C.densification_stats(x["m2d"], x["radii"], *st)
            _step()
            out.update(zip(("grad_accum", "grad_accum_abs", "grad_accum_abs_max", "denom", "max_radii2D"), st))
            return out
        return Case({"raw": raw, "up": up, "m2d": m2d, "radii": radii, "stats": stats}, run)
    return build


def filter3d_case(n_cams, P):
    def build():
        from test_gpu_activation_exact import filter_scene
        from rade_gs_b200.fused import compute_3D_filter
        xyz, cams = filter_scene(n_cams, P, seed=n_cams)
        return Case({"xyz": torch.from_numpy(xyz).to(DEV)}, lambda x: {"filter_3D": compute_3D_filter(x["xyz"], cams)})
    return build


def image_loss_case(C_, H, W):
    def build():
        C = _C()
        gen = torch.Generator().manual_seed(H * 100 + W)
        gt = torch.rand(C_, H, W, generator=gen)
        img = (gt + 0.1 * torch.randn(C_, H, W, generator=gen)).clamp(0, 1)
        n = torch.nn.functional.normalize(torch.randn(3, H, W, generator=gen), dim=0)
        depth = 1.0 + torch.rand(2, 1, H, W, generator=gen)
        coord = torch.randn(2, 3, H, W, generator=gen) + torch.tensor([0.0, 0.0, 4.0])[:, None, None]
        lo, hi = H // 3, H - H // 4

        def run(x):
            sums, dmaps = C.ssim_l1_forward(x["img"], x["gt"], True)
            _step()
            out = {"sums": sums, "dmaps": dmaps}
            out["sums.no_grad"], out["dmaps.no_grad"] = C.ssim_l1_forward(x["img"], x["gt"], False)
            _step()
            out["sums.rows"], dmaps_rows = C.ssim_l1_forward(x["img"], x["gt"], True, lo, hi)
            _step()
            out["dmaps.rows"] = dmaps_rows[..., lo:hi, :]     # a row range's maps are defined on its rows only: the backward reads no others
            out["d_img"] = C.ssim_l1_backward(x["img"], x["gt"], dmaps, 0.2, 0.8, x["up"])
            _step()
            out["d_img.rows"] = C.ssim_l1_backward(x["img"], x["gt"], dmaps_rows, 0.2, 0.8, x["up"], lo, hi)
            _step()
            for tag, e, m, from_depth in (("depth", x["depth"][0], x["depth"][1], True), ("coord", x["coord"][0], x["coord"][1], False)):
                r = C.normal_consistency(x["n"], e, m, from_depth, 1.0 / 50.0, 1.0 / 60.0, W / 2.0, H / 2.0, 0.4, 0.6)
                _step()
                out.update(zip((f"{tag}.loss", f"{tag}.d_normal", f"{tag}.d_expected", f"{tag}.d_median"), r))
            return out
        inputs = {k: v.to(DEV) for k, v in dict(img=img, gt=gt, n=n, depth=depth, coord=coord, up=torch.tensor(1.7)).items()}
        return Case(inputs, run, {k: ("sum",) for k in ("sums", "sums.no_grad", "sums.rows", "depth.loss", "coord.loss")})
    return build


def appearance_case(name):
    def build():
        import appearance_f64 as af
        C = _C()
        inp = af.make_inputs(name)
        H0, W0 = inp["image"].shape[1:]
        H, W = H0 // 32 * 32, W0 // 32 * 32
        gen = torch.Generator().manual_seed(7)
        t = lambda a: torch.as_tensor(a).to(DEV)  # noqa: E731
        x = dict(image=t(inp["image"]), gt=t(inp["gt"]), up4=torch.relu(torch.randn(1, 16, H // 2, W // 2, generator=gen)).to(DEV),
                 w2=t(inp["params"][10]), b2=t(inp["params"][11]), w3=t(inp["params"][12]), b3=t(inp["params"][13]),
                 d_down=torch.randn(3, H0 // 32, W0 // 32, generator=gen).to(DEV), d_image=torch.randn(3, H0, W0, generator=gen).to(DEV),
                 up=torch.tensor(0.6, device=DEV))

        def run(x):
            out = {"down": C.appearance_downsample(x["image"])}
            _step()
            C.appearance_downsample_backward(x["d_down"], x["d_image"])
            _step()
            out["d_image_accumulated"] = x["d_image"]
            w = (x["w2"], x["b2"], x["w3"], x["b3"])
            out["loss"], out["act"], out["transformed"] = C.appearance_l1_forward(x["image"], x["gt"], x["up4"], *w, True, True)
            _step()
            out["loss.bare"], _, _ = C.appearance_l1_forward(x["image"], x["gt"], x["up4"], *w, False, False)
            _step()
            g = C.appearance_l1_backward(x["image"], x["gt"], x["up4"], out["act"], *w, x["up"])
            _step()
            out.update(zip(("d_img", "d_up4", "d_w2", "d_b2", "d_w3", "d_b3"), g))
            return out
        return Case(x, run)
    return build


def knn_case(family, P):
    def build():
        from test_gpu_knn import cloud
        return Case({"p": torch.from_numpy(cloud(family, P)).to(DEV)}, lambda x: {"dist2": _C().knn_mean_dist2(x["p"])})
    return build


# ---- densify ----------------------------------------------------------------------------------------------------------

def densify_case(name):
    """The three stages and reset_opacity on a fixture model with the optimizer state of one real Adam step; the random offsets
    are fixed draws scaled by the plan's standard deviations."""
    def build():
        import densify_model as dm
        D = _C()._densify
        d = dm.make_inputs(name)
        mg, mo, ext, mss = dm.arguments(d)
        pd = float(d["percent_dense"])
        P = d["in_xyz"].shape[0]
        x = {k[3:]: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in d.items() if k.startswith("in_") and not k.endswith(".step")}
        x["noise"] = torch.randn(2 * P, 3, generator=torch.Generator().manual_seed(P)).to(DEV)
        moments = [k for k in ("f_dc", "f_rest", "opacity", "rotation", "xyz", "scaling") if k + ".exp_avg" in x]

        def run(x):
            flags, offsets, ratio_q, counts = D.select(x["xyz_gradient_accum"], x["xyz_gradient_accum_abs"], x["denom"], x["scaling"], x["opacity"], mg,
                                                       pd * ext, mo, bool(mss), float(mss or 0), 0.1 * ext)
            _step()
            out = {"flags": flags, "offsets": offsets, "ratio_q": ratio_q, "counts": torch.tensor(counts)}
            src, draw, std_clone, std_split = D.plan(flags, offsets, counts, x["scaling"])
            _step()
            out.update(src=src, draw=draw, std_clone=std_clone, std_split=std_split)
            C_, S = counts[0], counts[1]
            columns = [(x[k], False) for k in ("f_dc", "f_rest", "opacity", "rotation")]
            columns += [(x[f"{k}.{m}"], True) for k in moments for m in ("exp_avg", "exp_avg_sq")]
            xyz, scaling, outs = D.gather(src, draw, C_, x["xyz"], x["rotation"], x["scaling"], std_clone * x["noise"][:C_],
                                          std_split * x["noise"][:2 * S], columns)
            _step()
            out.update(xyz=xyz, scaling=scaling)
            out.update({f"column{i}": t for i, t in enumerate(outs)})
            out["reset_opacity"] = D.reset_opacity(x["scaling"], x["opacity"], x["filter_3D"])
            _step()
            return out
        return Case(x, run)
    return build


# ---- TSDF, DTU, TNT, tetra --------------------------------------------------------------------------------------------

def tsdf_case(family):
    """A VoxelBlockGrid of one block whose frame hash starts at two slots: every view forces the touch retry and the first ones
    _grow and tsdf_rehash.  The grid state is compared by block key (pool indices depend on allocation order)."""
    def build():
        import tsdf_scenes as ts
        from rade_gs_b200.tsdf import VoxelBlockGrid
        sc = ts.make(family)
        views = [dict(d=torch.from_numpy(v.depth).to(DEV), c=torch.from_numpy(v.color).to(DEV), K=v.K, E=v.E) for v in sc.views]

        def run(x):
            vbg = VoxelBlockGrid(sc.vs, block_count=1, device=DEV)
            out = {}
            for i, v in enumerate(x["views"]):
                coords = vbg.compute_unique_block_coordinates(v["d"], v["K"], v["E"], sc.depth_scale, sc.depth_max, sc.trunc_mult)
                _step()
                out[f"view{i}.coords"] = coords
                vbg.integrate(coords, v["d"], v["c"], v["K"], v["E"], sc.depth_scale, sc.depth_max, sc.trunc_mult)
                _step()
            keys, pools = vbg.active_blocks()
            _step()
            pools = pools.long()
            out.update(keys=keys, tsdf=vbg.attribute("tsdf")[pools], weight=vbg.attribute("weight")[pools], color=vbg.attribute("color")[pools],
                       capacity=vbg.capacity, frame_slots=vbg.frame_keys.numel())
            mesh = vbg.extract_triangle_mesh(1.0 if family == "few_views" else 3.0)
            _step()
            mesh.compute_vertex_normals()
            _step()
            out.update(vertices=mesh.vertices, triangles=mesh.triangles, vertex_colors=mesh.vertex_colors, vertex_normals=mesh.vertex_normals)
            return out
        return Case({"views": views}, run)
    return build


def dtu_case():
    def build():
        import test_dtu_eval_host as h
        from rade_gs_b200 import dtu_eval
        C = _C()
        rng = np.random.default_rng(5)
        v = rng.normal(500, 3, (60, 3))
        f = rng.integers(0, 60, (150, 3))
        cull = h.load("cull")
        cams = h.cull_cameras(cull)
        x = dict(v=torch.as_tensor(v, device=DEV), f=torch.as_tensor(f, device=DEV).int(), masks=dtu_eval.cull_masks(cams, DEV),
                 cv=torch.as_tensor(cull["vertices"], device=DEV).double(), proj=torch.as_tensor(dtu_eval.cull_projections(cams), device=DEV).double(),
                 cloud=torch.as_tensor(np.concatenate([rng.normal(c, 0.3, (3000, 3)) for c in rng.uniform(480, 520, (5, 3))]), device=DEV),
                 q=torch.as_tensor(rng.uniform(470, 530, (20000, 3)), device=DEV))

        def run(x):
            out = {"samples": C.dtu_sample_mesh(x["v"], x["f"], 0.2)}
            _step()
            # the round count depends on when a round's threads see each other's decisions (rgs_dtu_eval.cu, ds_round_kernel);
            # the kept mask does not
            out["kept"], _ = C.dtu_radius_downsample(x["cloud"], 0.2)
            _step()
            out["dist"], out["index"] = C.dtu_nearest(x["cloud"], x["q"])
            _step()
            out["dilated"] = C.dtu_dilate_masks(x["masks"])
            _step()
            out["keep"] = C.dtu_cull_vertices(x["cv"], x["proj"], out["dilated"])
            _step()
            return out
        return Case(x, run)
    return build


def tnt_case():
    def build():
        from test_gpu_tnt_eval import POLY, _crop_points, _icp_scene
        C = _C()
        rng = np.random.default_rng(11)
        T = np.eye(4)
        T[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) * 1.25
        T[:3, 3] = [0.125, -0.25, 0.0625]
        src, tgt = _icp_scene(40)
        x = dict(p=torch.as_tensor(_crop_points(rng), device=DEV), poly=torch.as_tensor(POLY, device=DEV), T=torch.as_tensor(T),
                 vox=torch.as_tensor(rng.uniform(-7.5, 3.0, (30000, 3)), device=DEV), src=torch.as_tensor(src, device=DEV),
                 tgt=torch.as_tensor(tgt, device=DEV))

        def run(x):
            out = {}
            out["kept"], out["cropped"] = C.tnt_crop(x["p"], x["T"], 2, -0.5, 0.5, x["poly"])
            _step()
            out["kept.no_volume"], out["cropped.no_volume"] = C.tnt_crop(x["p"], E, 0, 0.0, 0.0, E)
            _step()
            moved = x["p"].clone()
            C.tnt_transform(moved, x["T"])
            _step()
            out["moved"] = moved
            out["means"], out["counts"] = C.tnt_voxel_downsample(x["vox"], 0.05)
            _step()
            d, i = C.dtu_nearest(x["tgt"], x["src"])
            _step()
            out["moments"] = C.tnt_icp_moments(x["src"], x["tgt"], d, i, 0.05)
            _step()
            return out
        return Case(x, run)
    return build


def tetra_case(name):
    """The whole tetrahedra extraction: tetra points, the cull SDF over the fixture's views, marching tetrahedra, eight bisection
    steps and the filter (rade_gs_b200.tetra drives tetra_cull_add / _finish, _marching, _bisect and _filter)."""
    def build():
        import tetra_scenes as scenes
        from test_tetra_host import load
        from rade_gs_b200 import tetra
        d = load(name)
        views = scenes.views_of(d)
        t = lambda k: torch.from_numpy(d[k]).to(DEV)  # noqa: E731

        def evaluate(points):
            cull = tetra.CullSDF(points.shape[0], points.device)
            for v in views:
                r = scenes.integrate(points, v)
                gt = None if v.gt_mask is None else torch.from_numpy(v.gt_mask).to(points.device)
                cull.add(r["alpha_integrated"], r["point_coordinate"], r["render"][7], gt)
                _step()
            s = cull.sdf()
            _step()
            return s

        def run(x):
            out = dict(zip(("tetra_points", "tetra_scales"), tetra.tetra_points(x["xyz"], x["scaling"], x["rotation"])))
            _step()
            sdf = evaluate(x["points"])
            out["sdf"] = sdf
            (ends, esdf), escl, faces, interp = [b[0] for b in tetra.marching_tetrahedra(x["points"][None], x["cells"], sdf[None], x["scales"][None])]
            _step()
            out.update(ends=ends, end_sdf=esdf, end_scales=escl, faces=faces, interp_v=interp)
            out["vertices"], out["out_faces"] = tetra.extract_mesh(x["points"], x["scales"], x["cells"], evaluate)
            _step()
            return out
        return Case({k: t(k) for k in ("xyz", "scaling", "rotation", "points", "scales")} | {"cells": t("cells").long()}, run)
    return build


# ---- the case table ---------------------------------------------------------------------------------------------------

def _cases():
    """{case id: (the `_C` entries it calls, builder)}.  Scenes are built lazily, on the GPU, when a case runs."""
    import blend_scenes as bs
    from rade_gs_b200 import scenes
    edge = lambda: bs.frustum_edge(200, 150, 300)                                            # noqa: E731
    whole_scenes = {"frustum_edge": edge, "tiny_17x16": lambda: bs.tiny(17, 16, 40), "tiny_1000x3": lambda: bs.tiny(1000, 3, 31),
                    "deep_8193": lambda: bs.deep([255, 8193, 513], seed=13), "opaque": lambda: bs.opaque(64, 48, 300)}
    fwd, bwd, render, pre = "rasterize_gaussians", "rasterize_gaussians_backward", "rasterize_gaussians_backward_render", \
        "rasterize_gaussians_backward_preprocess"
    cases = {}
    for v, (coord, depth) in VARIANTS.items():
        for ks in (0.0, 0.1):
            for sname, make in whole_scenes.items():
                cases[f"raster/{v}/ks{ks}/{sname}"] = ({fwd, render, pre, bwd}, raster_whole(make, coord, depth, ks))
            for K in (2, 8):
                for compact in (False, True):
                    cases[f"slabs/{v}/ks{ks}/K{K}/{'compact' if compact else 'full'}"] = (
                        {"rasterize_gaussians_slab", render}, raster_slabs(edge, coord, depth, ks, K, compact))
    cases["raster/both/ks0.1/C1"] = ({fwd, render, pre, bwd}, raster_whole(lambda: scenes.make_config("C1")[0], True, True, 0.1))
    for v in ("depth", "both"):
        cases[f"split_sh/{v}"] = ({"rasterize_gaussians_split_sh", "rasterize_gaussians_backward_split_sh", render},
                                  raster_split_sh(edge, *VARIANTS[v], 0.1))
    cases["exchange/world1"] = ({"exchange_rows", "rasterize_gaussians_backward_render_exchange", fwd}, raster_exchange(edge, False, True, 0.1))
    cases["mark_visible"] = ({"mark_visible"}, mark_visible_case)
    for fam in ("ragged_97x61", "ragged_1x1", "deep_lists", "corners_crowding", "colour_precomp"):
        cases[f"integrate/{fam}"] = ({"integrate_gaussians_to_points"}, integrate_case(fam))
    for P in (1, 257, 100_003):
        cases[f"activation/P{P}"] = ({"activate_forward", "activate_backward", "densification_stats"}, activation_case(P))
    for n_cams, P in ((1, 1000), (257, 4097)):
        cases[f"filter3d/{n_cams}cams"] = ({"compute_3d_filter"}, filter3d_case(n_cams, P))
    for C_, H, W in ((3, 33, 101), (1, 17, 5), (3, 1, 32)):
        cases[f"image_loss/{C_}x{H}x{W}"] = ({"ssim_l1_forward", "ssim_l1_backward", "normal_consistency"}, image_loss_case(C_, H, W))
    for name in ("odd_offsets", "ragged_tiles"):
        cases[f"appearance/{name}"] = ({"appearance_downsample", "appearance_downsample_backward", "appearance_l1_forward", "appearance_l1_backward"},
                                       appearance_case(name))
    for family, P in (("uniform", 20000), ("lattice", 1000), ("identical", 33), ("uniform", 1)):
        cases[f"knn/{family}/{P}"] = ({"knn_mean_dist2"}, knn_case(family, P))
    import densify_model as dm
    for name in dm.CASES:
        cases[f"densify/{name}"] = ({"_densify." + s for s in DENSIFY_STAGES}, densify_case(name))
    for family in ("sphere", "occluders", "masked", "few_views"):
        cases[f"tsdf/{family}"] = ({"tsdf_touch", "tsdf_integrate", "tsdf_rehash", "tsdf_active_blocks", "tsdf_extract", "tsdf_vertex_normals"},
                                   tsdf_case(family))
    cases["dtu"] = ({"dtu_sample_mesh", "dtu_radius_downsample", "dtu_nearest", "dtu_dilate_masks", "dtu_cull_vertices"}, dtu_case())
    cases["tnt"] = ({"tnt_crop", "tnt_transform", "tnt_voxel_downsample", "tnt_icp_moments", "dtu_nearest"}, tnt_case())
    for name in ("sphere_gt", "sphere_nogt", "empty"):
        cases[f"tetra/{name}"] = ({"tetra_points", "tetra_cull_add", "tetra_cull_finish", "tetra_marching", "tetra_bisect", "tetra_filter"},
                                  tetra_case(name))
    return cases


CASES = _cases()


def test_every_entry_point_has_a_case():
    """A new `_C` entry point, or `_C._densify` stage, cannot skip this file."""
    import diff_gaussian_rasterization as dgr
    from test_glue_host import ENTRIES
    covered = set().union(*(entries for entries, _ in CASES.values()))
    stages = {n for n in dir(dgr._C._densify) if not n.startswith("_")}
    assert stages == DENSIFY_STAGES
    assert covered == set(ENTRIES) | {"_densify." + s for s in stages}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_poisoned_memory_and_a_late_side_stream_change_nothing(name, poisoned_allocator):
    check_case(CASES[name][1](), poisoned_allocator)
