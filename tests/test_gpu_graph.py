"""The rasterizer forward binned into a reserved capacity (rgs_forward_preset, `_C._graph`) and the training step captured in a
CUDA graph (rade_gs_b200.graphs): bit-identical to rgs_forward for every frame that fits, safe and flagged for one that does not."""
from __future__ import annotations

import ctypes
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden
from test_gpu_stale_memory import poisoned_allocator  # noqa: F401  (fixture)
from tolerances import grad_close_gpu

DEV = "cuda"
E = torch.Tensor([])
IMAGES = ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth")
GRADS = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")
pytestmark = pytest.mark.gpu


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(name, a, b):
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.equal(_bits(a), _bits(b)), f"{name}: not bit-identical"


def _call(sc, coord, depth, ks=0.0, deg=3, extra=None):
    """rawapi.forward's call description, so that rawapi's views and backward read a preset forward too."""
    extra = extra or {}
    cols, cov = extra.get("colors_precomp"), extra.get("cov3D_precomp")
    return dict(require_coord=coord, require_depth=depth, kernel_size=ks, sh_degree=deg, scale_modifier=1.0, debug=False, tile_rows=None,
                compact=False, shs=E if cols is not None else sc.shs, cols=cols if cols is not None else E,
                scales=E if cov is not None else sc.scales, rots=E if cov is not None else sc.rotations, cov=cov if cov is not None else E)


def _preset_forward(sc, c, instances, longest, status):
    from rade_gs_b200 import rawapi
    out = _C()._graph.rasterize_gaussians(*rawapi._forward_args(sc, c), E, instances, longest, status)
    res = dict(zip(rawapi.FWD_KEYS, out))
    res["_call"] = c
    return res


def _totals(f, sc):
    from rade_gs_b200 import rawapi
    R, L = (int(x) for x in rawapi.ours_views(f, sc)["totals"].tolist())
    return R, L


def _same_forward(tag, f, ref, sc, R):
    from rade_gs_b200 import rawapi
    for k in IMAGES + ("radii",):
        _same(f"{tag} {k}", f[k], ref[k])
    v, w = rawapi.ours_views(f, sc), rawapi.ours_views(ref, sc)
    for k in ("point_list", "keys"):
        _same(f"{tag} {k}", v[k][:R], w[k][:R])
    for k in ("ranges", "n_contrib", "totals"):
        _same(f"{tag} {k}", v[k], w[k])


def _grads_close(tag, b, ref, ref2):
    """Within the bars widened by GRAD_NOISE_FACTOR times the eager backward's own run-to-run spread (ref against ref2), the
    convention of tolerances.py: both accumulate with float atomics."""
    from tolerances import GRAD_ELEM_GPU, GRAD_NOISE_FACTOR, GRAD_REL_L2_GPU, rel_l2
    for k in GRADS:
        a, r, r2 = (np.asarray(t[k].cpu().numpy(), np.float64) for t in (b, ref, ref2))
        m = max(np.abs(r).max(), 1e-30) if r.size else 1.0
        rel = GRAD_REL_L2_GPU + GRAD_NOISE_FACTOR * rel_l2(r2, r)
        elem = GRAD_ELEM_GPU + GRAD_NOISE_FACTOR * (np.abs(r2 - r).max() / m if r.size else 0.0)
        grad_close_gpu(a, r, f"{tag} {k}", rel=rel, elem=elem)


# ---- 1. preset equals exact --------------------------------------------------------------------------------------------

def _golden_scene(name):
    from test_gpu_parity import _scene_from_golden
    d = load_golden(name)
    sc, extra = _scene_from_golden(d)
    return sc, _call(sc, bool(d["meta_coord"]), bool(d["meta_depth"]), float(d["meta_ks"]), int(d["meta_deg"]), extra)


def _c2_scene():
    from rade_gs_b200 import scenes
    sc, coord, depth = scenes.make_config("C2")
    sc = sc.to(DEV)
    return sc, _call(sc, coord, depth)


def _long_tile():
    from test_gpu_parity import _long_tile_scene
    _, both, coord, depth = _long_tile_scene()
    sc = both.to(DEV)
    return sc, _call(sc, coord, depth)


SCENES = {**{g: (lambda g=g: _golden_scene(g)) for g in GOLDEN_CASES}, "C2": _c2_scene, "long_tile": _long_tile}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_preset_equals_exact(name):
    from rade_gs_b200 import rawapi, scenes
    sc, c = SCENES[name]()
    C = _C()
    ref = rawapi.forward(C, sc, c["require_coord"], c["require_depth"], kernel_size=c["kernel_size"], sh_degree=c["sh_degree"],
                         colors_precomp=c["cols"] if c["cols"].numel() else None, cov3D_precomp=c["cov"] if c["cov"].numel() else None)
    R, L = _totals(ref, sc)
    assert R == ref["num_rendered"]
    if name == "long_tile":
        assert L > 8192, "the scene must have a list longer than the one-CTA sort"
    # exact fit, headroom, and a list capacity four merge passes beyond the need (every short list skips the long path)
    chunks = max(1, math.ceil(L / 4096))
    beyond = 4096 * 2 ** (math.ceil(math.log2(chunks)) + 4)
    presets = [(R, L), (R + R // 4 + 65536, L + L // 4 + 256), (R, beyond)]
    grads = scenes.make_upstream_grads(sc.height, sc.width, seed=5, device=DEV)
    b_ref, b_ref2 = rawapi.backward(C, sc, ref, grads), rawapi.backward(C, sc, ref, grads)
    for inst, lst in presets:
        status = torch.zeros(4, dtype=torch.int32, device=DEV)
        f = _preset_forward(sc, c, inst, lst, status)
        assert f["num_rendered"] == inst
        _same_forward(f"{name} preset ({inst}, {lst})", f, ref, sc, R)
        assert status.tolist() == [0, R, L, 0]
        _grads_close(f"{name} preset ({inst}, {lst})", rawapi.backward(C, sc, f, grads), b_ref, b_ref2)


# ---- scenes of the capture tests -----------------------------------------------------------------------------------------

def _views(n, radius=6.0, seed=3):
    from rade_gs_b200 import scenes
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        a = 2 * math.pi * i / n
        eye = (radius * 0.15 * math.sin(a), radius * 0.1 * math.cos(a), -0.3 + 0.2 * float(torch.rand(1, generator=g)))
        out.append(scenes.look_at_view(eye, (0.05 * math.cos(a), 0.0, 6.0)))
    return out


def _camera(sc, V):
    """viewmatrix, projmatrix, campos of sc's intrinsics for the maths-convention view V (as scenes.make_scene builds them)."""
    from rade_gs_b200 import scenes
    viewmatrix = V.t().contiguous()
    proj = scenes.projection_matrix(0.01, 100.0, 2 * math.atan(sc.tanfovx), 2 * math.atan(sc.tanfovy)).t()
    return viewmatrix, (viewmatrix @ proj).contiguous(), viewmatrix.inverse()[3, :3].contiguous()


def _settings(sc, view, proj, campos, coord=False, depth=True, deg=3):
    import diff_gaussian_rasterization as dgr
    return dgr.GaussianRasterizationSettings(sc.height, sc.width, sc.tanfovx, sc.tanfovy, 0.0, sc.bg, 1.0, view, proj, deg, campos, False, depth,
                                             coord, False)


# ---- 2. the rasterizer under capture -----------------------------------------------------------------------------------

def test_rasterizer_forward_backward_under_capture():
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import rawapi, scenes
    from rade_gs_b200.graphs import BinningReserve
    base = scenes.make_scene(60_000, 320, 240, 300.0, -4.0, seed=11, bg=(0.1, 0.2, 0.3)).to(DEV)
    cams = [_camera(base, V) for V in _views(8)]
    gen = torch.Generator(device=DEV).manual_seed(12)
    inputs = [(base.means3D + 0.01 * i * torch.randn(base.means3D.shape, generator=gen, device=DEV), base.shs, base.scales, base.rotations,
               base.opacities, *[t.to(DEV) for t in cams[i]]) for i in range(8)]
    up = scenes.make_upstream_grads(base.height, base.width, seed=13, device=DEV)

    # the reserve fitted to every frame of the test, so that no replay overflows
    reserve = BinningReserve(DEV)
    want = []
    for x in inputs:
        sc = scenes.Scene(x[0], x[2], x[3], x[4], x[1], x[5], x[6], x[7], base.bg, base.width, base.height, base.tanfovx, base.tanfovy)
        want.append(_totals(rawapi.forward(_C(), sc, False, True), sc))
    reserve.fit(max(r for r, _ in want), max(l for _, l in want))

    static = [t.clone() for t in inputs[0]]
    means, shs, scales, rots, opac, view, proj, campos = static
    params = [means, shs, scales, rots, opac]
    for p in params:
        p.requires_grad_(True)
    means2D = torch.zeros_like(means, requires_grad=True)
    params.append(means2D)
    rast = dgr.GaussianRasterizer(_settings(base, view, proj, campos), reserve)

    def step():
        color, radii, coord, mcoord, depth, mdepth, alpha, normal = rast(means, means2D, opac, shs=shs, scales=scales, rotations=rots)
        loss = (color * up["color"]).sum() + (depth * up["depth"]).sum() + (mdepth * up["mdepth"]).sum() + (alpha * up["alpha"]).sum() \
            + (normal * up["normal"]).sum()
        loss.backward()
        return color.detach(), depth.detach(), mdepth.detach(), alpha.detach(), normal.detach(), radii

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        reserve.clear()
        for p in params:
            p.grad.zero_()
        outs = step()

    for i, x in enumerate(inputs):
        with torch.no_grad():
            for s, v in zip(static, x):
                s.copy_(v)
        graph.replay()
        torch.cuda.synchronize()
        got = [o.clone() for o in outs]
        got_grads = [p.grad.clone() for p in params]
        assert reserve.read() == (0, *want[i])

        e = [t.clone().requires_grad_(k < 5) for k, t in enumerate(x)]
        e2D = torch.zeros_like(e[0], requires_grad=True)
        er = dgr.GaussianRasterizer(_settings(base, e[5], e[6], e[7]))
        color, radii, coord, mcoord, depth, mdepth, alpha, normal = er(e[0], e2D, e[4], shs=e[1], scales=e[2], rotations=e[3])
        ((color * up["color"]).sum() + (depth * up["depth"]).sum() + (mdepth * up["mdepth"]).sum() + (alpha * up["alpha"]).sum()
         + (normal * up["normal"]).sum()).backward()
        for name, a, b in zip(("color", "depth", "mdepth", "alpha", "normal", "radii"), got, (color, depth, mdepth, alpha, normal, radii)):
            _same(f"camera {i} {name}", a, b)
        for name, a, b in zip(("means3D", "shs", "scales", "rotations", "opacity", "means2D"), got_grads, [t.grad for t in e[:5]] + [e2D.grad]):
            grad_close_gpu(a.cpu().numpy(), b.cpu().numpy(), f"camera {i} {name}")


# ---- 3. the whole step under StepGraph ----------------------------------------------------------------------------------

class _Up(torch.nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.shuffle = torch.nn.PixelShuffle(2)
        self.conv = torch.nn.Conv2d(cin, cout, 3, padding=1)
        self.relu = torch.nn.ReLU()


class _Net(torch.nn.Module):
    """The architecture of the appearance network (scene/appearance_network.py; layer names and parameter order)."""

    def __init__(self):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(67, 256, 3, padding=1)
        self.up1, self.up2, self.up3, self.up4 = _Up(64, 128), _Up(32, 64), _Up(16, 32), _Up(8, 16)
        self.conv2 = torch.nn.Conv2d(16, 16, 3, padding=1)
        self.conv3 = torch.nn.Conv2d(16, 3, 3, padding=1)
        self.relu = torch.nn.ReLU()


class _Model:
    """The parameters a training step reads, raw (before activation) as GaussianModel keeps them."""

    def __init__(self, sc, n_views, seed=21):
        torch.manual_seed(seed)
        self._xyz = sc.means3D.clone().requires_grad_(True)
        self._scaling = torch.log(sc.scales).clone().requires_grad_(True)
        self._opacity = torch.logit(sc.opacities.clamp(1e-4, 1 - 1e-4)).clone().requires_grad_(True)
        self._rotation = (sc.rotations * 1.7).clone().requires_grad_(True)
        self._features_dc = sc.shs[:, :1].clone().requires_grad_(True)
        self._features_rest = sc.shs[:, 1:].clone().contiguous().requires_grad_(True)
        self.filter_3D = torch.full((sc.means3D.shape[0], 1), 0.01, device=DEV)
        self.appearance_network = _Net().to(DEV)
        self._appearance_embeddings = torch.nn.Parameter(0.1 * torch.randn(n_views, 64, device=DEV))

    def get_apperance_embedding(self, idx):
        # the view's row without a host read: a 0-dim CUDA index through index_select (plain indexing would call .item())
        return self._appearance_embeddings.index_select(0, idx.reshape(1))[0]

    def params(self):
        return [self._xyz, self._scaling, self._opacity, self._rotation, self._features_dc, self._features_rest, self._appearance_embeddings,
                *self.appearance_network.parameters()]


class _Step:
    """train.py's step with the fused pieces: activation, split-SH depth-variant render, L1+SSIM, depth-normal consistency and the
    decoupled-appearance L1; the camera, ground truth and view index live in static device tensors."""

    def __init__(self, model, sc, reserve):
        import diff_gaussian_rasterization as dgr
        self.m, self.sc = model, sc
        self.view, self.proj, self.campos = (torch.zeros(4, 4, device=DEV), torch.zeros(4, 4, device=DEV), torch.zeros(3, device=DEV))
        self.gt = torch.zeros(3, sc.height, sc.width, device=DEV)
        self.view_idx = torch.zeros((), dtype=torch.int64, device=DEV)
        self.means2D = torch.zeros_like(model._xyz, requires_grad=True)
        self.cam = SimpleNamespace(FoVx=2 * math.atan(sc.tanfovx), FoVy=2 * math.atan(sc.tanfovy))
        self.rast = dgr.GaussianRasterizer(_settings(sc, self.view, self.proj, self.campos, deg=3), reserve)

    def load(self, cam, gt, idx):
        with torch.no_grad():
            for s, v in zip((self.view, self.proj, self.campos), cam):
                s.copy_(v)
            self.gt.copy_(gt)
            self.view_idx.fill_(idx)

    def params(self):
        return self.m.params() + [self.means2D]

    def __call__(self):
        from rade_gs_b200.appearance import L1_loss_appearance
        from rade_gs_b200.fused import activate_gaussians
        from rade_gs_b200.losses import depth_normal_consistency_loss, l1_ssim_loss
        m = self.m
        scales, opacity, rotations = activate_gaussians(m._scaling, m._opacity, m._rotation, m.filter_3D)
        color, radii, coord, mcoord, depth, mdepth, alpha, normal = self.rast(m._xyz, self.means2D, opacity, shs=(m._features_dc, m._features_rest),
                                                                              scales=scales, rotations=rotations)
        loss = l1_ssim_loss(color, self.gt, 0.2) + 0.05 * depth_normal_consistency_loss(self.cam, normal, depth, mdepth) \
            + L1_loss_appearance(color, self.gt, m, self.view_idx)
        loss.backward()
        return loss.detach(), radii


def _step_scene(P=40_000, seed=41):
    from rade_gs_b200 import scenes
    return scenes.make_scene(P, 256, 192, 240.0, -3.8, seed=seed, bg=(0.0, 0.0, 0.0)).to(DEV)


def _eager_step(sc, model_state, cam, gt, idx, n_views):
    m = _Model(sc, n_views)
    with torch.no_grad():
        for p, v in zip(m.params(), model_state):
            p.copy_(v)
    s = _Step(m, sc, None)
    s.load(cam, gt, idx)
    loss, radii = s()
    return loss, radii, [p.grad for p in s.params()]


def _key(sc, step):
    return (sc.height, sc.width, sc.tanfovx, sc.tanfovy, 3, 0.0, False, True, sc.means3D.shape[0], *(p.data_ptr() for p in step.params()))


def _check_step(tag, loss, radii, grads, ref):
    rloss, rradii, rgrads = ref
    assert abs(float(loss) - float(rloss)) <= 1e-5 * abs(float(rloss)) + 1e-7, (tag, float(loss), float(rloss))
    _same(f"{tag} radii", radii, rradii)
    for i, (a, b) in enumerate(zip(grads, rgrads)):
        grad_close_gpu(a.cpu().numpy(), b.cpu().numpy(), f"{tag} grad {i}")


def test_whole_step_under_stepgraph():
    from rade_gs_b200.graphs import BinningReserve, StepGraph
    sc = _step_scene()
    n = 8
    cams = [tuple(t.to(DEV) for t in _camera(sc, V)) for V in _views(n, seed=5)]
    gts = [torch.rand(3, sc.height, sc.width, generator=torch.Generator(device=DEV).manual_seed(100 + i), device=DEV) for i in range(n)]
    model = _Model(sc, n)
    state = [p.detach().clone() for p in model.params()]
    reserve = BinningReserve(DEV)
    step = _Step(model, sc, reserve)
    sg = StepGraph(reserve)
    key = _key(sc, step)
    for i in range(n):
        step.load(cams[i], gts[i], i)
        loss, radii = sg.run(key, step, step.params())
        torch.cuda.synchronize()
        grads = [p.grad.clone() for p in step.params()]
        _check_step(f"camera {i}", loss.clone(), radii.clone(), grads, _eager_step(sc, state, cams[i], gts[i], i, n))
    assert sg.captures + sg.fallbacks >= 1 and len(sg) <= 1


# ---- 4. overflow ---------------------------------------------------------------------------------------------------------

class _CCam(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float),
                ("kernel_size", ctypes.c_float), ("scale_modifier", ctypes.c_float), ("viewmatrix", ctypes.c_void_p), ("projmatrix", ctypes.c_void_p),
                ("cam_pos", ctypes.c_void_p), ("background", ctypes.c_void_p), ("sh_degree", ctypes.c_int32), ("sh_coeffs", ctypes.c_int32),
                ("require_coord", ctypes.c_int32), ("require_depth", ctypes.c_int32), ("prefiltered", ctypes.c_int32), ("debug", ctypes.c_int32),
                ("tile_row_begin", ctypes.c_int32), ("tile_row_end", ctypes.c_int32), ("compact_slab", ctypes.c_int32)]


class _CGs(ctypes.Structure):
    _fields_ = [("P", ctypes.c_int32)] + [(n, ctypes.c_void_p) for n in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations",
                                                                         "cov3D_precomp", "shs_rest")]


class _CPreset(ctypes.Structure):
    _fields_ = [("instances", ctypes.c_int64), ("longest_list", ctypes.c_int32), ("status", ctypes.c_void_p)]


_RESIZE = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
CANARY = 1 << 16


def _ctypes_preset(sc, instances, longest):
    """rgs_forward_preset through the C ABI; the binning callback hands out CANARY more bytes than asked, filled with 0xA5."""
    from rade_gs_b200 import LIB_PATH
    lib = ctypes.CDLL(LIB_PATH)
    lib.rgs_forward_preset.restype = ctypes.c_int64
    lib.rgs_last_error.restype = ctypes.c_char_p
    keep = {}

    def grower(name, canary):
        def fn(user, nbytes):
            t = torch.full((nbytes + (CANARY if canary else 0),), 0xA5 if canary else 0, dtype=torch.uint8, device=DEV)
            keep[name] = (t, nbytes)
            return t.data_ptr()
        return _RESIZE(fn)

    cbs = [grower("geom", False), grower("binning", True), grower("image", False)]
    H, W = sc.height, sc.width
    maps = {k: torch.full((3 if k in ("color", "coord", "mcoord", "normal") else 1, H, W), 7.0, device=DEV) for k in IMAGES}
    radii = torch.full((sc.means3D.shape[0],), -5, dtype=torch.int32, device=DEV)
    status = torch.zeros(4, dtype=torch.int32, device=DEV)
    cam = _CCam(W, H, sc.tanfovx, sc.tanfovy, 0.0, 1.0, sc.viewmatrix.data_ptr(), sc.projmatrix.data_ptr(), sc.campos.data_ptr(), sc.bg.data_ptr(),
                3, 16, 0, 1, 0, 0, 0, -1, 0)
    gs = _CGs(sc.means3D.shape[0], sc.means3D.data_ptr(), sc.opacities.data_ptr(), sc.shs.data_ptr(), None, sc.scales.data_ptr(),
              sc.rotations.data_ptr(), None, None)
    out = (ctypes.c_void_p * 8)(*[maps[k].data_ptr() for k in ("color", "coord", "mcoord", "alpha", "normal", "depth", "mdepth")], radii.data_ptr())
    bufs = (ctypes.c_void_p * 6)(ctypes.cast(cbs[0], ctypes.c_void_p), None, ctypes.cast(cbs[1], ctypes.c_void_p), None,
                                 ctypes.cast(cbs[2], ctypes.c_void_p), None)
    preset = _CPreset(instances, longest, status.data_ptr())
    rc = lib.rgs_forward_preset(ctypes.byref(cam), ctypes.byref(gs), out, bufs, ctypes.byref(preset),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == instances, lib.rgs_last_error()
    binning, nbytes = keep["binning"]
    return maps, radii, status, binning[nbytes:]


@pytest.mark.parametrize("which", ["instances", "list", "both"])
def test_overflow_is_flagged_and_writes_nothing_outside(which):
    from rade_gs_b200 import rawapi, scenes
    sc = scenes.make_scene(50_000, 320, 240, 300.0, -4.0, seed=61, bg=(0.25, 0.5, 0.75)).to(DEV)
    ref = rawapi.forward(_C(), sc, False, True)
    R, L = _totals(ref, sc)
    inst = R // 3 if which in ("instances", "both") else R
    lst = L // 2 if which in ("list", "both") else L
    maps, radii, status, tail = _ctypes_preset(sc, inst, lst)
    bits = {"instances": 1, "list": 2, "both": 3}[which]
    assert status.tolist() == [bits, R, L, 0]
    assert bool((tail == 0xA5).all()), "bytes after the binning buffer were written"
    _same("radii", radii, ref["radii"])
    assert torch.equal(maps["color"], sc.bg[:, None, None].expand(3, sc.height, sc.width).contiguous()), "maps must be the background"
    assert bool((maps["alpha"] == 0).all())
    # the same frame in a reserve that fits: rgs_forward's maps
    maps, radii, status, tail = _ctypes_preset(sc, R, L)
    assert status.tolist() == [0, R, L, 0] and bool((tail == 0xA5).all())
    for k in IMAGES:
        _same(k, maps[k], ref[k])


def test_stepgraph_overflow_grows_the_reserve_and_runs_the_step_eagerly():
    from rade_gs_b200.graphs import BinningReserve, StepGraph
    from rade_gs_b200 import scenes
    from rade_gs_b200 import rawapi
    sc = _step_scene(P=300_000, seed=43)
    far = tuple(t.to(DEV) for t in _camera(sc, scenes.look_at_view((0.0, 0.0, 0.0), (8.0, 0.0, 6.0))))     # sees the scene's edge only
    near = tuple(t.to(DEV) for t in _camera(sc, scenes.look_at_view((0.0, 0.0, 0.0), (0.0, 0.0, 6.0))))    # sees all of it
    counts = []
    for cam in (far, near):
        s2 = scenes.Scene(sc.means3D, sc.scales, sc.rotations, sc.opacities, sc.shs, *cam, sc.bg, sc.width, sc.height, sc.tanfovx, sc.tanfovy)
        counts.append(_totals(rawapi.forward(_C(), s2, False, True), s2)[0])
    fitted = BinningReserve("cpu")
    fitted.fit(counts[0], 0)
    assert counts[1] > fitted.instances, ("the near frame must outgrow the far frame's reserve", counts)
    gt = torch.rand(3, sc.height, sc.width, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    model = _Model(sc, 2)
    state = [p.detach().clone() for p in model.params()]
    reserve = BinningReserve(DEV)
    step = _Step(model, sc, reserve)
    sg = StepGraph(reserve)
    key = _key(sc, step)
    step.load(far, gt, 0)
    sg.run(key, step, step.params())
    small = (reserve.instances, reserve.longest_list)
    step.load(near, gt, 1)
    loss, radii = sg.run(key, step, step.params())
    torch.cuda.synchronize()
    assert sg.fallbacks == 1 and len(sg) == 0, "the near frame must overflow the far frame's reserve"
    assert reserve.instances > small[0] or reserve.longest_list > small[1]
    _check_step("overflowed step", loss, radii, [p.grad.clone() for p in step.params()], _eager_step(sc, state, near, gt, 1, 2))
    loss, radii = sg.run(key, step, step.params())
    torch.cuda.synchronize()
    assert sg.fallbacks == 1 and sg.captures == 2
    _check_step("recaptured step", loss, radii, [p.grad.clone() for p in step.params()], _eager_step(sc, state, near, gt, 1, 2))


# ---- 5. edge frames ------------------------------------------------------------------------------------------------------

def test_edge_frames():
    import diff_gaussian_rasterization as dgr
    from rade_gs_b200 import rawapi, scenes
    from rade_gs_b200.graphs import BinningReserve
    C = _C()
    sc = scenes.make_scene(5000, 96, 64, 100.0, -3.0, seed=71, bg=(0.3, 0.2, 0.1)).to(DEV)
    c = _call(sc, False, True)
    # P = 0
    empty = scenes.Scene(*[t[:0] for t in (sc.means3D, sc.scales, sc.rotations, sc.opacities, sc.shs)], sc.viewmatrix, sc.projmatrix, sc.campos,
                         sc.bg, sc.width, sc.height, sc.tanfovx, sc.tanfovy)
    ce = _call(empty, False, True)
    status = torch.zeros(4, dtype=torch.int32, device=DEV)
    f = _preset_forward(empty, ce, 65536, 256, status)
    ref = rawapi.forward(C, empty, False, True)
    assert f["num_rendered"] == 65536 and status.tolist() == [0, 0, 0, 0]
    for k in IMAGES + ("radii",):
        _same(f"P=0 {k}", f[k], ref[k])
    # nothing in view: the camera looks away from every splat
    away = scenes.Scene(sc.means3D, sc.scales, sc.rotations, sc.opacities, sc.shs, *_camera(sc, scenes.look_at_view((0.0, 0.0, 0.0), (0.0, 0.0, -5.0))),
                        sc.bg, sc.width, sc.height, sc.tanfovx, sc.tanfovy).to(DEV)
    ref = rawapi.forward(C, away, False, True)
    assert ref["num_rendered"] == 0
    for inst in (0, 65536):
        f = _preset_forward(away, c, inst, 0, status)
        assert status.tolist() == [0, 0, 0, 0]
        _same_forward(f"R=0 ({inst})", f, ref, away, 0)
    # a reserve of 0 grows on the first eager call and gives rgs_forward's frame
    reserve = BinningReserve(DEV)
    means2D = torch.zeros_like(sc.means3D, requires_grad=True)
    out = dgr.GaussianRasterizer(_settings(sc, sc.viewmatrix, sc.projmatrix, sc.campos), reserve)(
        sc.means3D, means2D, sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations)
    ref = rawapi.forward(C, sc, False, True)
    R, L = _totals(ref, sc)
    assert R > 0 and reserve.instances >= R and reserve.longest_list >= L
    for name, a in zip(("color", "radii", "coord", "mcoord", "depth", "mdepth", "alpha", "normal"), out):
        _same(f"grown reserve {name}", a, ref[name])


# ---- 6. stale memory and a late side stream ------------------------------------------------------------------------------

def test_graph_entry_on_stale_memory_and_a_late_side_stream(poisoned_allocator):
    from test_gpu_stale_memory import Case, _step, _upstream, check_case
    from rade_gs_b200 import rawapi, scenes
    C = _C()
    sc = scenes.make_scene(20_000, 200, 136, 200.0, -3.6, seed=81, bg=(0.2, 0.1, 0.0)).to(DEV)
    c = _call(sc, True, True, ks=0.1)
    ref = rawapi.forward(C, sc, True, True, kernel_size=0.1)
    R, L = _totals(ref, sc)

    def run(x):
        sc, g = x["sc"], x["g"]
        f = _preset_forward(sc, c, R + 1000, L + 300, x["status"])
        _step()
        v = rawapi.ours_views(f, sc)
        out = {k: f[k] for k in IMAGES + ("radii", "num_rendered")}
        out.update(point_list=v["point_list"][:R], keys=v["keys"][:R], ranges=v["ranges"], n_contrib=v["n_contrib"], status=x["status"])
        out["acc"] = rawapi.backward_render(C, sc, f, g)
        _step()
        out.update({"bwd." + k: t for k, t in rawapi.backward(C, sc, f, g).items()})
        _step()
        return out

    loose = {"acc": ("acc",), **{"bwd." + k: ("grad", "acc") for k in rawapi.BWD_KEYS}}
    check_case(Case({"sc": sc, "g": _upstream(sc), "status": torch.zeros(4, dtype=torch.int32, device=DEV)}, run, loose), poisoned_allocator)
