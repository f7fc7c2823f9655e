"""`GaussianRasterizer.integrate` at every pixel and every query point against the fp64 model (tests/integrate_f64.py), on scene
families aimed at the kernels' edges (tests/integrate_scenes.py): ragged images, points on pixel / tile / image edges and at the
near plane, degenerate covariances, lists beyond 65 536 entries, the 2048-contributor stop, corner-only entries, crowded pixels.

Per family: channels 0-4, 6, 7 within bound on every pixel (channel 5 exactly 0, channel 8 exactly the points reporting the
pixel); every in-image point's alpha inside its envelope, its SDF within bound and its colour equal to its pixel's; every
culled point exactly (1, 0, 0, -1000); the printed overflow count equal to the model's; identical bits on a second run and
after a permutation of the points.  `-s` prints the worst error/bound ratio per output, the ambiguous fractions and times."""
import time

import numpy as np
import pytest
import torch

import integrate_f64 as mf
import integrate_scenes as isc
from rade_gs_b200 import rawapi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# The ambiguous fraction of pixels / in-image points, measured on an H100 (80 GB HBM3, 700 W power limit): 0.138 / 0.139 for
# C1 (lists up to ~1000 entries keep T next to 1e-4 for hundreds of layers, where the T test is within the fp32 bound),
# 0.225 / 0.206 for the needles and discs, 0.052 / 0.129 for the deep lists; every other family below 0.016.
CEILING = {"generic_C1": 0.2, "degenerate": 0.3, "deep_lists": 0.2}


class _Capture:
    """Stands in for the extension module and keeps the raw 10-tuple of the integrate call (the buffers included)."""

    def __init__(self, C):
        self._C, self.out = C, None

    def __getattr__(self, k):
        return getattr(self._C, k)

    def integrate_gaussians_to_points(self, *a):
        self.out = self._C.integrate_gaussians_to_points(*a)
        return self.out


def _run(case, pts, monkeypatch):
    import diff_gaussian_rasterization as dgr
    sc = case.sc.to(DEV)
    cap = _Capture(dgr._C)
    monkeypatch.setattr(dgr, "_C", cap)
    s = dgr.GaussianRasterizationSettings(image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, kernel_size=0.0,
                                          bg=sc.bg, scale_modifier=1.0, viewmatrix=sc.viewmatrix, projmatrix=sc.projmatrix, sh_degree=case.deg,
                                          campos=sc.campos, prefiltered=False, require_depth=True, require_coord=True, debug=False)
    M = (case.deg + 1) ** 2
    kw = dict(colors_precomp=case.colors_precomp.to(DEV)) if case.colors_precomp is not None else dict(shs=sc.shs[:, :M].contiguous())
    out = dgr.GaussianRasterizer(s).integrate(points3D=pts.to(DEV), means3D=sc.means3D, means2D=None, opacities=sc.opacities, scales=sc.scales,
                                              rotations=sc.rotations, **kw)
    torch.cuda.synchronize()
    monkeypatch.setattr(dgr, "_C", cap._C)
    raw = cap.out
    fwd = dict(num_rendered=raw[0], geom=raw[7], binning=raw[8], img=raw[9], _call=dict(require_coord=False, require_depth=True))
    return out, rawapi.ours_views(fwd, sc), sc


def _overflow(text):
    for line in text.splitlines():
        if "Maximal contributors are met in" in line:
            return int(line.split("met in")[1].split()[0])
    return 0


def _fmt(stats):
    return " ".join(f"{k}={v:.3g}" for k, v in stats.items())


@pytest.mark.parametrize("fam", list(isc.FAMILIES))
def test_integrate_exact(fam, monkeypatch, capfd):
    case = isc.FAMILIES[fam]()
    pts = case.points
    t0 = time.perf_counter()
    out, v, scd = _run(case, pts, monkeypatch)
    t_kernel = time.perf_counter() - t0
    n_over = _overflow(capfd.readouterr().out)
    color, alpha, cint, coord, sdf, radii = out
    st = dict(means2D=v["means2D"], conic_opacity=v["conic_opacity"], rgb=v["rgb"], ts=v["ts"], ray_planes=v["ray_planes"], radii=radii,
              ranges=v["ranges"], point_list=v["point_list"], sigma_inv=v["sigma_inv"])
    it = mf.make_integrate(st, scd.width, scd.height, scd.tanfovx, scd.tanfovy, case.sc.bg.numpy(), case.sc.viewmatrix.numpy(),
                           case.sc.means3D.numpy(), device=DEV)
    inn = ~mf.culled(alpha, cint, coord, sdf)
    t1 = time.perf_counter()
    ref = mf.integrate(it, pts.numpy(), coord.cpu().numpy(), inn)
    t_model = time.perf_counter() - t1
    given = dict(color=color, alpha_integrated=alpha, color_integrated=cint, point_coordinate=coord, point_sdf=sdf, overflow_count=n_over)
    stats = mf.check(ref, given, it, fam)
    with capfd.disabled():
        print(f"\n[{fam}] P={scd.means3D.shape[0]} PN={pts.shape[0]} {scd.width}x{scd.height} in-image={int(inn.sum())} "
              f"longest list={int((v['ranges'][:, 1] - v['ranges'][:, 0]).max())} overflow={n_over}; integrate {t_kernel:.2f}s, model {t_model:.2f}s\n"
              f"[{fam}] {_fmt(stats)}")
    ceil = CEILING.get(fam, mf.AMBIGUOUS_CEILING)
    assert stats["ambiguous_pixels"] <= ceil and stats["ambiguous_points"] <= ceil, f"{fam}: ambiguous fraction above {ceil}"
    assert n_over == ref["overflow_count"] or stats["ambiguous_pixels"] > 0, f"{fam}: {n_over} overflowing pixels, model {ref['overflow_count']}"
    if fam == "overflow":
        assert n_over == scd.width * scd.height
    if fam == "deep_lists":
        n = (v["ranges"][:, 1] - v["ranges"][:, 0]).cpu().numpy()
        assert {255, 256, 8191, 8192} <= set(n.tolist()) and n.max() > 65_536
        assert (v["ranges"][1:, 0].cpu().numpy() % 32 != 0).any()
        assert int(ref["last"].max()) > 65_536, "no contributor past list position 65 536"
    if fam == "degenerate":
        cond = ref["invray"]["condition"].cpu().numpy()
        live = (radii.cpu().numpy() > 0)
        assert (~cond & live).any() and (cond & live).any(), "both condition branches must occur"
    # identical bits: a second run, and a permutation of the points
    out2, _, _ = _run(case, pts, monkeypatch)
    for a, b in zip(out, out2):
        assert torch.equal(a, b), f"{fam}: a second run differs"
    perm = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(5))
    out3, _, _ = _run(case, pts[perm].contiguous(), monkeypatch)
    assert torch.equal(out3[0], out[0])
    pd = perm.to(DEV)
    for k, (a, b) in enumerate(zip(out[1:5], out3[1:5])):
        assert torch.equal(a[pd], b), f"{fam}: output {k + 1} of a point depends on the order of the points"
