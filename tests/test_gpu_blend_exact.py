"""Both blend kernels at every pixel and every accumulator row against the fp64 blend (tests/blend_f64.py), on scene families
aimed at their culling (the forward box test, the backward's cut at the block / warp maximum of last_contributor, the ballot
masks) and list handling (batches of 256, the multi-CTA sort beyond 8192), in all four coord/depth variants.

Forward: exact n_contrib on every unambiguous pixel, every map (and accum_depth, accum_coord, normal_length) within bound.
Backward, fed this build's own forward state: every row and channel of `_C.rasterize_gaussians_backward_render` within bound,
rows that received nothing exactly zero.  `-s` prints the worst error/bound ratio per map and channel and the ambiguous fraction."""
import numpy as np
import pytest
import torch

import blend_f64 as bf
import blend_scenes as bs
from rade_gs_b200 import rawapi, scenes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VARIANTS = [(False, False), (False, True), (True, False), (True, True)]

FAMILIES = {
    "needles_ks0": (lambda: bs.needles(320, 240, 400), 0.0),
    "needles_ks01": (lambda: bs.needles(320, 240, 400, seed=12), 0.1),
    "huge_near": (lambda: bs.huge_near(200, 150, 200), 0.0),
    "deep_low": (lambda: bs.deep([255, 256, 257, 511, 512, 513, 8191, 8192, 8193, 20000]), 0.0),
    "deep_opaque": (lambda: bs.deep([255, 256, 257, 511, 512, 513, 8191, 8192, 8193], opaque=True, seed=13), 0.0),
    "opaque": (lambda: bs.opaque(200, 150, 3000), 0.0),
    "faint": (lambda: bs.faint(200, 150, 4000), 0.0),
    "frustum_edge": (lambda: bs.frustum_edge(200, 150, 300), 0.1),
    "tiny_1x1": (lambda: bs.tiny(1, 1, 31), 0.0),
    "tiny_7x5": (lambda: bs.tiny(7, 5, 33), 0.0),
    "tiny_17x16": (lambda: bs.tiny(17, 16, 1), 0.0),
    "tiny_16x17": (lambda: bs.tiny(16, 17, 33), 0.0),
    "tiny_1000x3": (lambda: bs.tiny(1000, 3, 31), 0.0),
    "C1": (lambda: scenes.make_config("C1")[0], 0.0),
}


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _run(sc, coord, depth, ks, name):
    C = _C()
    scd = sc.to(DEV)
    grads = {k: v.to(DEV) for k, v in scenes.make_upstream_grads(sc.height, sc.width, seed=17).items()}
    f = rawapi.forward(C, scd, coord, depth, kernel_size=ks)
    v = rawapi.ours_views(f, scd)
    st = dict(means2D=v["means2D"], conic_opacity=v["conic_opacity"], rgb=v["rgb"], ts=v["ts"], ray_planes=v["ray_planes"], normals=v["normals"],
              camera_planes=v["camera_planes"], view_points=v["view_points"], ranges=v["ranges"], point_list=v["point_list"])
    bl = bf.make_blend(st, sc.width, sc.height, sc.tanfovx, sc.tanfovy, sc.bg.numpy(), coord, depth, device=DEV)
    ref = bf.forward(bl)
    given = {k: f[k] for k in ("color", "alpha", "depth", "mdepth", "normal", "coord", "mcoord")}
    given["n_contrib"] = v["n_contrib"]
    for k in ("accum_depth", "accum_coord", "normal_length"):
        if v[k] is not None:
            given[k] = v[k]
    fstats = bf.check_forward(ref, given, bl, name, hitmask=v["hitmask"].cpu(), chunk_base=v["chunk_base"].cpu())

    E = torch.Tensor([])
    grid_y = (sc.height + 15) // 16
    acc = C.rasterize_gaussians_backward_render(scd.bg, scd.means3D, f["radii"], E, scd.scales, scd.rotations, 1.0, E, scd.viewmatrix, scd.projmatrix,
                                                scd.tanfovx, scd.tanfovy, ks, grads["color"], grads["coord"], grads["mcoord"], grads["depth"],
                                                grads["mdepth"], grads["alpha"], grads["normal"], f["normal"], scd.shs, 3, scd.campos, f["geom"],
                                                f["num_rendered"], f["binning"], f["img"], f["alpha"], coord, depth, False, 0, grid_y)
    torch.cuda.synchronize()
    state = dict(alpha=f["alpha"], n_contrib=v["n_contrib"], normal=f["normal"], accum_depth=v["accum_depth"], accum_coord=v["accum_coord"],
                 normal_length=v["normal_length"])
    state = {k: (val if val is not None else torch.zeros(1)) for k, val in state.items()}
    rb = bf.backward(bl, state, grads)
    bstats = bf.check_backward(rb, bf.accumulator_to_sg(acc, bl), name)
    return v, fstats, bstats


def _fmt(stats):
    return " ".join(f"{k}={v:.3g}" for k, v in stats.items() if v)


@pytest.mark.parametrize("coord,depth", VARIANTS, ids=["none", "depth", "coord", "both"])
@pytest.mark.parametrize("fam", list(FAMILIES))
def test_blend_kernels_exact(fam, coord, depth):
    make, ks = FAMILIES[fam]
    sc = make()
    name = f"{fam}/{'coord' if coord else ''}{'depth' if depth else ''}{'' if coord or depth else 'none'}"
    v, fs, bs_ = _run(sc, coord, depth, ks, name)
    print(f"\n[{name}] forward: {_fmt(fs)}\n[{name}] backward: {_fmt(bs_)}")
    assert fs["ambiguous_frac"] <= bf.AMBIGUOUS_CEILING, f"{name}: {fs['ambiguous_frac']:.3e} of the pixels are ambiguous"
    if fam.startswith("deep"):
        n = (v["ranges"][:, 1] - v["ranges"][:, 0]).cpu().numpy()
        assert sorted(n[n > 0].tolist()) == sorted([255, 256, 257, 511, 512, 513, 8191, 8192, 8193] + ([20000] if fam == "deep_low" else []))
