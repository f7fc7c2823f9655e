"""Parity of the CUDA path (through `diff_gaussian_rasterization._C`, i.e. through the C ABI) on a real GPU:
  * against the golden fixtures produced by the unmodified reference build,
  * against the CPU oracle on fresh seeded scenes,
  * against what the reference build computed at BASELINE.json's full sizes (digests and samples, tools/gen_golden_refbuild.py),
  * and, at BASELINE.json's full sizes, through size-independent properties.
Integer work (radii, keys, sort order, ranges, n_contrib) is compared bit-exactly; floats per tests/tolerances.py."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, ROOT, golden_oracle_inputs, golden_upstream, load_golden
from tolerances import grad_close_vs_reference_runs, IMG_OUTLIER_FRAC_CPU, IMG_OUTLIER_FRAC_GPU, grad_close_cpu, grad_close_gpu, image_close

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT, "tools"))   # gen_golden_refbuild: the digests the reference-build fixtures store
DEV = "cuda:0"
IMG_KEYS = ("color", "alpha", "depth", "mdepth", "normal", "coord", "mcoord")
GRAD_KEYS = ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations")


def _C():
    import diff_gaussian_rasterization as dgr
    return dgr._C


def _scene_from_golden(d):
    from rade_gs_b200 import scenes
    t = lambda k: torch.from_numpy(d[k]).to(DEV)
    sc = scenes.Scene(t("in_means3D"), t("in_scales"), t("in_rotations"), t("in_opacities"), t("in_shs"), t("in_viewmatrix"), t("in_projmatrix"),
                      t("in_campos"), t("in_bg"), int(d["meta_W"]), int(d["meta_H"]), float(d["in_tanfov"][0]), float(d["in_tanfov"][1]))
    extra = {}
    if "in_colors_precomp" in d:
        extra["colors_precomp"] = t("in_colors_precomp")
    if "in_cov3D_precomp" in d:
        extra["cov3D_precomp"] = t("in_cov3D_precomp")
    return sc, extra


def _run_golden(d):
    from rade_gs_b200 import rawapi
    sc, extra = _scene_from_golden(d)
    f = rawapi.forward(_C(), sc, bool(d["meta_coord"]), bool(d["meta_depth"]), kernel_size=float(d["meta_ks"]), sh_degree=int(d["meta_deg"]), **extra)
    grads = {k: torch.from_numpy(v).to(DEV) for k, v in golden_upstream(d).items()}
    b = rawapi.backward(_C(), sc, f, grads)
    torch.cuda.synchronize()
    return sc, f, b


def test_golden_integer_contract(golden):
    from rade_gs_b200 import rawapi
    name, d = golden
    sc, f, _ = _run_golden(d)
    v = rawapi.ours_views(f, sc)
    assert f["num_rendered"] == int(d["num_rendered"])
    assert np.array_equal(f["radii"].cpu().numpy(), d["out_radii"])
    vis = d["out_radii"] > 0
    assert np.array_equal(v["tiles_touched"].cpu().numpy(), d["st_tiles_touched"])
    assert np.array_equal(v["depths"].cpu().numpy()[vis].view(np.int32), d["st_depths"][vis].view(np.int32))
    assert np.array_equal(v["means2D"].cpu().numpy()[vis].view(np.int32), d["st_means2D"][vis].view(np.int32))
    assert np.array_equal(v["point_list"].cpu().numpy(), d["st_point_list"])
    assert np.array_equal(v["keys"].cpu().numpy(), d["st_keys"])
    assert np.array_equal(v["ranges"].cpu().numpy(), d["st_ranges"])
    assert np.array_equal(v["n_contrib"].cpu().numpy(), d["st_n_contrib"])


def test_golden_images_and_gradients(golden):
    name, d = golden
    sc, f, b = _run_golden(d)
    for k in IMG_KEYS:
        image_close(f[k].cpu().numpy(), d["out_" + k], IMG_OUTLIER_FRAC_GPU, f"{name}/{k}")
    for k in GRAD_KEYS:
        # the fixture stores the mean of two reference runs and their spread (float atomics): allow that spread too
        noise = float(d["grad_noise_" + k]) / (np.abs(d["grad_" + k]).max() + 1e-30) if d["grad_" + k].size else 0.0
        grad_close_gpu(b[k].cpu().numpy(), d["grad_" + k], f"{name}/{k}", rel=1e-3 + 4 * noise, elem=1e-3 + 4 * noise)


@pytest.mark.parametrize("seed,coord,depth,ks,deg", [(101, False, True, 0.0, 3), (102, True, True, 0.1, 2), (103, True, False, 0.0, 3), (104, False, False, 0.3, 0)])
def test_against_oracle_fresh_scene(seed, coord, depth, ks, deg):
    """Same seeded inputs through the CUDA path and through the CPU oracle."""
    import oracle
    from rade_gs_b200 import rawapi, scenes
    sc = scenes.make_scene(3000, 150, 100, 110.0, -2.6, seed=seed, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.3, 0.1, 0.2))
    grads = scenes.make_upstream_grads(sc.height, sc.width, seed=seed + 1)
    inp = oracle.Inputs(sc.means3D.numpy(), sc.opacities.numpy(), sc.viewmatrix.numpy(), sc.projmatrix.numpy(), sc.campos.numpy(), sc.bg.numpy(),
                        sc.width, sc.height, sc.tanfovx, sc.tanfovy, shs=sc.shs.numpy(), scales=sc.scales.numpy(), rotations=sc.rotations.numpy(),
                        sh_degree=deg, kernel_size=ks, require_coord=coord, require_depth=depth)
    fo = oracle.forward(inp)
    bo = oracle.backward(inp, fo, {k: v.numpy() for k, v in grads.items()})
    scd = sc.to(DEV)
    f = rawapi.forward(_C(), scd, coord, depth, kernel_size=ks, sh_degree=deg)
    b = rawapi.backward(_C(), scd, f, {k: v.to(DEV) for k, v in grads.items()})
    v = rawapi.ours_views(f, scd)
    assert np.array_equal(f["radii"].cpu().numpy(), fo["radii"])
    assert f["num_rendered"] == fo["num_rendered"]
    assert np.array_equal(v["point_list"].cpu().numpy().astype(np.uint32), fo["binning"]["point_list"])
    assert np.array_equal(v["keys"].cpu().numpy().astype(np.uint64), fo["binning"]["keys"])
    assert np.array_equal(v["ranges"].cpu().numpy().astype(np.uint32), fo["binning"]["ranges"])
    nc = v["n_contrib"].cpu().numpy().astype(np.uint32) != fo["image"]["n_contrib"]
    assert nc.mean() < 1e-3  # exp / FMA last-bit differences can flip a 1/255 or 1e-4 threshold on isolated pixels
    for k in IMG_KEYS:
        image_close(f[k].cpu().numpy(), fo[k], IMG_OUTLIER_FRAC_CPU, k)
    for k in GRAD_KEYS:
        grad_close_cpu(b[k].cpu().numpy(), bo[k], k)


@pytest.mark.parametrize("cfg,ks", [("C1", 0.0), ("C1", 0.1), ("C2", 0.0), ("C3", 0.0), ("C4", 0.0)])
def test_against_reference_build(cfg, ks):
    """BASELINE configs C1 (300k, 800x800), C2 (1M, 1600x1200, headline), C3 (3M, 1920x1080, coordinate map) and C4 (10M,
    4096x4096) against what the reference's own CUDA build computed on identical inputs: every integer quantity bit-exact
    (digests of the whole arrays), images within the stated tolerance and n_contrib equal at the stored pixels, every gradient
    tensor within 1e-3 relative L2 on the stored sample of rows the reference itself determines (its atomics make two of ITS runs differ;
    see tolerances.grad_close_vs_reference_runs)."""
    from gen_golden_refbuild import digest, scene_digest
    from rade_gs_b200 import rawapi, scenes
    d = load_golden(f"refbuild_{cfg}_ks{str(ks).replace('.', '')}")
    sc, coord, depth = scenes.make_config(cfg)
    grads = scenes.make_upstream_grads(sc.height, sc.width)
    assert scene_digest(sc, grads) == str(d["in_digest"]), "the synthetic inputs differ from the ones the fixture was made from"
    sc = sc.to(DEV)
    grads = {k: v.to(DEV) for k, v in grads.items()}
    fo = rawapi.forward(_C(), sc, coord, depth, kernel_size=ks)
    vo = rawapi.ours_views(fo, sc)
    assert fo["num_rendered"] == int(d["num_rendered"])
    assert digest(fo["radii"]) == str(d["sha_radii"])
    for k in ("point_list", "keys", "ranges"):
        assert digest(vo[k]) == str(d["sha_" + k]), k
    pix = torch.from_numpy(d["pix"]).to(DEV)
    assert (vo["n_contrib"].reshape(2, -1)[:, pix].cpu().numpy() != d["n_contrib"]).mean() < 1e-5
    for k in IMG_KEYS:
        image_close(fo[k].reshape(fo[k].shape[0], -1)[:, pix].cpu().numpy(), d["img_" + k], IMG_OUTLIER_FRAC_GPU, k)
    del vo
    bo = rawapi.backward(_C(), sc, fo, grads)
    rows = torch.from_numpy(d["rows"]).to(DEV)
    failures = []
    for k in GRAD_KEYS:
        try:
            grad_close_vs_reference_runs(bo[k][rows].cpu().numpy(), d["grad1_" + k], d["grad2_" + k], k, ill_frac=float(d["ill_frac_" + k]),
                                         scale=float(d["scale_" + k]))
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, failures


# ---- size-independent properties at the headline size (1M splats, 1600x1200) -----------------------------------------

@pytest.fixture(scope="module")
def c2():
    from rade_gs_b200 import rawapi, scenes
    sc, coord, depth = scenes.make_config("C2")
    sc = sc.to(DEV)
    f = rawapi.forward(_C(), sc, coord, depth)
    return sc, coord, depth, f


def test_c2_binning_invariants(c2):
    from rade_gs_b200 import rawapi
    sc, coord, depth, f = c2
    v = rawapi.ours_views(f, sc)
    R = f["num_rendered"]
    keys = v["keys"]
    assert R == int(v["tiles_touched"].long().sum().item())                      # every instance accounted for
    assert bool((keys[1:] >= keys[:-1]).all())                                    # sortedness
    tile_of = (keys >> 32).int()
    rg = v["ranges"].long()
    nonempty = rg[:, 1] > rg[:, 0]
    assert int((rg[:, 1] - rg[:, 0]).sum().item()) == R                           # ranges partition the list
    starts = rg[nonempty, 0]
    assert bool((tile_of[starts] == torch.nonzero(nonempty).squeeze(1).int()).all())
    # stable tie-break: equal keys keep ascending Gaussian index
    same = keys[1:] == keys[:-1]
    assert bool((v["point_list"][1:][same] > v["point_list"][:-1][same]).all())
    # depth bits of every key are its Gaussian's view-space z
    ids = v["point_list"].long()
    assert bool(((keys & 0xFFFFFFFF).int() == v["depths"][ids].view(torch.int32)).all())
    assert bool((f["radii"][ids] > 0).all())


def test_c2_image_invariants(c2):
    sc, coord, depth, f = c2
    a = f["alpha"]
    assert torch.isfinite(f["color"]).all() and torch.isfinite(f["depth"]).all() and torch.isfinite(f["normal"]).all()
    assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0 + 1e-5
    n = f["normal"].norm(dim=0)
    covered = a[0] > 0
    assert bool(((n[covered] - 1).abs() < 1e-3).all()) and bool((n[~covered] == 0).all())  # unit normals where anything was blended
    assert bool((f["coord"] == 0).all()) and bool((f["mcoord"] == 0).all())                 # coord variant off -> zero-filled maps


def test_c2_backward_is_linear_in_upstream_gradients(c2):
    from rade_gs_b200 import rawapi, scenes
    sc, coord, depth, f = c2
    g1 = scenes.make_upstream_grads(sc.height, sc.width, seed=7, device=DEV)
    g2 = {k: 2.0 * v for k, v in g1.items()}
    b1, b2 = rawapi.backward(_C(), sc, f, g1), rawapi.backward(_C(), sc, f, g2)
    for k in ("colors", "sh", "means2D", "opacity"):  # purely linear outputs (kernel_size = 0)
        if k == "means2D":
            a, b = b1[k][:, :2], b2[k][:, :2]
        else:
            a, b = b1[k], b2[k]
        err = (2 * a - b).abs().max().item()
        assert err <= 2e-4 * b.abs().max().item() + 1e-6, (k, err)
    inv = f["radii"] <= 0
    for k in GRAD_KEYS:
        assert not bool(b1[k][inv].any()), k  # nothing flows to Gaussians that were not rendered


def test_c2_slabs_compose_to_the_whole(c2):
    """Tile-row sharding (multi-GPU path) on one GPU: two slabs reproduce the whole image bit-for-bit, their sorted
    lists concatenate to the whole list, and the summed gradient accumulators give the same parameter gradients."""
    from rade_gs_b200 import scenes
    C = _C()
    sc, coord, depth, f = c2
    grid_y = (sc.height + 15) // 16
    cut = grid_y // 2
    args = (sc.bg, sc.means3D, torch.Tensor([]), sc.opacities, sc.scales, sc.rotations, 1.0, torch.Tensor([]), sc.viewmatrix, sc.projmatrix,
            sc.tanfovx, sc.tanfovy, 0.0, sc.height, sc.width, sc.shs, 3, sc.campos, False, coord, depth, False)
    s0 = C.rasterize_gaussians_slab(*args, 0, cut)
    s1 = C.rasterize_gaussians_slab(*args, cut, grid_y)
    assert s0[0] + s1[0] == f["num_rendered"]
    assert torch.equal(s0[8], f["radii"]) and torch.equal(s1[8], f["radii"])
    rows = cut * 16
    for idx, k in ((1, "color"), (4, "alpha"), (5, "normal"), (6, "depth"), (7, "mdepth")):
        assert torch.equal(s0[idx][:, :rows], f[k][:, :rows]), k
        assert torch.equal(s1[idx][:, rows:], f[k][:, rows:]), k
        assert not bool(s0[idx][:, rows:].any())
    whole_list = f["binning"][: 4 * f["num_rendered"]].view(torch.int32)
    l0 = s0[10][: 4 * s0[0]].view(torch.int32)
    l1 = s1[10][: 4 * s1[0]].view(torch.int32)
    assert torch.equal(torch.cat([l0, l1]), whole_list)
    g = scenes.make_upstream_grads(sc.height, sc.width, seed=9, device=DEV)
    E = torch.Tensor([])

    def stage1(s, b, e):
        return C.rasterize_gaussians_backward_render(sc.bg, sc.means3D, s[8], E, sc.scales, sc.rotations, 1.0, E, sc.viewmatrix, sc.projmatrix,
                                                     sc.tanfovx, sc.tanfovy, 0.0, g["color"], g["coord"], g["mcoord"], g["depth"], g["mdepth"],
                                                     g["alpha"], g["normal"], s[5], sc.shs, 3, sc.campos, s[9], s[0], s[10], s[11], s[4],
                                                     coord, depth, False, b, e)
    acc = stage1(s0, 0, cut) + stage1(s1, cut, grid_y)
    out = C.rasterize_gaussians_backward_preprocess(acc, sc.bg, sc.means3D, f["radii"], E, sc.opacities, sc.scales, sc.rotations, 1.0, E,
                                                    sc.viewmatrix, sc.projmatrix, sc.tanfovx, sc.tanfovy, 0.0, sc.height, sc.width, sc.shs, 3,
                                                    sc.campos, s0[9], coord, depth, False)
    from rade_gs_b200 import rawapi
    whole = rawapi.backward(C, sc, f, g)
    for k, o in zip(GRAD_KEYS, out):
        # float-atomic summation order differs between the two paths; at 1M splats a handful of ill-conditioned splats
        # amplify that to ~2e-3 of the tensor maximum (the reference's own run-to-run spread is 1.6e-3 here)
        grad_close_gpu(o.cpu().numpy(), whole[k].cpu().numpy(), k, rel=1e-3, elem=1e-2)


def _oracle_inputs(sc, coord, depth, ks, deg, shs=None):
    import oracle
    return oracle.Inputs(sc.means3D.numpy(), sc.opacities.numpy(), sc.viewmatrix.numpy(), sc.projmatrix.numpy(), sc.campos.numpy(), sc.bg.numpy(),
                         sc.width, sc.height, sc.tanfovx, sc.tanfovy, shs=(sc.shs if shs is None else shs).numpy(), scales=sc.scales.numpy(),
                         rotations=sc.rotations.numpy(), sh_degree=deg, kernel_size=ks, require_coord=coord, require_depth=depth)


@pytest.mark.parametrize("n_splats", [12000, 20000, 70000])
def test_long_tile_lists_take_the_multi_cta_sort(n_splats):
    """Tile lists longer than the one-CTA shared-memory sort (8192) are split over several CTAs (chunk sort + global merge
    passes; 2, 3 and 5 passes here, so both ping-pong parities) and must still give the reference order: splats piled onto a
    few pixels.  No library sort is involved (the global radix path only runs when RGS_BINNING=radix asks for it)."""
    import oracle
    from rade_gs_b200 import rawapi, scenes
    sc = scenes.make_scene(n_splats, 64, 48, 200.0, -4.0, seed=31)
    sc.means3D[:, 0] = 0.02 * torch.randn(n_splats, generator=torch.Generator().manual_seed(1))
    sc.means3D[:, 1] = 0.02 * torch.randn(n_splats, generator=torch.Generator().manual_seed(2))
    sc.opacities[:] = 0.02 * 12000 / n_splats  # keep transmittance alive so the whole list matters
    grads = scenes.make_upstream_grads(sc.height, sc.width, seed=32)
    fo = oracle.forward(_oracle_inputs(sc, False, True, 0.0, 3))
    scd = sc.to(DEV)
    n0 = _C().launch_count()
    f = rawapi.forward(_C(), scd, False, True)
    launches = _C().launch_count() - n0
    v = rawapi.ours_views(f, scd)
    longest = int(v["totals"][1])
    assert longest > 8192, "scene did not produce a long tile list"
    passes = int(np.ceil(np.log2(np.ceil(longest / 4096))))
    assert launches == 5 + 2 + passes, (launches, passes)   # preprocess, scan, scatter, tile sort, render + chunk sort, finalize + merge passes
    assert f["num_rendered"] == fo["num_rendered"]
    assert np.array_equal(v["point_list"].cpu().numpy().astype(np.uint32), fo["binning"]["point_list"])
    assert np.array_equal(v["ranges"].cpu().numpy().astype(np.uint32), fo["binning"]["ranges"])
    keys = v["keys"]
    assert bool((keys[1:] >= keys[:-1]).all())
    if n_splats > 12000:
        return
    for k in ("color", "alpha", "depth", "normal"):
        image_close(f[k].cpu().numpy(), fo[k], IMG_OUTLIER_FRAC_CPU, k)
    b = rawapi.backward(_C(), scd, f, {k: v_.to(DEV) for k, v_ in grads.items()})
    bo = oracle.backward(_oracle_inputs(sc, False, True, 0.0, 3), fo, {k: v_.numpy() for k, v_ in grads.items()})
    for k in ("means3D", "sh", "opacity", "scales"):
        grad_close_cpu(b[k].cpu().numpy(), bo[k], k)


def _long_tile_scene():
    """C1-sized scene (300k splats, 800x800) plus 12k small splats piled onto one spot."""
    from rade_gs_b200 import scenes
    sc, coord, depth = scenes.make_config("C1")
    g = torch.Generator().manual_seed(9)
    n_extra = 12000
    pile = scenes.make_scene(n_extra, sc.width, sc.height, 1100.0, -6.0, seed=77)
    pile.means3D[:, 0] = 0.5 + 0.004 * torch.randn(n_extra, generator=g)
    pile.means3D[:, 1] = -0.3 + 0.004 * torch.randn(n_extra, generator=g)
    pile.means3D[:, 2] = 4.0 + 0.5 * torch.rand(n_extra, generator=g)
    pile.opacities[:] = 0.01
    both = scenes.Scene(*[torch.cat([getattr(sc, k), getattr(pile, k)]) for k in ("means3D", "scales", "rotations", "opacities", "shs")],
                        sc.viewmatrix, sc.projmatrix, sc.campos, sc.bg, sc.width, sc.height, sc.tanfovx, sc.tanfovy)
    return sc, both, coord, depth


def test_one_long_tile_inside_a_large_scene_leaves_the_other_tiles_alone():
    """C1-sized scene plus 12k small splats piled onto one spot: only the tiles under the pile take the multi-CTA sort; every
    other tile's list and the images away from the pile agree, and the whole result agrees with the reference build's."""
    from gen_golden_refbuild import digest, scene_digest
    from rade_gs_b200 import rawapi
    sc, both, coord, depth = _long_tile_scene()
    d = load_golden("refbuild_long_tile")
    assert scene_digest(both) == str(d["in_digest"]), "the synthetic inputs differ from the ones the fixture was made from"
    base, big = sc.to(DEV), both.to(DEV)
    f0, f1 = rawapi.forward(_C(), base, coord, depth), rawapi.forward(_C(), big, coord, depth)
    v0, v1 = rawapi.ours_views(f0, base), rawapi.ours_views(f1, big)
    assert int(v0["totals"][1]) <= 8192 < int(v1["totals"][1])
    r0, r1 = v0["ranges"].long(), v1["ranges"].long()
    n0, n1 = r0[:, 1] - r0[:, 0], r1[:, 1] - r1[:, 0]
    same = torch.nonzero(n0 == n1).squeeze(1)
    assert same.numel() > 0.95 * n0.numel() and int((n1 > 8192).sum()) >= 1
    # tiles the pile does not reach: identical sorted id lists (pile ids are >= P0, so equality of the lists says none leaked in)
    pl0, pl1 = v0["point_list"].long(), v1["point_list"].long()
    for t in same[torch.linspace(0, same.numel() - 1, 400).long()].tolist():
        assert torch.equal(pl0[r0[t, 0]:r0[t, 1]], pl1[r1[t, 0]:r1[t, 1]]), t
    keys = v1["keys"]
    assert bool((keys[1:] >= keys[:-1]).all())
    tile_of = (keys >> 32).long()
    assert bool((tile_of[r1[:, 0][n1 > 0]] == torch.nonzero(n1 > 0).squeeze(1)).all())
    for k in ("point_list", "keys", "ranges"):
        assert digest(v1[k]) == str(d["sha_" + k]), k
    pix = torch.from_numpy(d["pix"]).to(DEV)
    for k in IMG_KEYS:
        image_close(f1[k].reshape(f1[k].shape[0], -1)[:, pix].cpu().numpy(), d["img_" + k], IMG_OUTLIER_FRAC_GPU, k)


@pytest.mark.parametrize("M,deg,W,H", [(1, 0, 70, 50), (4, 1, 33, 17), (9, 2, 96, 64)])
def test_sh_storage_sizes_and_ragged_images(M, deg, W, H):
    """SH tensors with fewer stored coefficients ([P,1,3], [P,4,3], [P,9,3]: rows of 12/48/108 bytes, the last two not
    16-byte multiples of the row index) and image sizes that are not multiples of the 16x16 tile."""
    import oracle
    from rade_gs_b200 import rawapi, scenes
    sc = scenes.make_scene(2500, W, H, 0.9 * W, -2.4, seed=40 + M, view=scenes.look_at_view((0.2, 0.1, -0.3), (0.0, 0.0, 6.0)), bg=(0.05, 0.1, 0.2))
    shs = sc.shs[:, :M].contiguous()
    grads = scenes.make_upstream_grads(H, W, seed=50 + M)
    inp = _oracle_inputs(sc, True, True, 0.1, deg, shs=shs)
    fo = oracle.forward(inp)
    bo = oracle.backward(inp, fo, {k: v.numpy() for k, v in grads.items()})
    scd = sc.to(DEV)
    scd.shs = shs.to(DEV)
    f = rawapi.forward(_C(), scd, True, True, kernel_size=0.1, sh_degree=deg)
    b = rawapi.backward(_C(), scd, f, {k: v.to(DEV) for k, v in grads.items()})
    v = rawapi.ours_views(f, scd)
    assert f["num_rendered"] == fo["num_rendered"] and np.array_equal(f["radii"].cpu().numpy(), fo["radii"])
    assert np.array_equal(v["point_list"].cpu().numpy().astype(np.uint32), fo["binning"]["point_list"])
    assert b["sh"].shape == (2500, M, 3)
    for k in IMG_KEYS:
        image_close(f[k].cpu().numpy(), fo[k], IMG_OUTLIER_FRAC_CPU, k)
    for k in GRAD_KEYS:
        grad_close_cpu(b[k].cpu().numpy(), bo[k], k)
