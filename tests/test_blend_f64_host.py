"""The fp64 blend checker (tests/blend_f64.py) validated without a GPU: the reference build's own golden state and the CPU oracle
pass it at every pixel and every row, its screen-space rows reproduce the goldens' parameter gradients, and defects planted
into the oracle's results are caught and located."""
import numpy as np
import pytest
import torch

import blend_f64 as bf
import blend_scenes as bs
import oracle
from conftest import GOLDEN_CASES, golden_oracle_inputs, golden_upstream, load_golden
from rade_gs_b200 import scenes
from tolerances import grad_close_gpu

MAPS = ("color", "alpha", "depth", "mdepth", "normal", "coord", "mcoord")
STATE = ("alpha", "n_contrib", "normal", "accum_depth", "accum_coord", "normal_length")


def _golden_blend(d):
    """The reference build's own per-Gaussian state (`st_*`); with precomputed colours it leaves rgb unwritten and blends
    `in_colors_precomp`."""
    st = {k[3:]: d[k] for k in d if k.startswith("st_")}
    if "in_colors_precomp" in d:
        st["rgb"] = d["in_colors_precomp"]
    return bf.make_blend(st, d["meta_W"], d["meta_H"], d["in_tanfov"][0], d["in_tanfov"][1], d["in_bg"], bool(d["meta_coord"]),
                         bool(d["meta_depth"]))


def _oracle_blend(inp, fo, colors_precomp=None):
    st = dict(fo["geom"], ranges=fo["binning"]["ranges"], point_list=fo["binning"]["point_list"].astype(np.int64))
    if colors_precomp is not None:
        st["rgb"] = colors_precomp
    return bf.make_blend(st, inp.W, inp.H, inp.tanfovx, inp.tanfovy, inp.bg, inp.require_coord, inp.require_depth)


def _oracle_given(inp, fo):
    img = fo["image"]
    keep = set(MAPS) | {"n_contrib"}
    keep |= {"accum_depth"} if inp.require_depth else set()
    keep |= {"accum_coord"} if inp.require_coord else set()
    keep |= {"normal_length"} if (inp.require_coord or inp.require_depth) else set()
    return {k: img[k] for k in keep}


def _scene_inputs(sc, coord, depth, ks):
    return oracle.Inputs(sc.means3D.numpy(), sc.opacities.numpy(), sc.viewmatrix.numpy(), sc.projmatrix.numpy(), sc.campos.numpy(),
                         sc.bg.numpy(), sc.width, sc.height, sc.tanfovx, sc.tanfovy, shs=sc.shs.numpy(), scales=sc.scales.numpy(),
                         rotations=sc.rotations.numpy(), sh_degree=3, kernel_size=ks, require_coord=coord, require_depth=depth)


def _oracle_roundtrip(inp, up, name, colors_precomp=None):
    """Oracle forward and backward (fed the oracle's own pixel state) against the fp64 blend; returns the pieces."""
    fo = oracle.forward(inp)
    bl = _oracle_blend(inp, fo, colors_precomp)
    ref = bf.forward(bl)
    bf.check_forward(ref, _oracle_given(inp, fo), bl, name)
    sg = oracle.render_backward(inp, fo, up)
    state = {k: fo["image"][k] for k in STATE}
    rb = bf.backward(bl, state, up)
    bf.check_backward(rb, sg, name)
    return fo, bl, ref, sg, rb


def test_reference_build_golden_state_passes(golden):
    """The unmodified reference build's maps and n_contrib against the fp64 blend of its own state: exact n_contrib on every
    unambiguous pixel, every map within bound."""
    name, d = golden
    bl = _golden_blend(d)
    ref = bf.forward(bl)
    given = {k: d["out_" + k] for k in MAPS}
    given["n_contrib"] = d["st_n_contrib"]
    stats = bf.check_forward(ref, given, bl, name)
    assert stats["ambiguous_frac"] <= bf.AMBIGUOUS_CEILING


def test_oracle_passes_on_goldens(golden):
    name, d = golden
    inp = golden_oracle_inputs(d)
    _oracle_roundtrip(inp, golden_upstream(d), name, d.get("in_colors_precomp"))


FAMILIES = {
    "needles_ks0": (lambda: bs.needles(64, 48, 40), False, True, 0.0),
    "needles_ks01": (lambda: bs.needles(64, 48, 40, seed=11), True, True, 0.1),
    "huge_near": (lambda: bs.huge_near(64, 48, 30), True, False, 0.0),
    "deep_low": (lambda: bs.deep([255, 256, 257]), False, True, 0.0),
    "deep_opaque": (lambda: bs.deep([256, 257, 300], opaque=True), True, True, 0.0),
    "opaque": (lambda: bs.opaque(48, 32, 150), True, True, 0.0),
    "faint": (lambda: bs.faint(48, 32, 200), False, False, 0.0),
    "frustum_edge": (lambda: bs.frustum_edge(64, 48, 40), False, True, 0.1),
    "tiny_7x5": (lambda: bs.tiny(7, 5, 33), True, True, 0.0),
    "tiny_1x1": (lambda: bs.tiny(1, 1, 31), False, True, 0.0),
}


@pytest.mark.parametrize("fam", sorted(FAMILIES))
def test_oracle_passes_on_fresh_families(fam):
    make, coord, depth, ks = FAMILIES[fam]
    sc = make()
    up = {k: v.numpy() for k, v in scenes.make_upstream_grads(sc.height, sc.width, seed=5).items()}
    fo, _, ref, _, _ = _oracle_roundtrip(_scene_inputs(sc, coord, depth, ks), up, fam)
    assert int(ref["n_contrib"][0].max()) > 0, "the scene blends nothing"


def test_fp64_rows_reproduce_golden_parameter_gradients(golden):
    """Units and semantics close the loop: fp64 screen-space rows (pixel state from the fp64 forward of the reference's state) through
    the oracle's backward preprocess give the golden parameter gradients within the GPU bar (1e-3 + 4x the reference's own spread).
    Rows of Gaussians whose preprocess state the CPU oracle does not reproduce (the fixtures' hand-placed degenerate splat: its
    conic differs beyond 1e-3, as test_oracle_golden.test_preprocess_state allows) are left out: that chain is not the blend."""
    name, d = golden
    bl = _golden_blend(d)
    r = bf.forward(bl)
    state = {k: r[k].numpy().astype(np.float32) for k in ("alpha", "normal", "accum_depth", "accum_coord", "normal_length")}
    state["n_contrib"] = r["n_contrib"].numpy().astype(np.uint32)
    rb = bf.backward(bl, state, golden_upstream(d))
    sg = {k: np.ascontiguousarray(rb[k].numpy().reshape(-1) if bf.SG_WIDTH[k] == 1 else rb[k].numpy()) for k in bf.SG_KEYS}
    inp = golden_oracle_inputs(d)
    g = oracle.preprocess(inp)
    vis = d["out_radii"] > 0
    same = ~((np.abs(g["conic_opacity"] - d["st_conic_opacity"]) > 1e-3 * (1 + np.abs(d["st_conic_opacity"]))).any(1) & vis)
    assert (~same).sum() <= 1
    geo = dict(g, radii=d["out_radii"])
    for k in ("cov3D", "clamped", "conic_opacity"):
        if not (k == "clamped" and "in_colors_precomp" in d) and not (k == "cov3D" and "in_cov3D_precomp" in d):
            geo[k] = np.ascontiguousarray(d["st_" + k])
    out = oracle.preprocess_backward(inp, {"geom": geo}, sg)
    for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations"):
        ref = d["grad_" + k]
        noise = float(d["grad_noise_" + k]) / (np.abs(ref).max() + 1e-30) if ref.size else 0.0
        grad_close_gpu(out[k][same], ref[same], f"{name}/{k}", rel=1e-3 + 4 * noise, elem=1e-3 + 4 * noise)


# ---- planted defects -------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def planted():
    """A small scene with opaque stacks (clamped alpha) and both geometry variants on (median terms), through the oracle."""
    a, b = bs.opaque(48, 32, 120, seed=21), bs.tiny(48, 32, 150, seed=22)
    sc = scenes.Scene(*[torch.cat([getattr(a, k), getattr(b, k)]) for k in ("means3D", "scales", "rotations", "opacities", "shs")],
                      a.viewmatrix, a.projmatrix, a.campos, a.bg, a.width, a.height, a.tanfovx, a.tanfovy)
    inp = _scene_inputs(sc, True, True, 0.0)
    up = {k: v.numpy() for k, v in scenes.make_upstream_grads(sc.height, sc.width, seed=23).items()}
    fo, bl, ref, sg, rb = _oracle_roundtrip(inp, up, "planted")
    return inp, up, fo, bl, ref, sg, rb


def _busy_pixel(ref):
    amb = ref["ambiguous"].numpy()
    last = ref["n_contrib"][0].numpy()
    y, x = np.unravel_index(np.argmax(np.where(amb, 0, last)), last.shape)
    return int(y), int(x)


def test_planted_dropped_list_entry_is_caught(planted):
    inp, up, fo, bl, ref, _, _ = planted
    y, x = _busy_pixel(ref)
    gx = (inp.W + 15) // 16
    tile = (y // 16) * gx + x // 16
    rg = fo["binning"]["ranges"].astype(np.int64)
    drop = int(rg[tile, 0])  # the first entry of the tile: the busy pixel blends it
    pl = np.delete(fo["binning"]["point_list"], drop)
    rg2 = rg.copy()
    rg2[tile, 1] -= 1
    rg2[tile + 1:] -= 1
    rg2[rg2 < 0] = 0
    img = oracle.render_forward(inp, fo["geom"], dict(point_list=pl, ranges=rg2.astype(np.uint32)))
    with pytest.raises(AssertionError, match=r"pixel \(y=\d+, x=\d+\)"):
        bf.check_forward(ref, _oracle_given(inp, dict(image=img)), bl, "dropped")


def test_planted_median_shift_is_caught(planted):
    inp, up, fo, bl, ref, _, rb = planted
    y, x = _busy_pixel(ref)
    img = {k: v.copy() for k, v in fo["image"].items()}
    img["n_contrib"][1, y, x] += 1
    with pytest.raises(AssertionError, match=rf"n_contrib at pixel \(y={y}, x={x}\)"):
        bf.check_forward(ref, _oracle_given(inp, dict(image=img)), bl, "median")
    sg = oracle.render_backward(inp, dict(fo, image=img), up)  # backward fed the shifted median, checked against the true state
    with pytest.raises(AssertionError, match=r"of row \d+"):
        bf.check_backward(rb, sg, "median")


def test_planted_missing_pixel_in_one_row_is_caught(planted):
    inp, up, fo, bl, ref, sg, rb = planted
    y, x = _busy_pixel(ref)
    one = {k: np.zeros_like(v) for k, v in up.items()}
    for k in one:
        one[k][:, y, x] = up[k][:, y, x]
    sp = oracle.render_backward(inp, fo, one)  # the backward is linear in the upstream gradients: this is pixel (y, x) alone
    row = int(np.argmax(np.abs(sp["opacity"])))
    given = {k: v.copy() for k, v in sg.items()}
    for k in given:
        given[k][row] -= sp[k][row]
    with pytest.raises(AssertionError, match=rf"of row {row}:"):
        bf.check_backward(rb, given, "missing pixel")


def test_planted_conic_scale_is_caught(planted):
    _, _, _, _, _, sg, rb = planted
    b = rb["b_conic"][:, 0].numpy()
    r = np.abs(rb["conic"][:, 0].numpy())
    row = int(np.argmax(np.where(b > 0, r / np.where(b > 0, b, 1), 0)))
    assert r[row] * 1e-3 > 2 * b[row]
    given = {k: v.copy() for k, v in sg.items()}
    given["conic"][row] *= 1 + 1e-3
    with pytest.raises(AssertionError, match=rf"conic\[0\] of row {row}:"):
        bf.check_backward(rb, given, "conic")


def test_planted_clamp_gradient_zeroed_is_caught(planted):
    inp, up, fo, bl, ref, sg, rb = planted
    state = {k: fo["image"][k] for k in STATE}
    wrong = bf.backward(bl, state, up, clamp_keeps_gradient=False)
    given = {k: v + (wrong[k].numpy().reshape(v.shape) - rb[k].numpy().reshape(v.shape)) for k, v in sg.items()}
    with pytest.raises(AssertionError, match=r"(mean2D|conic|opacity)\[\d\] of row \d+"):
        bf.check_backward(rb, given, "clamp")
