"""The fp64 integrate model (tests/integrate_f64.py) validated without a GPU: the CPU oracle's `integrate` must lie within the
model's bounds at every pixel and every point (on the three integrate fixtures' inputs and two fresh scenes), the model's
invray must contain the oracle's, and defects planted in the oracle's outputs must be caught with a message naming the pixel
or point."""
import numpy as np
import pytest

import integrate_f64 as mf
import oracle
from conftest import INTEGRATE_CASES, integrate_oracle_inputs, load_golden


def _oracle_case(inp, pts):
    ref = oracle.integrate(inp, pts)
    g, b = ref["geom"], ref["binning"]
    st = dict(means2D=g["means2D"], conic_opacity=g["conic_opacity"], rgb=g["rgb"], ts=g["ts"], ray_planes=g["ray_planes"], radii=g["radii"],
              ranges=b["ranges"], point_list=b["point_list"], sigma_inv=ref["sigma_inv"])
    it = mf.make_integrate(st, inp.W, inp.H, inp.tanfovx, inp.tanfovy, inp.bg, inp.viewmatrix, inp.means3D)
    given = dict(color=ref["color"].copy(), alpha_integrated=ref["alpha_integrated"].copy(), color_integrated=ref["color_integrated"].copy(),
                 point_coordinate=ref["point_coordinate"].copy(), point_sdf=ref["point_sdf"].copy(), overflow_count=ref["overflowed"])
    return ref, it, given


def _model(it, pts, given, trace=None):
    inn = ~mf.culled(given["alpha_integrated"], given["color_integrated"], given["point_coordinate"], given["point_sdf"])
    return mf.integrate(it, pts, given["point_coordinate"], inn, trace=trace)


def _fresh(seed, P, W, H, focal, PN):
    from integrate_scenes import make_points
    from rade_gs_b200 import scenes
    sc = scenes.make_scene(P, W, H, focal, -2.2, seed=seed, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.3, 0.1, 0.2))
    pts = make_points(sc, PN, seed + 1).numpy()
    inp = oracle.Inputs(sc.means3D.numpy(), sc.opacities.numpy(), sc.viewmatrix.numpy(), sc.projmatrix.numpy(), sc.campos.numpy(), sc.bg.numpy(),
                        W, H, sc.tanfovx, sc.tanfovy, sh_degree=3, kernel_size=0.0, require_coord=True, require_depth=True, shs=sc.shs.numpy(),
                        scales=sc.scales.numpy(), rotations=sc.rotations.numpy())
    return inp, pts


def _inputs(name):
    if name.startswith("fresh"):
        return _fresh(*((11, 900, 72, 56, 70.0, 4000) if name == "fresh_a" else (12, 1500, 61, 37, 55.0, 6000)))
    d = load_golden(name)
    return integrate_oracle_inputs(d), d["in_points3D"]


CASES = list(INTEGRATE_CASES) + ["fresh_a", "fresh_b"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_within_model_bounds(name):
    inp, pts = _inputs(name)
    ref, it, given = _oracle_case(inp, pts)
    m = _model(it, pts, given)
    stats = mf.check(m, given, it, name)
    print(f"\n[{name}] " + " ".join(f"{k}={v:.3g}" for k, v in stats.items()))
    # invray: the oracle's matrix within the model's bound wherever the kernels use it (radii > 0)
    live = it.radii.numpy() > 0
    d = np.abs(m["invray"]["M"].numpy() - ref["invraycov"])[live]
    b = m["invray"]["b_M"].numpy()[live]
    assert (d <= b).all(), f"{name}: invray outside its bound for Gaussians {np.nonzero(live)[0][np.nonzero((d > b).any(1))[0]][:8]}"
    assert np.array_equal(m["invray"]["condition"].numpy()[live], ref["condition"][live].astype(bool))


# ---- planted defects ---------------------------------------------------------------------------------------------------

def _traced(name="integrate_tilt", want=None):
    """The oracle on a fixture, and the trace of a pixel with several points and several used entries."""
    inp, pts = _inputs(name)
    ref, it, given = _oracle_case(inp, pts)
    m = _model(it, pts, given)
    cnt = given["color"][8]
    amb = m["ambiguous"].numpy()
    cands = np.argwhere((cnt >= 2) & ~amb)
    for y, x in cands:
        t = _model(it, pts, given, trace=(int(y), int(x)))["trace"]
        if t is not None and len(t["pt_id"]) and (want is None or want(t)):
            return it, pts, given, m, t, (int(y), int(x))
    raise AssertionError("no suitable pixel")


def _expect_fail(it, pts, given, what):
    m = _model(it, pts, given)
    with pytest.raises(AssertionError) as e:
        mf.check(m, given, it, "planted")
    assert what in str(e.value), str(e.value)[:2000]
    return str(e.value)


def _drop(given, t, sel):
    """Remove one entry's factor from the alpha of the points of the traced pixel that composited it."""
    ids, pos, al = t["pt_id"].numpy(), t["pt_pos"].numpy(), t["pt_alpha"].numpy()
    k = np.nonzero(sel(pos))[0]
    k = k[np.argmax(al[k])]
    p = int(pos[k])
    hit = np.nonzero(pos == p)[0]
    for j in hit:
        i = int(ids[j])
        a = float(given["alpha_integrated"][i])
        given["alpha_integrated"][i] = np.float32(1 - (1 - a) / (1 - al[j]))
    return int(ids[hit[0]])


def test_planted_used_entry_dropped():
    it, pts, given, m, t, (y, x) = _traced()
    i = _drop(given, t, lambda pos: np.ones_like(pos, bool))
    _expect_fail(it, pts, given, f"point {i} (pixel y={y}, x={x})")


def test_planted_corner_only_entry_dropped():
    def corner(t):
        co = np.nonzero(t["used_corner_only"].numpy())[0]
        return bool(np.isin(t["pt_pos"].numpy(), co).any())
    it, pts, given, m, t, (y, x) = _traced("integrate_dense", want=corner)
    co = np.nonzero(t["used_corner_only"].numpy())[0]
    i = _drop(given, t, lambda pos: np.isin(pos, co))
    _expect_fail(it, pts, given, f"point {i} (pixel y={y}, x={x})")


def test_planted_alpha_off_by_1e5():
    inp, pts = _inputs("integrate_tilt")
    ref, it, given = _oracle_case(inp, pts)
    m = _model(it, pts, given)
    lo, hi = m["alpha_lo"].numpy(), m["alpha_hi"].numpy()
    ok = m["in_given"].numpy() & ((hi - lo) < 5e-6) & (given["alpha_integrated"] > 0.05) & (given["alpha_integrated"] < 0.95)
    i = int(np.nonzero(ok)[0][0])
    given["alpha_integrated"][i] += np.float32(1e-5)
    _expect_fail(it, pts, given, f"point {i} ")


def test_planted_points_swapped():
    inp, pts = _inputs("integrate_tilt")
    ref, it, given = _oracle_case(inp, pts)
    inn = ~mf.culled(given["alpha_integrated"], given["color_integrated"], given["point_coordinate"], given["point_sdf"])
    a = given["alpha_integrated"]
    i = int(np.nonzero(inn & (a > 0.3))[0][0])
    j = int(np.nonzero(inn & (np.abs(a - a[i]) > 0.1))[0][0])
    for k in ("alpha_integrated", "color_integrated", "point_coordinate", "point_sdf"):
        given[k][[i, j]] = given[k][[j, i]]
    msg = _expect_fail(it, pts, given, f"point {i}")
    assert f"point {j}" in msg


def test_planted_point_moved_to_neighbour_pixel():
    inp, pts = _inputs("integrate_tilt")
    ref, it, given = _oracle_case(inp, pts)
    inn = ~mf.culled(given["alpha_integrated"], given["color_integrated"], given["point_coordinate"], given["point_sdf"])
    c = given["point_coordinate"]
    i = int(np.nonzero(inn & (c[:, 0] > 2) & (c[:, 0] < inp.W - 2))[0][0])
    given["point_coordinate"][i, 0] += 1.0
    _expect_fail(it, pts, given, f"point {i}: coordinate")


def test_planted_median_shifted_by_one():
    def has_next(t):
        uc = np.nonzero(t["used_centre"].numpy())[0]
        return t["median"] >= 0 and (uc > t["median"]).any()
    it, pts, given, m, t, (y, x) = _traced(want=has_next)
    uc = np.nonzero(t["used_centre"].numpy())[0]
    nxt = int(uc[uc > t["median"]][0])
    gid = int(t["ids"][nxt])
    W = it.W
    pix = m["pixel"].numpy()
    pids = np.nonzero(pix == y * W + x)[0]
    ts, rx, ry = float(it.ts[gid]), float(it.ray_planes[gid, 0]), float(it.ray_planes[gid, 1])
    mx, my = float(it.means2D[gid, 0]), float(it.means2D[gid, 1])
    qd = m["proj"]["qd"].numpy()
    for i in pids:
        qx, qy = given["point_coordinate"][i]
        given["point_sdf"][i] = np.float32(ts + (rx * (mx - qx) + ry * (my - qy)) - qd[i])
    _expect_fail(it, pts, given, f"point {int(pids[0])} (pixel y={y}, x={x}): point_sdf")
