"""The fused activation kernels at every Gaussian against the fp64 model of tests/activation_f64.py: every output element
within its own bound, no outlier budget.  Rows whose `|r| > 1e-12` decision the fp32 norm may flip admit both branches.

The families aim at the kernels' edges: scales down to exp(-20) per axis and flat Gaussians, filter_3D of 0, 1e-6, 1e-4 and
0.05, saturated opacities, quaternions of norm 0 to 1e6, P around the 256-thread block, and upstream gradients that are zero
for some outputs, as autograd passes them."""
import math

import pytest
import torch

import activation_f64 as af
from f32_error import check, excess

pytestmark = pytest.mark.gpu

FAMILIES = af.families(seed=11)
WORST = {}


def _table(P, seed):
    """All families' rows, then typical rows, tiled to P rows."""
    cols = [torch.cat([FAMILIES[k][i] for k in sorted(FAMILIES)]) for i in range(4)]
    n = cols[0].shape[0]
    idx = torch.randperm(max(P, n), generator=torch.Generator().manual_seed(seed)) % n
    return tuple(c[idx[:P]].contiguous() for c in cols)


def _record(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


def _check_backward(raw, grads, d_s, d_o, d_r, tag):
    bw = af.backward(*raw, *grads, device="cuda")
    _record("d_raw_scaling", check(d_s, bw["d_raw_scaling"], f"{tag} d_raw_scaling"))
    _record("d_raw_opacity", check(d_o, bw["d_raw_opacity"], f"{tag} d_raw_opacity"))
    amb = bw["ambiguous"]
    x = torch.minimum(excess(d_r, bw["d_raw_rotation"]), torch.where(amb[:, None], excess(d_r, bw["d_raw_rotation_alt"]), float("inf")))
    bad = torch.nonzero(~(x <= 1.0))
    assert bad.numel() == 0, f"{tag} d_raw_rotation: {bad.shape[0]} elements outside their bound, first at {bad[0].tolist()}"
    _record("d_raw_rotation", float(x.max()))


@pytest.mark.parametrize("P", [1, 255, 256, 257, 100_003])
def test_activate_forward_every_row_within_bound(P):
    from diff_gaussian_rasterization import _C

    raw = _table(P, P)
    s, o, r = _C.activate_forward(*(t.cuda() for t in raw))
    fw = af.forward(*raw, device="cuda")
    for name, got in (("scales", s), ("opacity", o), ("rotations", r)):
        _record(name, check(got, fw[name], f"P={P} {name}"))


@pytest.mark.parametrize("P", [1, 255, 256, 257, 100_003])
def test_activate_backward_every_row_within_bound(P):
    from diff_gaussian_rasterization import _C

    raw = _table(P, P + 1)
    grads = af.upstream(P, P)
    d_s, d_o, d_r = _C.activate_backward(*(t.cuda() for t in raw), *(g.cuda() for g in grads))
    _check_backward(raw, grads, d_s, d_o, d_r, f"P={P}")


@pytest.mark.parametrize("used", ["opacity", "scales", "rotations", "scales+opacity"])
def test_activate_backward_through_autograd_with_unused_outputs(used):
    """Only some outputs reach the loss: autograd hands zero gradients for the others."""
    from rade_gs_b200.fused import activate_gaussians

    P = 4099
    raw = _table(P, 5)
    grads = af.upstream(P, 6, zero=tuple(k for k in ("scales", "opacity", "rotations") if k not in used))
    leaves = [t.cuda().requires_grad_(True) for t in raw[:3]]
    outs = activate_gaussians(*leaves, raw[3].cuda())
    loss = sum((o * g.cuda()).sum() for o, g, k in zip(outs, grads, ("scales", "opacity", "rotations")) if k in used)
    loss.backward()
    _check_backward(raw, grads, leaves[0].grad, leaves[1].grad, leaves[2].grad, used)


def test_flat_rows_have_finite_gradients():
    """The rows where autograd's det2^2 form leaves fp32: finite and within bound (-inf before the closed form)."""
    from diff_gaussian_rasterization import _C

    raw = (torch.tensor([[-9.0, -9.0, -16.0], [-8.0, -8.0, -15.0]]), torch.zeros(2, 1), torch.tensor([[1.0, 0, 0, 0]] * 2),
           torch.tensor([[1e-4], [2e-4]]))
    grads = (torch.zeros(2, 3), torch.ones(2, 1), torch.zeros(2, 4))
    d_s, d_o, d_r = _C.activate_backward(*(t.cuda() for t in raw), *(g.cuda() for g in grads))
    assert torch.isfinite(d_s).all(), d_s
    _check_backward(raw, grads, d_s, d_o, d_r, "flat rows")


# ---- 3D filter --------------------------------------------------------------------------------------------------------------

def filter_scene(n_cams, P, seed, one_seen=False):
    """Points around the origin, cameras 4 to 9 units away looking at it; then points placed on the z = 0.2 plane and on the four
    15 % margin lines of a few chosen cameras (the last of each 256-camera chunk among them)."""
    import numpy as np
    from types import SimpleNamespace

    rng = np.random.default_rng(seed)
    cams = []
    for _ in range(n_cams):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        if np.linalg.det(q) < 0:
            q[:, 0] = -q[:, 0]
        cams.append(SimpleNamespace(R=q, T=rng.normal(size=3) * 0.5 + np.array([0, 0, rng.uniform(4.0, 9.0)]), FoVx=float(rng.uniform(0.5, 1.2)),
                                    FoVy=float(rng.uniform(0.4, 1.0)), image_width=int(rng.integers(300, 1700)), image_height=int(rng.integers(200, 1300))))
    if one_seen:
        # every camera looks away from the cloud but one point sits in front of camera 0
        for c in cams:
            c.T = np.array([0, 0, -50.0])
        xyz = rng.normal(size=(P, 3)) * 2.0
        xyz[P // 2] = (np.array([0.1, -0.2, 60.0]) - cams[0].T) @ cams[0].R.T
        return xyz.astype(np.float32), cams
    xyz = [rng.normal(size=(P, 3)) * 3.0]
    chosen = sorted({0, min(255, n_cams - 1), n_cams - 1, n_cams // 2})
    for k in chosen:
        c = cams[k]
        W, H = c.image_width, c.image_height
        fx, fy = W / (2 * math.tan(c.FoVx / 2)), H / (2 * math.tan(c.FoVy / 2))
        m = 64
        zc = np.concatenate([np.full(m, 0.2), rng.uniform(0.5, 8.0, 4 * m)])
        u = np.concatenate([rng.uniform(-0.15 * W, 1.15 * W, m), np.full(m, -0.15 * W), np.full(m, 1.15 * W), rng.uniform(-0.15 * W, 1.15 * W, 2 * m)])
        v = np.concatenate([rng.uniform(-0.15 * H, 1.15 * H, 3 * m), np.full(m, -0.15 * H), np.full(m, 1.15 * H)])
        cam_pts = np.stack([(u - W / 2) / fx * zc, (v - H / 2) / fy * zc, zc], 1)
        xyz.append((cam_pts - c.T) @ c.R.T)
    return np.concatenate(xyz).astype(np.float32), cams


@pytest.mark.parametrize("n_cams,P", [(1, 1000), (255, 3001), (256, 2999), (257, 4097), (513, 2333)])
def test_compute_3D_filter_every_point_within_its_interval(n_cams, P):
    import filter3d_f64 as ff
    from rade_gs_b200.fused import compute_3D_filter

    xyz, cams = filter_scene(n_cams, P, seed=n_cams)
    assert xyz.shape[0] % 256 != 0
    out = compute_3D_filter(torch.from_numpy(xyz).cuda(), cams)[:, 0].double()
    lo, hi, d = ff.filter_intervals(xyz, cams, device="cuda")
    bad = torch.nonzero(~((out >= lo) & (out <= hi)))
    assert bad.numel() == 0, [(i, out[i].item(), lo[i].item(), hi[i].item(), bool(d["ambiguous"][i])) for i in bad[:6, 0].tolist()]
    assert d["ambiguous"].any() or n_cams == 1      # the placed points reach the decisions
    sure = ~d["ambiguous"] & d["surely_seen"]
    width = ((hi - lo) / hi.abs().clamp_min(1e-30))[sure]
    _record("filter_3D interval width (rel.)", float(width.max()))


def test_compute_3D_filter_with_one_seen_point():
    import filter3d_f64 as ff
    from rade_gs_b200.fused import compute_3D_filter

    xyz, cams = filter_scene(3, 777, seed=4, one_seen=True)
    out = compute_3D_filter(torch.from_numpy(xyz).cuda(), cams)[:, 0].double()
    lo, hi, d = ff.filter_intervals(xyz, cams, device="cuda")
    assert int(d["surely_seen"].sum()) == 1 and int(d["possibly_seen"].sum()) == 1
    assert ((out >= lo) & (out <= hi)).all()
    assert torch.unique(out).numel() == 1     # every point gets the one seen point's distance


def test_report_worst_ratios():
    """Runs last in this module: the worst error / bound ratio per output over the tests above."""
    print("\nactivation worst error/bound:", {k: f"{v:.3g}" for k, v in sorted(WORST.items())})
