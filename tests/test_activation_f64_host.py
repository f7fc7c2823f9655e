"""The fp64 activation model (tests/activation_f64.py) validated without a GPU: it equals fp64 autograd of the reference's
expressions, and its bounds hold an fp32 evaluation of the kernels' expressions and torch's own fp32 forward at every row."""
import pytest
import torch

import activation_f64 as af
from f32_error import check, check_shadow

FAMILIES = af.families(seed=7)
NORM_EPS_RTOL = 5e-9   # F.normalize's eps is the double 1e-12, the kernel's the float 1e-12f: 4e-9 apart


def _autograd64(raw, grads):
    leaves = [t.double().requires_grad_(True) for t in raw[:3]]
    outs = af.reference(*leaves, raw[3].double())
    torch.autograd.backward(list(outs), [g.double() for g in grads])
    return [o.detach() for o in outs], [t.grad for t in leaves]


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_model_equals_fp64_autograd_of_the_reference(family):
    raw = FAMILIES[family]
    grads = af.upstream(raw[0].shape[0], 3)
    (rs, ro, rr), (ds, do, dr) = _autograd64(raw, grads)
    fw = af.forward(*raw)
    bw = af.backward(*raw, *grads)
    n = raw[2].double().norm(dim=1)
    clamped = n <= 1e-12
    decided = ~bw["ambiguous"] & ~((n - af.NORM_EPS).abs() <= 1e-7 * n)   # both eps on the same side
    torch.testing.assert_close(fw["scales"].v, rs, rtol=1e-12, atol=0)
    torch.testing.assert_close(fw["opacity"].v, ro, rtol=1e-12, atol=0)
    torch.testing.assert_close(fw["rotations"].v[~clamped], rr[~clamped], rtol=1e-12, atol=0)
    torch.testing.assert_close(fw["rotations"].v[clamped], rr[clamped], rtol=NORM_EPS_RTOL, atol=0)
    torch.testing.assert_close(bw["d_raw_opacity"].v, do, rtol=1e-12, atol=1e-300)
    # autograd's chain through det1 and det2 cancels to f^2 / after_k of its terms: compare relative to those terms
    scale = ds.abs() + (grads[1].double() * ro).abs() + grads[0].double().abs()
    assert ((bw["d_raw_scaling"].v - ds).abs() <= 1e-12 * scale).all()
    keep = decided & ~clamped
    torch.testing.assert_close(bw["d_raw_rotation"].v[keep], dr[keep], rtol=1e-12, atol=1e-12 * dr[keep].abs().max().item())
    keep = decided & clamped
    torch.testing.assert_close(bw["d_raw_rotation"].v[keep], dr[keep], rtol=NORM_EPS_RTOL, atol=0)


@pytest.mark.parametrize("zero", [(), ("scales", "rotations"), ("opacity",)])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bounds_hold_an_fp32_evaluation(family, zero):
    raw = FAMILIES[family]
    grads = af.upstream(raw[0].shape[0], 4, zero)
    fw = af.forward(*raw, shadow=True)
    for k in ("scales", "opacity", "rotations"):
        check_shadow(fw[k], f"{family} {k}")
    bw = af.backward(*raw, *grads, shadow=True)
    for k in ("d_raw_scaling", "d_raw_opacity"):
        check_shadow(bw[k], f"{family} {k}")
    amb = bw["ambiguous"]
    check_shadow(bw["d_raw_rotation"][~amb], f"{family} d_raw_rotation")


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bounds_hold_torch_fp32_forward(family):
    """torch's own fp32 forward (the reference's expressions, torch.sigmoid included) within the bound at every row."""
    raw = FAMILIES[family]
    s, o, r = af.reference(*raw)
    fw = af.forward(*raw)
    check(s, fw["scales"], f"{family} scales")
    check(o, fw["opacity"], f"{family} opacity")
    n = raw[2].double().norm(dim=1)
    keep = n > 2e-12   # F.normalize divides by eps = 1e-12 below it, the kernel by 1e-12f
    check(r[keep], fw["rotations"][keep], f"{family} rotations")


def test_the_det2_squared_form_leaves_the_bound():
    """The autograd form -d_q det1 / (det2 det2) evaluated in fp32 is -inf on the flat row (-9, -9, -16), f = 1e-4, where the
    model is finite: the bound is tight enough to refuse it."""
    raw = (torch.tensor([[-9.0, -9.0, -16.0]]), torch.zeros(1, 1), torch.tensor([[1.0, 0, 0, 0]]), torch.tensor([[1e-4]]))
    grads = (torch.zeros(1, 3), torch.ones(1, 1), torch.zeros(1, 4))
    s = torch.exp(raw[0])
    sq = s * s
    after = sq + raw[3] * raw[3]
    det1, det2 = sq.prod(1), after.prod(1)
    coef = torch.sqrt(det1 / det2)
    o = torch.sigmoid(raw[1][:, 0])
    d_q = o / (2 * coef)
    d_det2 = -d_q * det1 / (det2 * det2)
    assert torch.isinf(d_det2).all()
    bw = af.backward(*raw, *grads)
    assert torch.isfinite(bw["d_raw_scaling"].v).all() and torch.isfinite(bw["d_raw_scaling"].e).all()
    with pytest.raises(AssertionError):
        check(torch.full((1, 3), float("-inf")), bw["d_raw_scaling"], "det2^2 form")
