"""fp64 model of the fused activations (csrc/rgs_activation.cu, activate_forward/backward_kernel) with a rigorous bound per
element on where an fp32 evaluation of the kernels' expressions may land (tests/f32_error.py).

The operation is the reference's GaussianModel.get_scaling_n_opacity_with_3D_filter and get_rotation
(scene/gaussian_model.py:156-166 and :125-126), written from the math:

    s_k = exp(raw_k),  after_k = s_k^2 + f^2,  scales_k = sqrt(after_k)
    coef = sqrt(prod s_k^2 / prod after_k),  opacity = sigmoid(raw_o) * coef
    rotations = r / max(|r|, 1e-12)                                    (F.normalize)

and its derivatives, with d coef / d raw_k = coef * f^2 / after_k (the form the kernel evaluates) and F.normalize's
clamp_min passing no gradient to the norm when |r| <= 1e-12.

Two decisions are not arithmetic:
  * `|r| > 1e-12` in backward.  A row whose fp32 norm may fall on either side is *ambiguous*: both branches are admitted.
  * sigmoid.  The kernel's 1/(1 + expf(-x)) returns 0 once expf(-x) overflows (x < -88.7), where torch's sigmoid returns the
    subnormal value (3.7e-44 at -100).  Below the smallest normal fp32 (2^-126) the bound therefore admits [0, 2^-126]:
    SIGMOID_SUBNORMAL is that documented allowance; above it sigmoid is within K_SIGMOID u.
"""
from __future__ import annotations

import torch

from f32_error import ETA, R, U, f32, stack

K_SIGMOID = 8.0                  # expf (2 ulp, damped by E / (1 + E)), the sum and the reciprocal, with margin
SIGMOID_SUBNORMAL = 2.0 ** -126  # sigmoid(x) below the normal range: 0 or the subnormal value are both admitted
NORM_EPS = f32(1e-12)


def _sigmoid(x: R) -> R:
    v = torch.sigmoid(x.v)
    e = K_SIGMOID * U * v + ETA + torch.where(v < SIGMOID_SUBNORMAL, torch.full_like(v, SIGMOID_SUBNORMAL), torch.zeros_like(v))
    s = None if x.s is None else 1.0 / (1.0 + torch.exp(-x.s))
    return R(v, e, s)


def _inputs(raw, shadow, device):
    return [R.input(t, shadow, device) for t in raw]


def _scaling(raw_scaling: R, filter_3D: R):
    f = filter_3D[:, 0]
    f2 = f * f
    s = [raw_scaling[:, k].exp() for k in range(3)]
    sq = [x * x for x in s]
    after = [q + f2 for q in sq]
    det1 = sq[0] * sq[1] * sq[2]
    det2 = after[0] * after[1] * after[2]
    coef = (det1 / det2).sqrt()
    return f2, s, sq, after, coef


def forward(raw_scaling, raw_opacity, raw_rotation, filter_3D, shadow=False, device="cpu") -> dict:
    """{scales [P,3], opacity [P,1], rotations [P,4]} as R (value, bound)."""
    rs, ro, rr, fl = _inputs((raw_scaling, raw_opacity, raw_rotation, filter_3D), shadow, device)
    _, _, _, after, coef = _scaling(rs, fl)
    scales = [a.sqrt() for a in after]
    o = _sigmoid(ro[:, 0])
    q = [rr[:, k] for k in range(4)]
    n = ((q[0] * q[0] + q[1] * q[1]) + (q[2] * q[2] + q[3] * q[3])).sqrt()   # the forward kernel's pairing
    d = n.maximum(NORM_EPS)
    return {"scales": stack(scales, 1), "opacity": stack([o * coef], 1), "rotations": stack([x / d for x in q], 1)}


def backward(raw_scaling, raw_opacity, raw_rotation, filter_3D, g_scales, g_opacity, g_rotations, shadow=False, device="cpu") -> dict:
    """{d_raw_scaling [P,3], d_raw_opacity [P,1], d_raw_rotation [P,4]} as R, and `ambiguous` [P]: rows whose |r| > 1e-12
    decision the fp32 norm may flip (their d_raw_rotation admits both branches: `d_raw_rotation_alt`)."""
    rs, ro, rr, fl, gs, go, gr = _inputs((raw_scaling, raw_opacity, raw_rotation, filter_3D, g_scales, g_opacity, g_rotations), shadow, device)
    f2, s, sq, after, coef = _scaling(rs, fl)
    o = _sigmoid(ro[:, 0])
    g_o = go[:, 0]
    d_raw_opacity = g_o * coef * o * (1.0 - o)
    d_coef_f2 = g_o * o * coef * f2
    d_raw_scaling = []
    for k in range(3):
        scale_out = after[k].sqrt()
        d_scale = gs[:, k] / (2.0 * scale_out) * 2.0 * s[k] * s[k]
        d_raw_scaling.append(d_coef_f2 / after[k] + d_scale)
    q = [rr[:, k] for k in range(4)]
    g = [gr[:, k] for k in range(4)]
    n = (((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]).sqrt()      # the backward kernel's order
    safe = n.v > 0
    inv = 1.0 / n.where(safe, 1.0)
    u = [x * inv for x in q]
    ug = ((u[0] * g[0] + u[1] * g[1]) + u[2] * g[2]) + u[3] * g[3]
    through = stack([(g[k] - u[k] * ug) * inv for k in range(4)], 1)
    clamped = stack([x / NORM_EPS for x in g], 1)
    above = n.v > NORM_EPS
    ambiguous = (n.v - NORM_EPS).abs() <= n.e
    primary = through.where(above[:, None], clamped)
    alternate = clamped.where(above[:, None], through)
    return {"d_raw_scaling": stack(d_raw_scaling, 1), "d_raw_opacity": stack([d_raw_opacity], 1), "d_raw_rotation": primary,
            "d_raw_rotation_alt": alternate, "ambiguous": ambiguous}


# ---- the reference expressions, for the host tests (fp64 autograd) ------------------------------------------------------

def reference(raw_scaling, raw_opacity, raw_rotation, filter_3D):
    """scene/gaussian_model.py:156-166 and :125-126 as torch expressions, in the dtype of the arguments."""
    opacity = torch.sigmoid(raw_opacity)
    scales = torch.exp(raw_scaling)
    scales_square = torch.square(scales)
    det1 = scales_square.prod(dim=1)
    scales_after_square = scales_square + torch.square(filter_3D)
    det2 = scales_after_square.prod(dim=1)
    coef = torch.sqrt(det1 / det2)
    return torch.sqrt(scales_after_square), opacity * coef[..., None], torch.nn.functional.normalize(raw_rotation)


# ---- input families ------------------------------------------------------------------------------------------------------

def families(seed=0) -> dict:
    """{name: (raw_scaling [n,3], raw_opacity [n,1], raw_rotation [n,4], filter_3D [n,1])} fp32 CPU tensors."""
    g = torch.Generator().manual_seed(seed)
    out = {}

    def typical(n):
        return ((torch.randn(n, 3, generator=g) * 1.5 - 3.0), torch.randn(n, 1, generator=g) * 2.0, torch.randn(n, 4, generator=g),
                torch.rand(n, 1, generator=g) * 0.05 + 1e-4)

    out["typical"] = typical(4096)
    # tiny scales: every axis down to -20, and one axis tiny with two ordinary ones (flat Gaussians); all four filter sizes
    filters = torch.tensor([0.0, 1e-6, 1e-4, 0.05])
    rows = []
    for lo in (-20.0, -16.0, -12.0, -9.0, -6.0):
        for f in filters:
            n = 64
            rs = torch.empty(n, 3).uniform_(lo, lo + 3.0, generator=g)
            flat = rs.clone()
            flat[:, :2] = torch.randn(n, 2, generator=g) * 0.7 - 2.5
            rows.append((torch.cat([rs, flat]), torch.full((2 * n, 1), float(f))))
    rs = torch.cat([r for r, _ in rows])
    fl = torch.cat([f for _, f in rows])
    # at f = 0 with all three raw below about -17, det1 = det2 underflow to 0 and the reference's fp32 expression is 0 / 0
    # (NaN in the kernel and in eager torch alike); compute_3D_filter never yields f = 0, so those rows are left out
    keep = (torch.exp(2.0 * rs.double()) + fl.double() ** 2).prod(1) >= 2.0 ** -140
    rs, fl = rs[keep], fl[keep]
    n = rs.shape[0]
    out["tiny_scales"] = (rs, torch.randn(n, 1, generator=g) * 2.0, torch.randn(n, 4, generator=g), fl)
    # det2 = prod(s_k^2 + f^2) near f^6: det2^2 leaves the fp32 range at (-9, -9, -16) with f = 1e-4
    out["tiny_scales"] = tuple(torch.cat([a, b]) for a, b in zip(out["tiny_scales"], (
        torch.tensor([[-8.0, -8.0, -15.0], [-9.0, -9.0, -16.0], [-3.0, -3.0, -3.0]]), torch.zeros(3, 1),
        torch.tensor([[1.0, 0.0, 0.0, 0.0]] * 3), torch.tensor([[2e-4], [1e-4], [1e-2]]))))
    rs, ro, rr, fl = typical(4 * 4 * 64)
    fl = filters.repeat_interleave(4 * 64)[:, None].clone()
    out["filters"] = (rs, ro, rr, fl)
    rs, _, rr, fl = typical(8 * 64)
    ro = torch.tensor([30.0, -30.0, 100.0, -100.0, 88.0, -88.0, 89.0, -89.0]).repeat_interleave(64)[:, None]
    out["saturated_opacity"] = (rs, ro, rr, fl)
    rs, ro, rr, fl = typical(5 * 64)
    direction = torch.nn.functional.normalize(torch.randn(5 * 64, 4, generator=g), dim=1)
    norms = torch.tensor([0.0, 1e-13, 1e-12, 1e-6, 1e6]).repeat_interleave(64)[:, None]
    out["quaternion_norms"] = (rs, ro, direction * norms, fl)
    return out


def upstream(n, seed, zero=()):
    """Upstream gradients (g_scales [n,3], g_opacity [n,1], g_rotations [n,4]); those named in `zero` are zero, as autograd
    passes them for unused outputs."""
    g = torch.Generator().manual_seed(seed)
    gs, go, gr = (torch.randn(n, k, generator=g) for k in (3, 1, 4))
    return tuple(torch.zeros_like(t) if name in zero else t for t, name in zip((gs, go, gr), ("scales", "opacity", "rotations")))
