"""fp64 models of the fused image losses (csrc/rgs_image_loss.cu) with a rigorous bound per element on where an fp32
evaluation of the kernels' expressions may land (tests/f32_error.py).  Everything is torch: CPU for the host tests, CUDA for
the GPU tests.

SSIM + L1 (utils/loss_utils.py:17-18 and :23-63, train.py:163), written from the math:
    mu1 = w * x, mu2 = w * y, s1 = w * x^2 - mu1^2, s2 = w * y^2 - mu2^2, s12 = w * xy - mu1 mu2  (11x11 Gaussian w, sigma 1.5,
    zero padding), SSIM = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s1 + s2 + C2)), L1 = |x - y|.
The window is the fp32 one-dimensional g the kernels use (`window()`), applied along both axes; the reference's fp32
outer product g g^T rounds each 2-D weight once more, which the kernel never does.  The gradient is carried as the kernel
splits it: three per-pixel partials of the SSIM map (`dmaps`: d/d mu1, d/d E[x^2], d/d E[xy]), convolved once more.

The bounds carry the cancellation of s = E[x^2] - mu^2: its error is that of E[x^2] and mu^2 (~u (E[x^2] + mu^2)), not
of s.  b = s1 + s2 + C2 >= C2 keeps every quotient's denominator away from 0.

The image sums are summed per CTA in fp32 (two pixels per thread, then a 32-lane shuffle tree: at most 6 additions deep),
then in fp64: their bound is the sum of the element bounds plus K_SUM u of the sum of magnitudes.  The normal loss is
summed the same way.

Normal consistency (train.py:143-156, utils/graphics_utils.py:97-126): back-projected points (or coordinate maps), central
differences dx (along H) and dy (along W) at interior pixels, n = normalize(dx x dy) with F.normalize's eps 1e-12,
error 1 - <N, n> (border pixels keep n = 0, error 1), weighted by w_e and w_m; the gradients of that weighted sum w.r.t.
the normal map and both depth (or coordinate) maps.  `len > 1e-12` is a decision: a pixel whose fp32 length may fall on
either side is *ambiguous* and admits both branches; at a clamped pixel the gradient is of order w / 1e-12 and the bound is
relative to it.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from f32_error import R, U, f32, stack

SW, SR = 11, 5
C1, C2 = (float(np.float32(np.float32(c) * np.float32(c))) for c in (0.01, 0.03))   # the kernel's 0.01f * 0.01f, 0.03f * 0.03f
K_SUM = 12.0                                  # fp32 additions in a CTA's partial sums: at most 4 per thread + 5 shuffle levels
NORM_EPS = f32(1e-12)


def window() -> list:
    """The kernel's fp32 taps: exp(-(x - 5)^2 / 4.5) rounded to fp32, divided by their fp32 sum (loss_utils.py:23-25)."""
    g = np.array([np.float32(math.exp(-((x - SW // 2) ** 2) / (2.0 * 1.5 * 1.5))) for x in range(SW)], np.float32)
    s = np.float32(0)
    for x in g:
        s = np.float32(s + x)
    return [float(np.float32(x / s)) for x in g]


def _shift(x: R, k, dim):
    """x shifted by k - SR along dim with zero fill: out[i] = x[i + k - SR]."""
    off = k - SR
    n = x.v.shape[dim]

    def one(t):
        if t is None:
            return None
        out = torch.zeros_like(t)
        length = n - abs(off)
        if length > 0:
            out.narrow(dim, max(-off, 0), length).copy_(t.narrow(dim, max(off, 0), length))
        return out

    return R(one(x.v), one(x.e), one(x.s))


def _conv(x: R, g, dim):
    acc = None
    for k in range(SW):
        xs = _shift(x, k, dim)
        acc = xs * g[k] if acc is None else xs.fma(g[k], acc)
    return acc


def _sum_bound(r: R, mask):
    """The fp64 sum of r over mask and the bound of the kernel's fp32-per-CTA, fp64-across sum."""
    v = torch.where(mask, r.v, 0).sum()
    e = torch.where(mask, r.e, 0).sum() + K_SUM * U * torch.where(mask, r.v.abs() + r.e, 0).sum()
    return v, e


def ssim_l1_forward(img, gt, row_lo=0, row_hi=None, shadow=False, device="cpu") -> dict:
    """img, gt: fp32 tensors with the same [.., H, W]; returns sums (ssim, l1) with bounds, dmaps [3, planes, H, W] as R and
    `rows`, the mask of counted rows."""
    H, W = img.shape[-2:]
    row_hi = H if row_hi is None else row_hi
    x = R.input(img.reshape(-1, H, W), shadow, device)
    y = R.input(gt.reshape(-1, H, W), shadow, device)
    g = window()
    # horizontal pass: wa = w a rounded, m += wa, e11 = fma(wa, a, e11) (the kernel's order)
    m1 = m2 = e11 = e22 = e12 = None
    for k in range(SW):
        a, b = _shift(x, k, 2), _shift(y, k, 2)
        wa, wb = a * g[k], b * g[k]
        if m1 is None:
            m1, m2, e11, e22, e12 = wa, wb, wa * a, wb * b, wa * b
        else:
            m1, m2 = m1 + wa, m2 + wb
            e11, e22, e12 = wa.fma(a, e11), wb.fma(b, e22), wa.fma(b, e12)
    mu1, mu2, e11, e22, e12 = (_conv(t, g, 1) for t in (m1, m2, e11, e22, e12))
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = e11 - mu1_sq, e22 - mu2_sq, e12 - mu12
    a_ = mu1_sq + mu2_sq + C1
    b_ = s1 + s2 + C2
    c_ = 2.0 * mu12 + C1
    d_ = 2.0 * s12 + C2
    inv_ab = 1.0 / (a_ * b_)
    cd = c_ * d_
    ssim = cd * inv_ab
    l1 = (x - y).abs()
    dm0 = 2.0 * mu2 * (d_ - c_) * inv_ab - 2.0 * mu1 * cd * (b_ - a_) * inv_ab * inv_ab
    dm1 = -cd * inv_ab / b_
    dm2 = 2.0 * c_ * inv_ab
    rows = torch.zeros(H, dtype=torch.bool, device=x.v.device)
    rows[row_lo:row_hi] = True
    mask = rows[None, :, None].expand_as(x.v)
    sums = [_sum_bound(ssim, mask), _sum_bound(l1, mask)]
    return {"sums": sums, "dmaps": stack([dm0, dm1, dm2], 0), "rows": rows, "ssim_map": ssim, "x": x, "y": y}


def ssim_l1_backward(fw: dict, w_ssim, w_l1, upstream=None, row_lo=0, row_hi=None) -> R:
    """d_img [planes, H, W] as R for the kernel's weights (fp32 w_ssim, w_l1, optional fp32 upstream scalar)."""
    x, y, rows = fw["x"], fw["y"], fw["rows"]
    planes, H, W = x.v.shape
    g = window()
    mask = rows[None, None, :, None]
    dm = fw["dmaps"]
    dm = R(dm.v * mask, dm.e * mask, None if dm.s is None else dm.s * mask)
    t = [_conv(_conv(dm[i], g, 2), g, 1) for i in range(3)]
    sgn = torch.sign(x.v - y.v) * rows[None, :, None]
    w_ssim, w_l1 = f32(w_ssim), f32(w_l1)
    inner = t[0] + (2.0 * x) * t[1] + y * t[2]
    sg = R(sgn, None, None if x.s is None else sgn.float())
    d = inner * w_ssim + sg * w_l1
    if upstream is not None:
        d = d * f32(upstream)
    return d


# ---- normal consistency --------------------------------------------------------------------------------------------------

def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def normal_consistency(normal, map_e, map_m, from_depth, inv_fx, inv_fy, cx, cy, w_e, w_m, shadow=False, device="cpu") -> dict:
    """normal [3,H,W]; map_e, map_m [1,H,W] depths (from_depth) or [3,H,W] coordinates; fp32 camera constants and weights as the
    kernel receives them.  Returns loss (value, bound), d_normal [3,H,W], d_e, d_m ([1,H,W] or [3,H,W]) as R, and
    `ambiguous` [2,H,W], the stencils whose `len > 1e-12` decision the fp32 length may flip."""
    H, W = normal.shape[-2:]
    N = [R.input(normal[i], shadow, device) for i in range(3)]
    inv_fx, inv_fy, cx, cy, w_e, w_m = (f32(v) for v in (inv_fx, inv_fy, cx, cy, w_e, w_m))
    gx = R.input(torch.arange(W, dtype=torch.float32).expand(H, W), shadow, device)
    gy = R.input(torch.arange(H, dtype=torch.float32)[:, None].expand(H, W), shadow, device)
    if from_depth:
        rx = (gx + 0.5) * inv_fx + cx
        ry = (gy + 0.5) * inv_fy + cy
    pts = []
    for m in (map_e, map_m):
        if from_depth:
            d = R.input(m.reshape(H, W), shadow, device)
            pts.append([d * rx, d * ry, d])
        else:
            pts.append([R.input(m.reshape(3, H, W)[i], shadow, device) for i in range(3)])
    dev = N[0].v.device
    interior = torch.zeros(H, W, dtype=torch.bool, device=dev)
    interior[1:H - 1, 1:W - 1] = True

    def sh(r: R, dr, dc):
        """out[i, j] = r[i + dr, j + dc], zero outside."""
        out = _shift(r, SR + dr, 0)
        return _shift(out, SR + dc, 1)

    loss_terms, dn, grads, amb = [], None, [], []
    for k, w in ((0, w_e), (1, w_m)):
        P = pts[k]
        dx = [sh(p, 1, 0) - sh(p, -1, 0) for p in P]
        dy = [sh(p, 0, 1) - sh(p, 0, -1) for p in P]
        cr = _cross(dx, dy)
        ln = _dot(cr, cr).sqrt()
        den = ln.maximum(NORM_EPS)
        n = [c / den for c in cr]
        nr = _dot(n, N)
        term = (1.0 - nr) * w
        loss_terms.append(term.where(interior, w))
        dn_k = [(nn * w).where(interior, 0.0) for nn in n]
        dn = dn_k if dn is None else [a + b for a, b in zip(dn, dn_k)]
        through = [(N[i] - n[i] * nr) * (-w) / den for i in range(3)]
        clamped = [N[i] * (-w) / den for i in range(3)]
        above = ln.v > NORM_EPS
        a = interior & ((ln.v - NORM_EPS).abs() <= ln.e)
        amb.append(a)
        gc = []
        for t, c in zip(through, clamped):
            p, q = t.where(above, c), c.where(above, t)
            # an ambiguous stencil admits both branches: centre and half-width of the two outcomes on top of their bounds
            both = R((p.v + q.v) / 2, (p.v - q.v).abs() / 2 + torch.maximum(p.e, q.e), None if p.s is None else p.s)
            gc.append(p.where(~a, both).where(interior, 0.0))
        gdx = [c.where(interior, 0.0) for c in _cross(dy, gc)]
        gdy = [c.where(interior, 0.0) for c in _cross(gc, dx)]
        # a pixel is the +row neighbour of the stencil a row up and the -row one of the stencil a row down (columns alike)
        gpt = [((sh(gdx[i], -1, 0) - sh(gdx[i], 1, 0)) + sh(gdy[i], 0, -1)) - sh(gdy[i], 0, 1) for i in range(3)]
        grads.append(stack([(gpt[0] * rx + gpt[1] * ry) + gpt[2]], 0) if from_depth else stack(gpt, 0))
    d_normal = stack([-x for x in dn], 0)
    tot = loss_terms[0] + loss_terms[1]
    ones = torch.ones(H, W, dtype=torch.bool, device=dev)
    loss = _sum_bound(tot, ones)
    return {"loss": loss, "d_normal": d_normal, "d_e": grads[0], "d_m": grads[1], "ambiguous": torch.stack(amb), "interior": interior}
