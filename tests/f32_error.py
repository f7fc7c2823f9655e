"""Running error analysis of an fp32 expression, evaluated in fp64 torch.

`R` holds, for one expression over fp32 inputs, its exact value `v` (fp64, to fp64 rounding) and a rigorous bound `e` on how
far an fp32 evaluation of the same operations, in the same order, may land from `v`: every +, -, *, / and fma rounds once
to nearest (an fma is bounded as a product and a sum, which covers both the fused and the separate form), every result may
be subnormal (an absolute ETA per operation), `expf` is within 2 ulp and `sqrtf` within 1 ulp.  Errors of the operands are
carried to first order *and* their products, so the bound holds for any operand error within the operands' bounds.

With `shadow=True` every operation is also evaluated in torch fp32 (`s`), rounded after every step as the kernels do: the
host tests check `|s - v| <= e` at every element, i.e. that the bounds admit an actual fp32 evaluation.

The comparison helpers take `slack` for the fp64 model's own rounding: the bounds are >= 2^-24 |v| wherever a rounding
happened, so a relative 1e-6 of the bound covers fp64 rounding (2^-53) with room to spare.
"""
from __future__ import annotations

import numpy as np
import torch

U = 2.0 ** -24        # unit roundoff of fp32, round to nearest
ETA = 2.0 ** -150     # half the spacing of the fp32 subnormals: the absolute error of a rounding in the subnormal range
K_EXP = 4.0           # expf: 2 ulp, and an ulp is <= 2u |v|
K_SQRT = 2.0          # sqrtf: IEEE on the GPU; torch's vectorised CPU sqrt is within 1 ulp
SLACK = 1e-6


def f32(x) -> float:
    """A Python/fp64 constant as the kernels see it (an fp32 literal)."""
    return float(np.float32(x))


def _rnd(v, d):
    return U * (v.abs() + d) + ETA


class R:
    __slots__ = ("v", "e", "s")

    def __init__(self, v, e=None, s=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e
        self.s = s

    # ---- construction ----------------------------------------------------------------------------------------------------
    @staticmethod
    def input(x, shadow=False, device=None):
        """An fp32 input: exact."""
        t = torch.as_tensor(x)
        if device is not None:
            t = t.to(device)
        t32 = t.to(torch.float32)
        return R(t32.double(), None, t32.clone() if shadow else None)

    def const(self, c):
        """The fp32 constant c broadcast like self."""
        c = f32(c)
        return R(torch.full_like(self.v, c), None, None if self.s is None else torch.full_like(self.s, c))

    @property
    def shadow(self):
        return self.s is not None

    def _sh(self, other):
        return other.s if isinstance(other, R) else None

    # ---- arithmetic --------------------------------------------------------------------------------------------------------
    def _lift(self, o):
        return o if isinstance(o, R) else self.const(o)

    def __add__(self, o):
        o = self._lift(o)
        v = self.v + o.v
        d = self.e + o.e
        return R(v, d + _rnd(v, d), None if self.s is None else self.s + o.s)

    __radd__ = __add__

    def __neg__(self):
        return R(-self.v, self.e, None if self.s is None else -self.s)

    def __sub__(self, o):
        return self + (-self._lift(o))

    def __rsub__(self, o):
        return self._lift(o) - self

    def __mul__(self, o):
        o = self._lift(o)
        v = self.v * o.v
        d = self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e
        return R(v, d + _rnd(v, d), None if self.s is None else self.s * o.s)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = self._lift(o)
        v = self.v / o.v
        den = o.v.abs() - o.e
        d = torch.where(den > 0, (self.e + v.abs() * o.e) / den.clamp_min(1e-300), torch.full_like(v, float("inf")))  # no claim
        return R(v, d + _rnd(v, d), None if self.s is None else self.s / o.s)

    def __rtruediv__(self, o):
        return self._lift(o) / self

    def fma(self, b, c):
        """fmaf(self, b, c)."""
        b, c = self._lift(b), self._lift(c)
        out = self * b + c
        if self.s is not None:
            out.s = (self.s.double() * b.s.double() + c.s.double()).float()  # the product of two fp32 is exact in fp64
        return out

    def exp(self):
        v = torch.exp(self.v)
        d = v * torch.expm1(self.e)
        return R(v, d + K_EXP * U * (v + d) + ETA, None if self.s is None else torch.exp(self.s))

    def sqrt(self):
        v = torch.sqrt(self.v.clamp_min(0))
        d = torch.minimum(torch.sqrt(self.e), self.e / v.clamp_min(1e-300))
        return R(v, d + K_SQRT * U * (v + d) + ETA, None if self.s is None else torch.sqrt(self.s))

    def abs(self):
        return R(self.v.abs(), self.e, None if self.s is None else self.s.abs())

    def maximum(self, c):
        """fmaxf(self, c) for an fp32 constant c: 1-Lipschitz."""
        c = f32(c)
        return R(self.v.clamp_min(c), self.e, None if self.s is None else self.s.clamp_min(c))

    def where(self, mask, other):
        other = self._lift(other)
        return R(torch.where(mask, self.v, other.v), torch.where(mask, self.e, other.e),
                 None if self.s is None else torch.where(mask, self.s, other.s))

    def __getitem__(self, idx):
        return R(self.v[idx], self.e[idx], None if self.s is None else self.s[idx])

    def widen(self, extra):
        """The bound plus an allowance the rounding model does not describe (stated where it is used)."""
        return R(self.v, self.e + extra, self.s)


def stack(rs, dim):
    return R(torch.stack([r.v for r in rs], dim), torch.stack([r.e for r in rs], dim),
             None if rs[0].s is None else torch.stack([r.s for r in rs], dim))


def excess(given, r: R, slack=SLACK):
    """|given - v| / bound per element (<= 1 passes); a zero bound with an exact match is 0, with a mismatch inf."""
    g = torch.as_tensor(given).to(r.v.device).double()
    err = (g - r.v).abs()
    bound = r.e * (1 + slack)
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, float("inf"))))
    return torch.where(torch.isnan(g) | torch.isnan(r.v), torch.full_like(err, float("inf")), ratio)


def check(given, r: R, name, max_report=6) -> float:
    """Every element of `given` within its bound; returns the worst error/bound ratio."""
    x = excess(given, r)
    bad = torch.nonzero(~(x <= 1.0))
    if bad.numel():
        g = torch.as_tensor(given).to(r.v.device).double()
        rows = [f"  at {tuple(i.tolist())}: got {g[tuple(i)].item():.9g}, fp64 {r.v[tuple(i)].item():.9g}, bound {r.e[tuple(i)].item():.3g}"
                for i in bad[:max_report]]
        raise AssertionError(f"{name}: {bad.shape[0]} of {x.numel()} elements outside their bound\n" + "\n".join(rows))
    return float(x.max()) if x.numel() else 0.0


def check_shadow(r: R, name) -> float:
    """The fp32 shadow evaluation lies within the bound at every element."""
    return check(r.s, r, name + " (fp32 evaluation)")
