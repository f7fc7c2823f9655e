"""What one step of the peer gradient exchange (csrc/rgs_exchange.cu) may return, as a numpy model.

The contract (the comment at the top of rgs_exchange.cu, include/rgs_b200.h above `rgs_exchange_create`):
  * rank r pushes the 16-byte quarter q of row i when `tiles_touched[i] != 0` on r and some element of the quarter is not
    `== 0` (NaN counts as non-zero, -0.0 does not);
  * the owner's `sum` starts the step at +0.0 and every pushing rank adds its quarter with one fp32 round-to-nearest
    `red.add` per element, in an order across ranks the hardware chooses -- per element, not per row;
  * `red.add.f32` flushes subnormal inputs and results to sign-preserving zero (PTX ISA, `red` semantics);
  * every rank ends with the same bits: the owner's sum, spread everywhere.
So an element's admissible set is the fp32 left fold from +0.0, with that flush, over every permutation of the ranks that
pushed its quarter.  The set does not depend on earlier steps: a row pushed last step and not now, or any row after P
changed, reads exactly +0.0.  Each rank's accumulator is zero after the step, and +0.0 bits in every quarter it pushed.

NaN results are the canonical NaN 0x7fffffff the GPU's float adds produce; callers feed NaN inputs with those same bits.
"""
from __future__ import annotations

import itertools

import numpy as np

CANONICAL_NAN = np.uint32(0x7FFFFFFF)
_MIN_NORMAL = np.float32(2.0 ** -126)


def f32(bits) -> np.ndarray:
    return np.asarray(bits, np.uint32).view(np.float32)


def bits(x) -> np.ndarray:
    return np.asarray(x, np.float32).view(np.uint32)


def flush(x: np.ndarray) -> np.ndarray:
    """Subnormals to the zero of their sign; everything else unchanged (bits included)."""
    x = np.asarray(x, np.float32)
    sub = (x != 0) & (np.abs(x) < _MIN_NORMAL)
    return np.where(sub, np.copysign(np.float32(0), x), x).astype(np.float32)


def red_add(acc: np.ndarray, v: np.ndarray) -> np.ndarray:
    """One `red.add.f32`: flushed inputs, round-to-nearest sum, flushed result, canonical NaN."""
    with np.errstate(invalid="ignore", over="ignore"):
        s = flush(flush(acc) + flush(v))
    return np.where(np.isnan(s), f32(CANONICAL_NAN), s).astype(np.float32)


def pushed_quarters(rows: np.ndarray, touched: np.ndarray) -> np.ndarray:
    """[..., P, F] rows and [..., P] touched -> [..., P, F/4] bool: this quarter goes to its owner."""
    rows = np.asarray(rows, np.float32)
    q = rows.reshape(rows.shape[:-1] + (rows.shape[-1] // 4, 4))
    return (q != 0).any(-1) & (np.asarray(touched) != 0)[..., None]


def admissible(rows: np.ndarray, touched: np.ndarray) -> np.ndarray:
    """rows [W, P, F] float32 (what each rank's accumulator held), touched [W, P] -> [W!, P, F] uint32: the result bits each
    permutation of the ranks produces, element by element.  Any element may take any of its permutations' values."""
    rows = np.asarray(rows, np.float32)
    W, P, F = rows.shape
    push = np.repeat(pushed_quarters(rows, touched), 4, axis=-1)   # [W, P, F]
    out = []
    for perm in itertools.permutations(range(W)):
        acc = np.zeros((P, F), np.float32)
        for r in perm:
            acc = np.where(push[r], red_add(acc, rows[r]), acc)
        out.append(bits(acc))
    return np.stack(out)


def check_result(result: np.ndarray, adm: np.ndarray) -> np.ndarray:
    """[P, F] bool: the result's bits are one of the element's admissible values."""
    return (adm == bits(result)[None]).any(0)


def multi_admissible(adm: np.ndarray) -> np.ndarray:
    """[P, F] bool: the element has more than one admissible value (the order across ranks can show)."""
    return (adm != adm[:1]).any(0)


def accumulator_after(rows: np.ndarray, touched: np.ndarray) -> np.ndarray:
    """[W, P, F] float32: each rank's accumulator after the step -- +0.0 in every pushed quarter, the rest as it was (zero:
    only the -0.0 of quarters that were not pushed may remain)."""
    rows = np.asarray(rows, np.float32)
    push = np.repeat(pushed_quarters(rows, touched), 4, axis=-1)
    return np.where(push, np.float32(0), rows).astype(np.float32)
