"""The exchange model (tests/exchange_model.py) on hand-computed cases: what the peer gradient exchange may return."""
import numpy as np

import exchange_model as em

NAN = em.f32(em.CANONICAL_NAN)
TINY = np.float32(2.0 ** -126)          # smallest normal
SUB = np.float32(2.0 ** -130)           # a subnormal


def _rows(*per_rank):
    """One row of four floats per rank, every rank touching it -> (rows [W, 1, 4], touched [W, 1])."""
    rows = np.array([[list(r)] for r in per_rank], np.float32)
    return rows, np.ones(rows.shape[:2], np.int32)


def _values(adm):
    """The admissible values of element 0 of row 0 as a set of bit patterns."""
    return set(int(b) for b in adm[:, 0, 0])


def test_world2_is_one_rounded_sum_in_either_order():
    rng = np.random.default_rng(1)
    a = (rng.standard_normal(4096) * 10.0 ** rng.integers(-20, 20, 4096)).astype(np.float32)
    b = (rng.standard_normal(4096) * 10.0 ** rng.integers(-20, 20, 4096)).astype(np.float32)
    rows = np.stack([a.reshape(-1, 4), b.reshape(-1, 4)])
    adm = em.admissible(rows, np.ones((2, rows.shape[1]), np.int32))
    assert adm.shape[0] == 2
    assert np.array_equal(adm[0], adm[1])                    # fl(a + b) == fl(b + a)
    assert np.array_equal(adm[0], em.bits((a + b).reshape(-1, 4)))
    assert not em.multi_admissible(adm).any()


def test_three_rank_cancellation_admits_zero_and_one():
    rows, touched = _rows((1e8, 0, 0, 0), (1, 0, 0, 0), (-1e8, 0, 0, 0))
    adm = em.admissible(rows, touched)
    assert adm.shape[0] == 6
    assert _values(adm) == {int(em.bits(np.float32(0.0))), int(em.bits(np.float32(1.0)))}
    assert em.multi_admissible(adm)[0, 0] and not em.multi_admissible(adm)[0, 1:].any()
    # every permutation is counted: 1 vanishes beside 1e8 unless the two 1e8 cancel first
    vals = em.f32(adm[:, 0, 0])
    assert sorted(vals.tolist()) == [0.0, 0.0, 0.0, 0.0, 1.0, 1.0]


def test_exact_cancellation_is_positive_zero():
    rows, touched = _rows((3.5, -2.0, 0, 0), (-3.5, 2.0, 0, 0))
    adm = em.admissible(rows, touched)
    assert (adm[:, 0, :] == 0).all()                         # +0.0 bits, not -0.0


def test_negative_zero_quarter_is_not_pushed_and_reads_positive_zero():
    rows, touched = _rows((-0.0, -0.0, -0.0, -0.0), (-0.0, -0.0, -0.0, -0.0))
    assert not em.pushed_quarters(rows, touched).any()
    adm = em.admissible(rows, touched)
    assert (adm == 0).all()
    # -0.0 beside a non-zero element is pushed and adds to +0.0: +0.0
    rows, touched = _rows((-0.0, 1.0, 0, 0), (-0.0, 0, 0, 0))
    assert em.pushed_quarters(rows, touched)[:, 0, 0].tolist() == [True, False]
    adm = em.admissible(rows, touched)
    assert (adm[:, 0, 0] == 0).all() and (em.f32(adm[:, 0, 1]) == 1.0).all()


def test_untouched_rows_are_not_pushed_whatever_they_hold():
    rows = np.array([[[1, 2, 3, 4]], [[5, 6, 7, 8]]], np.float32)
    touched = np.array([[1], [0]], np.int32)
    adm = em.admissible(rows, touched)
    assert (em.f32(adm[:, 0]) == rows[0, 0]).all()
    acc = em.accumulator_after(rows, touched)
    assert (em.bits(acc[0]) == 0).all() and np.array_equal(acc[1], rows[1])


def test_nan_counts_as_non_zero_and_propagates():
    rows, touched = _rows((NAN, 0, 0, 0), (1.0, 0, 0, 0))
    assert em.pushed_quarters(rows, touched).all()
    adm = em.admissible(rows, touched)
    assert _values(adm) == {int(em.CANONICAL_NAN)}
    rows, touched = _rows((NAN, 0, 0, 0), (0, 0, 0, 0))       # rank 1's quarter is zero: not pushed
    assert _values(em.admissible(rows, touched)) == {int(em.CANONICAL_NAN)}


def test_infinities():
    inf = np.float32(np.inf)
    rows, touched = _rows((inf, -inf, inf, 1.0), (5.0, 7.0, -inf, -inf))
    adm = em.admissible(rows, touched)
    assert (em.f32(adm[:, 0, 0]) == inf).all()
    assert (em.f32(adm[:, 0, 1]) == -inf).all()
    assert (adm[:, 0, 2] == em.CANONICAL_NAN).all()          # Inf + -Inf: the canonical NaN
    assert (em.f32(adm[:, 0, 3]) == -inf).all()
    # overflow of two finite values rounds to Inf
    big = np.float32(3e38)
    rows, touched = _rows((big, 0, 0, 0), (big, 0, 0, 0))
    assert (em.f32(em.admissible(rows, touched)[:, 0, 0]) == inf).all()


def test_subnormal_inputs_are_flushed_keeping_their_sign():
    # a quarter of subnormals only is pushed (it is not == 0) but adds zeros
    rows, touched = _rows((SUB, -SUB, 0, 0), (SUB, 0, 0, 0))
    assert em.pushed_quarters(rows, touched).all()
    adm = em.admissible(rows, touched)
    assert (adm[:, 0, :] == 0).all()                         # +0.0 + +0.0, +0.0 + -0.0: +0.0
    # a subnormal beside a normal value vanishes: 1 + SUB == 1 anyway, TINY + SUB would not be TINY without the flush
    rows, touched = _rows((TINY, 0, 0, 0), (SUB, 0, 0, 0))
    assert _values(em.admissible(rows, touched)) == {int(em.bits(TINY))}


def test_subnormal_results_are_flushed_keeping_their_sign():
    # -1.5 * 2^-126 + 2^-126 = -2^-127: subnormal, flushed to -0.0 in both orders
    rows, touched = _rows((-1.5 * TINY, 1.5 * TINY, 0, 0), (TINY, -TINY, 0, 0))
    adm = em.admissible(rows, touched)
    assert (adm[:, 0, 0] == 0x80000000).all()
    assert (adm[:, 0, 1] == 0).all()
    # the flush makes the order show where exact arithmetic would not: T - 1.5T + T is 0.5T in every order without it;
    # with it, (T - 1.5T) flushes to -0.0 and + T gives T, while (T + T) - 1.5T = 0.5T flushes to +0.0
    rows, touched = _rows((TINY, 0, 0, 0), (-1.5 * TINY, 0, 0, 0), (TINY, 0, 0, 0))
    adm = em.admissible(rows, touched)
    assert _values(adm) == {0, int(em.bits(TINY))}
    assert int((adm[:, 0, 0] == 0).sum()) == 2                # the orders that add the two +T first


def test_flush_and_fold_primitives():
    x = np.array([SUB, -SUB, TINY, -TINY, 0.0, -0.0, 1.0], np.float32)
    f = em.flush(x)
    assert em.bits(f).tolist() == [0, 0x80000000, int(em.bits(TINY)), int(em.bits(-TINY)), 0, 0x80000000, int(em.bits(np.float32(1)))]
    assert int(em.bits(em.red_add(np.float32(0.0), np.float32(-0.0)))) == 0
    assert int(em.bits(em.red_add(np.float32(-0.0), np.float32(-0.0)))) == 0x80000000


def test_accumulator_after_clears_pushed_quarters_to_positive_zero():
    rows = np.array([[[1, -0.0, 0, 0, -0.0, 0, -0.0, 0]], [[0, 0, 0, 0, 0, 0, 0, 0]]], np.float32)
    touched = np.ones((2, 1), np.int32)
    acc = em.accumulator_after(rows, touched)
    assert (em.bits(acc[0, 0, :4]) == 0).all()              # pushed: cleared to +0.0
    assert em.bits(acc[0, 0, 4:]).tolist() == [0x80000000, 0, 0x80000000, 0]   # not pushed: left as it was
    assert (acc == 0).all()


def test_world4_enumerates_24_orders():
    rows, touched = _rows((1e8, 0, 0, 0), (1, 0, 0, 0), (-1e8, 0, 0, 0), (0.5, 0, 0, 0))
    adm = em.admissible(rows, touched)
    assert adm.shape[0] == 24
    vals = set(em.f32(adm[:, 0, 0]).tolist())
    assert vals == {0.0, 0.5, 1.0, 1.5}
