"""CPU checks of tests/tc_guard_cases.py: the operand mirror against DESIGN.md 3.2's closed form and the A/B tool, the
hi / lo split, and the exact family's exactness and planted ratios."""
from fractions import Fraction

import numpy as np
import pytest

from tests import tc_guard_cases as tg

U = 2.0**-24


@pytest.mark.parametrize("F", range(1, 65))
def test_kappa_closed_form(F):
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
    from ab_linear_tc import thresholds

    ops = tg.operands(np.ones((3, F)), np.ones(3))
    f_pad = 32 if F <= 32 else 64
    thr = float(np.float32(2 * (F + 4) * U * (1 + F * 2.0**-21) * 1.0001))
    step = 64 * U * f_pad / 16
    e_rel = (2.0**-21 + step * (1 + 2.0**-10) + 4 * U) * (1 + 2.0**-10)
    kappa = float(np.float32((2 * e_rel + 2.5 * thr * (1 + (F + 2) * U)) / (1 - step) * (1 + 2.0**-10)))
    assert (ops.thr, ops.step, ops.e_rel, ops.kappa) == (thr, step, e_rel, kappa)
    t_thr, t_kappa = thresholds(F)
    assert t_thr == thr and float(np.float32(t_kappa)) == kappa


@pytest.mark.parametrize("seed", range(6))
def test_hi_lo_split_is_exact_up_to_its_remainder(seed):
    """hi + lo + remainder = the scaled weight exactly; the remainder is within 2^-22 |v| + 2^-25 (DESIGN.md 3.2)."""
    rng = np.random.default_rng(seed)
    W, b = tg.rounding_model(64, 10, rng)
    ops = tg.operands(W, b)
    for c in range(ops.C):
        for f in range(0, 64, 3):
            v = Fraction(float(np.ldexp(ops.W[c, f], ops.sigma)))
            hi, lo = Fraction(ops.hi[c, f]), Fraction(ops.lo[c, f])
            rem = v - hi - lo
            assert hi + lo + rem == v
            assert abs(rem) <= Fraction(2.0**-22) * abs(v) + Fraction(2.0**-25)
            assert abs(rem) <= Fraction(2.0**-22) * Fraction(ops.wb[f])
            assert float(hi) == float(np.float16(hi)) and float(lo) == float(np.float16(lo))


def test_binary_layout_is_expanded():
    ops = tg.operands(np.array([[0.5, -2.0]]), np.array([0.25]))
    assert ops.C == 2 and np.all(ops.W[0] == 0) and ops.b[0] == 0 and ops.tb[1] == np.float32(0.25 * 2.0**ops.sigma)


@pytest.mark.parametrize("F,C", [(1, 2), (1, 16), (16, 3), (33, 9), (64, 8), (64, 16)])
def test_exact_family_is_exact_and_on_its_rungs(F, C):
    parts = tg.exact_family(F, C, seed=7000 + 97 * F + C)
    rungs = []
    for coef, intercept, X in parts:
        ops = tg.operands(coef, intercept)
        assert ops.sigma == tg.SIGMA and ops.eligible
        for x in X:  # a row of lo features on the grid of 1/4, a row of hi features on the grid of 8
            assert tg.exact_column_bound_ok(ops, x[None], 0.25) or tg.exact_column_bound_ok(ops, x[None], 8.0), x
        labels, margins = tg.truth(X, coef, intercept)
        lab_x, m_x = tg.exact_linear(X[:20], coef, intercept)
        assert np.array_equal(labels[:20], lab_x) and np.array_equal(margins[:20], m_x)
        rung = tg.rung_of(ops, X, margins)
        assert not np.isnan(rung).any()
        rungs.append(rung)
    rungs = np.concatenate(rungs)
    for r in tg.RUNGS:
        assert (rungs == r).sum() >= (4 if F == 1 else 12), (r, np.unique(rungs, return_counts=True))


def test_rounding_family_populates_every_verdict():
    seen = np.zeros(3, int)
    for F, C in ((16, 9), (33, 16), (64, 3)):
        for route in ("byte", "half"):
            rng = np.random.default_rng(F + C)
            W, b = tg.rounding_model(F, C, rng)
            X = tg.rounding_rows(F, rng, 3001, route)
            ops = tg.operands(W, b)
            assert ops.eligible
            _, m = tg.truth(X, W, b)
            seen += np.bincount(tg.verdicts(ops, X, m) + 1, minlength=3)
    assert np.all(seen > 0), seen


def test_lossy_case_differs_from_its_cast():
    W, b, X = tg.lossy_case(16, 3, np.random.default_rng(0), 500)
    exact, _ = tg.truth(X, W, b)
    cast, _ = tg.truth(X.astype(np.float32), W, b)
    assert (exact != cast).sum() > 0 and np.all(X.astype(np.float32) == np.rint(X.astype(np.float32)))
