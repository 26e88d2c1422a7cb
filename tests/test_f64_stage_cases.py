"""CPU checks of the constructions in tests/f64_stage_cases.py: the planted rows sit where the margin ladder says, the
underflow construction is what float64 gets wrong, and the greedy mean makes a plain sequential scaler fold (replayed
in numpy scalar operations) drift far outside the float64 bound.  A broken construction then shows up without a GPU."""
from fractions import Fraction

import numpy as np
import pytest

from tests import f64_stage_cases as K


@pytest.mark.parametrize("F,C,binary", [(32, 10, False), (65, 16, False), (1, 2, True), (48, 40, False)])
def test_ladder_rows_sit_on_the_ladder(F, C, binary):
    rng = np.random.default_rng(F + C)
    dups = [] if binary else [(0, C - 1)]
    coef, intercept, tune = K.ladder_model(F, C, rng, dups=dups, binary=binary)
    tops = [(1, 0)] * 4 if binary else [(1, 2)] * 4 + [(0, C - 1)] * 2
    state = rng.bit_generator.state
    X0 = K.ladder_rows(rng, coef, intercept, tune, tops, [0.0] * len(tops))
    beta = K.linear_beta(X0, coef, intercept)
    rng.bit_generator.state = state  # the same body features again, now with the margins set
    ks = [0.1, 0.5, 5.0, 50.0] + ([0.0, 0.0] if not binary else [])
    X = K.ladder_rows(rng, coef, intercept, tune, tops, [k * b for k, b in zip(ks, beta)])
    want, margin = K.exact_linear(X, coef, intercept)
    beta = K.linear_beta(X, coef, intercept)
    # each tuning value rounds once (<= u |score terms| <= beta / 16 per score), so a margin sits within beta / 8
    assert np.all(np.abs(margin[:4] / beta[:4] - ks[:4]) <= 0.125 + 0.02 * np.array(ks[:4])), margin[:4] / beta[:4]
    assert (want[:4] == [t[0] for t in tops[:4]]).all()
    if not binary:
        assert (margin[4:] == 0).all() and (want[4:] == 0).all()  # duplicate classes: exact ties, first index
    # heavy cancellation: each score is far smaller than the terms it sums
    terms = np.abs(X) @ np.abs(np.atleast_2d(coef)).T
    assert terms.max() > 2.0**30 * beta.max()
    certain, inside, straddle = K.rungs(margin, beta)
    assert set(inside) >= {0} and set(certain) >= {2, 3} and 1 in straddle


def test_int32_anchor_lets_the_ladder_reach_inside_beta():
    rng = np.random.default_rng(2)
    coef, intercept, tune = K.ladder_model(24, 5, rng, dups=[(0, 4)], wexp=(-26, -12), anchor=2.0**30)
    tops = [(1, 2)] * 3
    state = rng.bit_generator.state
    X0 = K.ladder_rows(rng, coef, intercept, tune, tops, [0.0] * 3, kind="i32", anchor_x=2.0**30)
    beta = K.linear_beta(X0.astype(np.float64), coef, intercept)
    rng.bit_generator.state = state
    X = K.ladder_rows(rng, coef, intercept, tune, tops, [0.0, 0.5 * beta[1], 8 * beta[2]], kind="i32", anchor_x=2.0**30)
    assert X.dtype == np.int32 and (X[:, 0] == 2**30).all()
    want, margin = K.exact_linear(X.astype(np.float64), coef, intercept)
    beta = K.linear_beta(X.astype(np.float64), coef, intercept)
    certain, inside, straddle = K.rungs(margin, beta)
    assert list(inside) == [0] and list(straddle) == [1] and list(certain) == [2] and (want == 1).all()


def test_exact_integer_scores_match_fractions():
    rng = np.random.default_rng(3)
    coef, intercept = K.spread64(rng, (3, 5), -60, 60), K.spread64(rng, 3)
    x = K.spread64(rng, 5, -600, 300)
    want = [Fraction(float(intercept[c])) + sum(Fraction(float(v)) * Fraction(float(w)) for v, w in zip(x, coef[c]))
            for c in range(3)]
    assert K.exact_linear_scores(x, coef, intercept) == want


def test_int64_rows_round_to_the_values_the_truth_uses():
    rng = np.random.default_rng(1)
    coef, intercept, tune = K.ladder_model(24, 5, rng, wexp=(-22, -10))
    X = K.ladder_rows(rng, coef, intercept, tune, [(1, 2)] * 3, [1e3] * 3, kind="i64")
    assert X.dtype == np.int64 and (np.abs(X) > 2**53).any()
    assert (X.astype(np.float64).astype(np.int64) != X).any()  # lossy in float64, as scikit-learn sees them


@pytest.mark.parametrize("binary", [False, True])
def test_underflow_construction(binary):
    coef, intercept, x = K.underflow_case(binary)
    want, margin = K.label_margin(K.exact_linear_scores(x, coef, intercept))
    assert want == 1 and 0 < margin < Fraction(2.0**-1074)
    # float64 with a lane per feature: each product rounds to 2^-1074 on its own, then the lanes are added
    prods = [np.float64(x[f]) * coef[:, f] for f in range(3)]
    s = np.sum(prods, axis=0)
    got = (1 if s[0] > 0 else 0) if binary else int(np.argmax(s))
    assert got == 0  # the wrong label, which the relative-only bound certified
    assert K.linear_beta(x[None, :], coef, intercept)[0] >= 16 * 2.0**-1074


def test_sequential_fold_replay_and_greedy_mean():
    mean, scale, coef, intercept = K.fold_model(F=200, seed=2)
    wsc = coef[0] * (1.0 / scale)
    replay = K.sequential_fold(mean, wsc, intercept[0])
    exact = Fraction(float(intercept[0])) - sum(Fraction(float(m)) * Fraction(float(w)) for m, w in zip(mean, wsc))
    # the greedy mean makes every step round the same way: the sequential sum drifts far beyond one rounding
    drift = Fraction(replay) - exact
    assert drift > 0
    assert float(drift) > 20 * abs(replay) * K.U
    # and beyond the fp64 bound of an unfolded model of the same size, which is what made the old fold unsound
    assert float(drift) > 2 * (200 / 32 + 8) * K.U * 2 * abs(replay) * 0.25


def test_fold_rows_sit_on_the_ladder():
    mean, scale, coef, intercept = K.fold_model(F=64, seed=3)
    rng = np.random.default_rng(4)
    sc, X1 = K.fold_rows(rng, mean, scale, coef, intercept, [1.0])
    beta = float(K.fold_beta(sc, X1, coef, intercept)[0])  # about the same for every row: x ~ mean_
    ks = [0.1, -0.1, 3.0, -8.0]
    sc, X = K.fold_rows(rng, mean, scale, coef, intercept, [k * beta for k in ks])
    want, margin = K.fold_truth(sc, X, coef, intercept)
    assert np.allclose(margin / beta, np.abs(ks), rtol=0.05)
    assert (want == [0, 1, 0, 1]).all()


def test_mlp_beta_is_dominated_by_cancelling_hidden_unit():
    F, H, C = 32, 16, 3
    w1 = np.zeros((H, F), np.float32)
    w1[0, :3] = [1, -1, 1]
    w2 = np.zeros((C, H), np.float32)
    w2[0, 0] = 1
    x = np.zeros((1, F), np.float32)
    x[0, :3] = [2.0**20, 2.0**20, 2.0**-25]
    b1, b2 = np.zeros(H, np.float32), np.array([0, 2.0**-25, -1], np.float32)
    beta = K.mlp_beta(x, w1, b1, w2, b2)[0]
    herr_part = 2 * (F + 6) * K.U * (2.0**21 + 2.0**-25)
    assert herr_part < beta < 1.01 * herr_part
    want, margin = K.exact_mlp(x, w1, b1, w2, b2)
    assert want[0] in (0, 1) and margin[0] == 0  # h0 = 2^-25 = b2_1: an exact tie, class 0 first
