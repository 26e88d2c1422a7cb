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


# ---------------------------------------------------------------------------------------------------------------
# top-k: the exact reference of the MLP ranks and the rank ladder of tests/test_gpu_mlp_topk_exactness.py
# ---------------------------------------------------------------------------------------------------------------
def test_topk_gap_orders_ties_by_lower_index():
    z = [Fraction(1), Fraction(3), Fraction(1), Fraction(3), Fraction(-2)]
    assert K.topk_gap(z, 1) == ([1], 0)  # 1 and 3 tie at the top: the lower index first, gap 0
    assert K.topk_gap(z, 3) == ([1, 3, 0], 0)
    assert K.topk_gap([Fraction(5), Fraction(1), Fraction(0)], 3) == ([0, 1, 2], 1)  # k == C: the gaps of ranks 1 .. C
    assert K.topk_gap([Fraction(5), Fraction(1), Fraction(0)], 1) == ([0], 4)
    assert list(np.argsort(-np.array([1.0, 3.0, 1.0, 3.0, -2.0]), kind="stable")) == [1, 3, 0, 2, 4]


@pytest.mark.parametrize("F,H,C,r,tie,big", [(64, 32, 10, 1, False, False), (64, 32, 10, 4, True, False),
                                             (50, 16, 3, 2, False, False), (32, 16, 3, 1, True, False),
                                             (40, 24, 5, 3, False, True), (128, 32, 10, 9, False, False)])
def test_mlp_rank_case_plants_the_gap_at_rank_r(F, H, C, r, tie, big):
    net, X, fs, beta, (a, b, t) = K.mlp_rank_case(F, H, C, r, tie=tie, big=big, seed=F + r)
    assert not (X.view(np.uint32) & np.uint32(0x1FFF)).any()  # tf32 values
    if big:
        assert (X == np.rint(X)).all()  # integer rows: an int64 frame holds them exactly
    for k in range(1, C + 1):
        idx, gap = K.exact_mlp_topk(X, *net, k)
        ex = [K.topk_gap(K._exact_mlp_logits(x, *net), k) for x in X]  # Fractions on every row
        assert [list(i) for i in idx] == [e[0] for e in ex]
        np.testing.assert_array_equal(gap, [float(e[1]) for e in ex])
        if k < r:  # the planted boundary lies beyond rank k + 1: only the wide gaps count
            assert (gap > 32 * beta).all(), (k, gap / beta)
            continue
        ratio = gap / beta
        if tie:  # a and its copy t tie exactly (below b on the - rows); the lower index of the two comes first
            assert (gap[(fs >= 0) | (k > r)] == 0).all()
            np.testing.assert_allclose(ratio[(fs < 0) & (k == r)], -fs[(fs < 0) & (k == r)], atol=0.02)
            lo, hi = min(a, t), max(a, t)
            for row in idx:
                row = list(row)
                assert hi not in row or row.index(lo) < row.index(hi)
        else:
            # float64 is exact and x2 is a tf32 value: each gap lands within 2 % of beta of its rung
            np.testing.assert_allclose(ratio, np.abs(fs), atol=0.02)
            # a above b on the + rows, below it on the - rows, at ranks r and r + 1
            top = np.where(fs > 0, a, b)
            if k >= r:
                assert (idx[:, r - 1] == top).all()
            if k > r:
                assert (idx[:, r] == np.where(fs > 0, b, a)).all()
    if not tie:  # both rungs of the bound factor are there, on both sides of beta
        assert (np.abs(fs) < 1).sum() >= 4 and (np.abs(fs) > 1).sum() >= 4


def test_exact_mlp_topk_uses_float64_only_where_it_is_sure():
    """Random rows plus rows whose logits tie in float64 but not exactly: the mixed sweep equals Fractions on every row."""
    rng = np.random.default_rng(6)
    F, H, C = 12, 8, 6
    w1 = K.spread64(rng, (H, F), -6, 6).astype(np.float32)
    b1 = K.spread64(rng, H, -6, 6).astype(np.float32)
    w2 = K.spread64(rng, (C, H), -6, 6).astype(np.float32)
    b2 = K.spread64(rng, C, -6, 6).astype(np.float32)
    w2[4], b2[4] = w2[1], b2[1]  # class 4 ties class 1 exactly
    # class 5 = h0 + 2^-40 against class 2 = h0: a gap far below float64's resolution of h0 ~ 2^40
    w1[0] = 0
    w1[0, 0] = 1.0
    w2[5], w2[2] = 0, 0
    w2[5, 0], w2[2, 0] = 1.0, 1.0
    b2[5], b2[2] = 2.0**-40, 0.0
    X = K.spread64(rng, (40, F), -6, 6).astype(np.float32)
    X[:20, 0] = 2.0**40
    for k in (1, 3, 6):
        idx, gap = K.exact_mlp_topk(X, w1, b1, w2, b2, k)
        ex = [K.topk_gap(K._exact_mlp_logits(x, w1, b1, w2, b2), k) for x in X]
        assert [list(i) for i in idx] == [e[0] for e in ex]
        bound = K.mlp_f64_bound(X, w1, b1, w2, b2)
        assert np.all(np.abs(gap - np.array([float(e[1]) for e in ex])) <= 2 * bound)
    z = X[:20].astype(np.float64)[:, 0]
    assert ((z + 2.0**-40) == z).all()  # float64 alone could not order classes 5 and 2 on these rows
