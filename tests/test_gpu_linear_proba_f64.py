"""Float64 class probabilities of the linear predictor (``uml_linear_predict_proba_f64*``,
``predictors.linear_predict_proba(..., dtype=np.float64)``, ``predictors.linear_predict_log_proba``).

Contract (DESIGN.md 3.9): from the float64 scores of 3.7, each within ``delta_c = ((F + 3) u + fold) a_c + (F + 3) 2^-1074``
of the exact score T_c, scikit-learn's formula in the same order gives

* multiclass: ``|p - p*| <= p* (e^K_c R - 1) + (C + 2) 2^-1074``, ``K_c = delta_c + max_k delta_k + 2 u L`` with
  ``L = max_k |s_k - m|``, ``R = (1 + 2u)(1 + u) / ((1 - 2u)(1 - gamma_{C-1}))``;
* binary ``p = expit(s)``: ``|p - p*| <= p* (e^delta (1 + 6u) - 1) + 2^-1022``, and the ``1 - p`` column
  ``|q - q*| <= B_p + u (q* + B_p)``;
* the logs: ``|l - l*| <= -ln(1 - r) + 2u (|l*| - ln(1 - r))`` with ``r = B / p*`` while ``r <= 1/2``; past that (a
  probability near DBL_TRUE_MIN, or ``1 - p`` near u) the probability's absolute bound is checked instead and the log
  must be the log of that probability.

``u = 2^-53``.  The exact values come from Fractions (the scores) and 60-digit decimals (exp / log).
"""
import math
from decimal import Decimal, localcontext
from fractions import Fraction
from typing import List

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

U = 2.0**-53
TRUE_MIN = 2.0**-1074
FOLD_REL = 8 * Fraction(1, 2**53)


@pytest.fixture(scope="module")
def eng():
    from unionml_b200.engine import get_engine

    return get_engine()


# ---- exact arithmetic ---------------------------------------------------------------------------------------------
def _fr(v) -> Fraction:
    return Fraction(int(v)) if isinstance(v, (int, np.integer)) else Fraction(float(v))


def _dec(f: Fraction) -> Decimal:
    return Decimal(f.numerator) / Decimal(f.denominator)


def exact_scores(X, W, b, bmag=None, fold=None, fold_rel=Fraction(0)):
    """Per row: (exact scores T_c, score bounds delta_c) of the caller's values X, both as Fractions.  W, b: the model
    the device scores (for a fold: w' and b', with fold = (mean_, scale_, coef_, intercept_)); bmag: bias magnitudes."""
    n, F = X.shape
    C = W.shape[0]
    Wf = [[_fr(W[c, f]) for f in range(F)] for c in range(C)]
    bm = [abs(_fr(v)) for v in b] if bmag is None else [_fr(v) for v in bmag]
    out = []
    for r in range(n):
        xr = [_fr(X[r, f]) for f in range(F)]
        if fold is not None:
            mean, scale, w0, b0 = fold
            z = [(xr[f] - _fr(mean[f])) / _fr(scale[f]) for f in range(F)]
        T, d = [], []
        for c in range(C):
            if fold is None:
                T.append(sum(xr[f] * Wf[c][f] for f in range(F)) + _fr(b[c]))
            else:
                T.append(sum(z[f] * _fr(w0[c, f]) for f in range(F)) + _fr(b0[c]))
            a = sum(abs(xr[f] * Wf[c][f]) for f in range(F)) + bm[c]
            d.append(((F + 3) * Fraction(1, 2**53) + fold_rel) * a + (F + 3) * Fraction(1, 2**1074))
        out.append((T, d))
    return out


def exact_proba_bounds(T, d, binary):
    """(p*, B) per column of one row, as Decimals: the exact probabilities and the 3.9 bound on the computed ones."""
    u = Decimal(U)
    if binary:
        s, delta = _dec(T[1]), _dec(d[1])
        p = 1 / (1 + (-s).exp())
        b1 = p * (delta.exp() * (1 + 6 * u) - 1) + Decimal(2.0**-1022)
        q = 1 - p
        return [q, p], [b1 + u * (q + b1), b1]
    C = len(T)
    Tm = max(T)
    dmax = max(d)
    L = _dec(Tm - min(T) + 2 * dmax)  # >= max_k |s_k - m| of the computed scores
    e = [_dec(t - Tm).exp() for t in T]
    S = sum(e)
    gamma = (C - 1) * u / (1 - (C - 1) * u)
    R = (1 + 2 * u) * (1 + u) / ((1 - 2 * u) * (1 - gamma))
    P, B = [], []
    for c in range(C):
        K = _dec(d[c] + dmax) + 2 * u * L
        p = e[c] / S
        P.append(p)
        B.append(p * (K.exp() * R - 1) + (C + 2) * Decimal(TRUE_MIN))
    return P, B


def check_exact(exact, got_p, got_lp, binary) -> List[str]:
    """Failures of the 3.9 bound for computed probabilities got_p and log-probabilities got_lp (n x C)."""
    fails = []
    u = Decimal(U)
    with localcontext() as ctx:
        ctx.prec = 60
        for r, (T, d) in enumerate(exact):
            P, B = exact_proba_bounds(T, d, binary)
            for c, (p, bnd) in enumerate(zip(P, B)):
                gp, gl = float(got_p[r, c]), float(got_lp[r, c])
                if not math.isfinite(gp) or abs(Decimal(gp) - p) > bnd:
                    fails.append(f"row {r} class {c}: p {gp!r}, exact {float(p)!r}, bound {float(bnd):.3g}")
                    continue
                rel = bnd / p if p > 0 else Decimal(1)
                if rel <= Decimal("0.5"):
                    lstar = p.ln()
                    lb = -(1 - rel).ln()
                    lb += 2 * u * (abs(lstar) + lb)
                    if not math.isfinite(gl) or abs(Decimal(gl) - lstar) > lb:
                        fails.append(f"row {r} class {c}: log {gl!r}, exact {float(lstar)!r}, bound {float(lb):.3g}")
                elif gp == 0.0:  # the relative bound says nothing here: the log is the log of the probability
                    if gl != -math.inf:
                        fails.append(f"row {r} class {c}: log {gl!r} of p = 0")
                elif abs(gl - math.log(gp)) > 4 * U * abs(math.log(gp)):
                    fails.append(f"row {r} class {c}: log {gl!r}, log of p {math.log(gp)!r}")
    return fails


def assert_rows_sum_to_one(got_p):
    C = got_p.shape[1]
    sums = np.array([math.fsum(row) for row in got_p])
    assert np.all(np.abs(sums - 1.0) <= (C + 2) * U), float(np.max(np.abs(sums - 1.0)))


def expanded(coef, intercept):
    """The model as the device stores it: a binary coef_ row becomes classes [0, s]."""
    coef = np.atleast_2d(np.asarray(coef, dtype=np.float64))
    intercept = np.atleast_1d(np.asarray(intercept, dtype=np.float64))
    if coef.shape[0] == 1:
        return np.vstack([np.zeros_like(coef), coef]), np.concatenate([[0.0], intercept])
    return coef, intercept


def planted_model(rng, C, F, binary=False):
    """Scores of a few units to a few tens: every probability, and most logs, carry information."""
    rows = 1 if binary else C
    return rng.standard_normal((rows, F)) * 0.3, rng.standard_normal(rows) * 2.0


def both(eng, dm, rows, **kw):
    """(probabilities, log-probabilities) of the host route."""
    return eng.predict_proba_f64_host(dm, rows, **kw)[0], eng.predict_proba_f64_host(dm, rows, log=True, **kw)[0]


def both_resident(eng, dm, batch):
    return eng.predict_proba_f64(dm, batch)[0], eng.predict_proba_f64(dm, batch, log=True)[0]


# ---- 1. against exact arithmetic, every row source ----------------------------------------------------------------
@pytest.mark.parametrize("binary", [False, True])
def test_exact_every_host_dtype_and_order(eng, binary):
    rng = np.random.default_rng(1)
    F, C = 33, 10
    coef, intercept = planted_model(rng, C, F, binary)
    coef /= 60  # features up to 200
    W, b = expanded(coef, intercept)
    dm = eng.load_linear(coef, intercept)
    base = rng.integers(0, 200, size=(64, F))
    for dt in (np.float64, np.float32, np.int64, np.int32, np.uint8):
        X = base.astype(dt)
        if dt in (np.float64, np.float32):
            X = (X - 100).astype(dt) * dt(0.37)
        exact = exact_scores(X, W, b)
        ref = None
        for order in ("C", "F"):
            p, lp = both(eng, dm, np.asarray(X, order=order))
            assert p.shape == (64, W.shape[0]) and p.dtype == np.float64, (dt, order)
            fails = check_exact(exact, p, lp, binary)
            assert not fails, (dt, order, fails[:5])
            assert_rows_sum_to_one(p)
            ref = p if ref is None else ref
            assert np.array_equal(p, ref), (dt, order)


@pytest.mark.parametrize("binary", [False, True])
def test_exact_resident_with_and_without_float64_copy(eng, binary):
    rng = np.random.default_rng(2)
    F, C = 65, 10
    coef, intercept = planted_model(rng, C, F, binary)
    W, b = expanded(coef, intercept)
    dm = eng.load_linear(coef, intercept)
    X = rng.standard_normal((64, F)) * 3 + rng.choice([-1e-9, 1e-9], size=(64, F))  # the fp32 cast is lossy
    b64 = eng.stage(X, keep_f64=True)
    p, lp = both_resident(eng, dm, b64)
    assert not check_exact(exact_scores(X, W, b), p, lp, binary)
    # a lossy batch without its float64 copy is refused: its fp32 rows are not the caller's values
    lossy = eng.stage(X, keep_f64=False)
    assert not lossy.lossless
    with pytest.raises(Exception, match="KEEP_F64|keep_f64|lossy"):
        eng.predict_proba_f64(dm, lossy)
    # fp32 rows that ARE the caller's values: no copy needed
    X32 = X.astype(np.float32)
    p, lp = both_resident(eng, dm, eng.stage(X32, keep_f64=False))
    assert not check_exact(exact_scores(X32, W, b), p, lp, binary)
    _, st = eng.predict_proba_f64(dm, b64, want_stats=True)
    assert st["path"] == 7


def test_exact_lossy_int64_frame(eng):
    rng = np.random.default_rng(3)
    F, C = 8, 3
    coef = rng.standard_normal((C, F)) * 2.0**-60
    intercept = rng.standard_normal(C)
    X = rng.integers(2**53, 2**62, size=(100, F), dtype=np.int64) * rng.choice([-1, 1], size=(100, F))
    X[::7, 0] = 2**53 + 1  # not a float64 value
    dm = eng.load_linear(coef, intercept)
    exact = exact_scores(X, coef, intercept)
    for name, (p, lp) in (("host C", both(eng, dm, X)), ("host F", both(eng, dm, np.asfortranarray(X))),
                          ("keep_f64", both_resident(eng, dm, eng.stage(X, keep_f64=True)))):
        fails = check_exact(exact, p, lp, False)
        assert not fails, (name, fails[:5])


def fold_operands(mean, scale_, coef, intercept):
    """w', b' magnitudes as uml_linear_set_affine computes them (sequential float64, no FMA contraction)."""
    sc = 1.0 / np.asarray(scale_, dtype=np.float64)
    w = coef * sc[None, :]
    bmag = []
    for c in range(coef.shape[0]):
        mag = abs(float(intercept[c]))
        for f in range(coef.shape[1]):
            mag += abs(-(float(mean[f]) * float(w[c, f])))
        bmag.append(mag)
    return sc, w, np.array(bmag)


def test_exact_standard_scaler_fold(eng):
    rng = np.random.default_rng(5)
    F, C = 16, 5
    coef, intercept = rng.standard_normal((C, F)) * 0.5, rng.standard_normal(C)
    mean = rng.uniform(1e2, 1e3, F)
    scale_ = rng.uniform(0.5, 2.0, F)
    X = mean + rng.standard_normal((64, F)) * scale_
    sc, w, bmag = fold_operands(mean, scale_, coef, intercept)
    dm = eng.load_linear(coef, intercept)
    dm.set_affine(shift=mean, scale=sc)
    exact = exact_scores(X, w, intercept, bmag=bmag, fold=(mean, scale_, coef, intercept), fold_rel=FOLD_REL)
    for name, (p, lp) in (("host", both(eng, dm, X)), ("keep_f64", both_resident(eng, dm, eng.stage(X, keep_f64=True)))):
        fails = check_exact(exact, p, lp, False)
        assert not fails, (name, fails[:5])


# ---- 2. against scikit-learn --------------------------------------------------------------------------------------
def make_est(coef, intercept):
    from sklearn.linear_model import LogisticRegression

    est = LogisticRegression()
    est.coef_, est.intercept_ = np.asarray(coef), np.atleast_1d(np.asarray(intercept))
    est.classes_ = np.arange(max(est.coef_.shape[0], 2))
    est.n_features_in_ = est.coef_.shape[1]
    return est


def sklearn_tolerance(X, coef, intercept, want):
    """The 3.9 bound of our result plus the same bound of scikit-learn's: its scores are within gamma_F a_c of the
    exact ones (a BLAS in another order), and numpy's float64 exp / log are taken as within 4 ulp."""
    F = X.shape[1]
    W, b = expanded(coef, intercept)
    a = np.abs(X) @ np.abs(W).T + np.abs(b)
    gF = F * U / (1 - F * U)
    delta = ((F + 3) * U + gF) * a * (1 + 1e-6) + (F + 3) * TRUE_MIN
    C = W.shape[0]
    if np.atleast_2d(coef).shape[0] == 1:
        rel = np.expm1(2 * delta[:, 1:2]) + 16 * U
        b1 = want[:, 1:2] * rel + 2 * 2.0**-1022
        return np.hstack([b1 + 2 * U * want[:, :1], b1]) * (1 + 1e-6)
    s = X @ W.T + b
    L = np.ptp(s, axis=1, keepdims=True) + 4 * delta.max(axis=1, keepdims=True)
    gamma = (C - 1) * U / (1 - (C - 1) * U)
    K = 2 * (delta + delta.max(axis=1, keepdims=True)) + 4 * U * L
    return (want * (np.expm1(K) + 2 * gamma + 24 * U) + 2 * (C + 2) * TRUE_MIN) * (1 + 1e-6)


def assert_close_to_sklearn(got, want, X, coef, intercept, log=False, want_p=None):
    assert got.shape == want.shape and got.dtype == np.float64
    if not log:
        tol = sklearn_tolerance(X, coef, intercept, want)
        err = np.abs(got - want)
        assert np.all(err <= tol), (float(np.max(err / np.maximum(tol, 1e-300))), int(np.sum(err > tol)))
        return
    assert np.array_equal(np.isneginf(got), np.isneginf(want))
    fin = np.isfinite(want)
    tolp = sklearn_tolerance(X, coef, intercept, want_p)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = tolp / want_p
        tol = -np.log1p(-np.minimum(r, 0.5)) * (1 + 1e-6) + 8 * U * np.abs(want)
    ok = np.abs(got - want) <= tol
    assert np.all(ok[fin & (r <= 0.5)]), float(np.max(np.abs(got - want)[fin & (r <= 0.5)]))


@pytest.mark.parametrize("F", [1, 32, 33, 64, 65, 784])
@pytest.mark.parametrize("C", [2, 3, 10, 16, 17, 40])
def test_shapes_against_sklearn(eng, F, C):
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    rng = np.random.default_rng(F * 100 + C)
    binary = C == 2
    coef, intercept = planted_model(rng, C, F, binary)
    coef *= 3.0 / np.sqrt(F)
    est = make_est(coef, intercept)
    X = rng.standard_normal((333, F))
    got = linear_predict_proba(est, X, dtype=np.float64)
    want = est.predict_proba(X)
    assert_close_to_sklearn(got, want, X, coef, intercept)
    assert_rows_sum_to_one(got)
    got_l = linear_predict_log_proba(est, X)
    assert_close_to_sklearn(got_l, est.predict_log_proba(X), X, coef, intercept, log=True, want_p=want)
    # the resident route agrees bitwise with the host route on the same values
    dm = eng.load_linear(est.coef_, est.intercept_)
    res, st = eng.predict_proba_f64(dm, eng.stage(X, keep_f64=True), want_stats=True)
    assert st["path"] == 7
    assert np.array_equal(res, got)
    assert np.array_equal(eng.predict_proba_f64(dm, eng.stage(X, keep_f64=True), log=True)[0], got_l)


def test_digits_logistic_regression_against_sklearn(digits_model, synthetic_digits):
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    est = make_est(digits_model["coef"], digits_model["intercept"])
    est.classes_ = digits_model["classes"]
    X = synthetic_digits["X"].astype(np.float64)
    want = est.predict_proba(X)
    assert_close_to_sklearn(linear_predict_proba(est, X, dtype=np.float64), want, X, est.coef_, est.intercept_)
    Xp = pd.DataFrame(X)
    assert_close_to_sklearn(linear_predict_log_proba(est, Xp), est.predict_log_proba(Xp), X, est.coef_,
                            est.intercept_, log=True, want_p=want)
    # the default stays the fp32 route
    assert linear_predict_proba(est, X).dtype == np.float32


def test_pipeline_standard_scaler_against_sklearn():
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import make_pipeline
    from sklearn.preprocessing import StandardScaler

    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    rng = np.random.default_rng(8)
    X = rng.standard_normal((800, 12)) * rng.uniform(1, 50, 12) + rng.uniform(-100, 100, 12)
    y = np.argmax(X[:, :4] - X[:, :4].mean(0), axis=1)
    pipe = make_pipeline(StandardScaler(), LogisticRegression(max_iter=2000)).fit(X, y)
    got = linear_predict_proba(pipe, X, dtype=np.float64)
    want = pipe.predict_proba(X)
    assert np.max(np.abs(got - want)) < 1e-12
    lg = linear_predict_log_proba(pipe, X)
    wl = pipe.predict_log_proba(X)
    assert np.array_equal(np.isneginf(lg), np.isneginf(wl))
    fin = np.isfinite(wl) & (want > 1e-200)
    assert np.max(np.abs(lg[fin] - wl[fin]) / np.maximum(1, np.abs(wl[fin]))) < 1e-10


# ---- 3. the two normalisation forms -------------------------------------------------------------------------------
def test_grouped_and_one_group_forms_agree_bitwise(eng):
    rng = np.random.default_rng(9)
    F = 40
    coef16, b16 = planted_model(rng, 16, F)
    coef17 = np.vstack([coef16, np.zeros((1, F))])
    b17 = np.concatenate([b16, [-1e6]])  # exp(-1e6 - m) = 0 exactly, added last: the sum does not move
    d16, d17 = eng.load_linear(coef16, b16), eng.load_linear(coef17, b17)
    X = rng.standard_normal((1000, F))
    for log in (False, True):
        p16, st16 = eng.predict_proba_f64_host(d16, X, log=log)
        p17, st17 = eng.predict_proba_f64_host(d17, X, log=log)
        assert st16["path"] == st17["path"] == 7
        assert np.array_equal(p17[:, :16], p16), log
        assert np.all(p17[:, 16] == (-np.inf if log else 0.0))
        bt = eng.stage(X, keep_f64=True)
        assert np.array_equal(eng.predict_proba_f64(d17, bt, log=log)[0], p17)
        assert np.array_equal(eng.predict_proba_f64(d16, bt, log=log)[0], p16)


# ---- 4. host layouts and the labels -------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [10, 17])
def test_host_layouts_bitwise_equal_resident(eng, digits_model, C):
    if C == 10:
        coef, intercept = digits_model["coef"], digits_model["intercept"]
    else:
        coef, intercept = planted_model(np.random.default_rng(10), C, 64)
        coef *= 0.01
    dm = eng.load_linear(coef, intercept)
    rng = np.random.default_rng(11)
    n = 5000
    base = rng.integers(0, 256, size=(n, 64)) * 1.0
    base[::3] += 0.5 + 1e-7  # lossy in fp32 as float64
    for dt in (np.float32, np.float64, np.int32, np.int64, np.uint8):
        X = base.astype(dt)
        for log in (False, True):
            want = eng.predict_proba_f64(dm, eng.stage(X, keep_f64=True), log=log)[0]
            for order in ("C", "F"):
                Xo = np.asarray(X, order=order)
                for pinned in (False, True):
                    if pinned:
                        P = eng.pinned_empty(Xo.T.shape if order == "F" else Xo.shape, dt)
                        P[...] = Xo.T if order == "F" else Xo
                        Xo = P.T if order == "F" else P
                    for chunk in (0, 1300):  # 1300 -> 1408-row chunks: the last one ragged
                        got, st = eng.predict_proba_f64_host(dm, Xo, log=log, chunk_rows=chunk)
                        assert st["path"] == 7
                        assert np.array_equal(got, want), (dt, order, pinned, chunk, log)
            got = eng.predict_proba_f64_host(dm, pd.DataFrame(X), log=log)[0]  # a feature-major pandas block
            assert np.array_equal(got, want), (dt, log)


def test_small_batches_take_the_pipeline(eng, digits_model):
    dm = eng.load_linear(digits_model["coef"], digits_model["intercept"])
    X = np.random.default_rng(12).integers(0, 17, size=(64, 64)).astype(np.float64)
    for n in (1, 7, 64):
        got, st = eng.predict_proba_f64_host(dm, X[:n])
        assert st["path"] == 7 and got.shape == (n, 10)
        assert np.array_equal(got, eng.predict_proba_f64(dm, eng.stage(X[:n], keep_f64=True))[0])


@pytest.mark.parametrize("binary", [False, True])
def test_argmax_matches_exact_labels_outside_twice_the_bound(eng, digits_model, binary):
    from tests.conftest import digits_batch

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    if binary:
        coef, intercept = coef[:1], intercept[:1]
    dm = eng.load_linear(coef, intercept)
    X = digits_batch(21, 50_000)
    b = eng.stage(X)
    labels, _ = eng.predict(dm, b, exact=True)
    p = eng.predict_proba_f64(dm, b)[0]
    tol = sklearn_tolerance(X.astype(np.float64), coef, intercept, p)
    top = np.argsort(p, axis=1)[:, ::-1][:, :2]
    rows = np.arange(len(p))
    p1, p2 = p[rows, top[:, 0]], p[rows, top[:, 1]]
    clear = p1 - p2 > 2 * np.maximum(tol[rows, top[:, 0]], tol[rows, top[:, 1]])
    assert clear.sum() > 0.99 * len(p)
    assert np.array_equal(np.argmax(p, axis=1)[clear], labels[clear])


# ---- 5. edges -----------------------------------------------------------------------------------------------------
def test_scores_spanning_800_underflow_like_sklearn():
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    est = make_est(np.array([[1.0], [0.0], [-1.0], [0.5]]), np.zeros(4))
    X = np.linspace(-800, 800, 4001)[:, None] + 0.0123  # the scores are exact products: the same bits as sklearn's
    got, want = linear_predict_proba(est, X, dtype=np.float64), est.predict_proba(X)
    assert np.array_equal(got == 0, want == 0) and np.any(want == 0)
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-322)  # (a subnormal e_c: a few of its ulps)
    gl, wl = linear_predict_log_proba(est, X), est.predict_log_proba(X)
    assert np.array_equal(np.isneginf(gl), np.isneginf(wl)) and np.any(np.isneginf(wl))
    fin = np.isfinite(wl)
    np.testing.assert_allclose(gl[fin], wl[fin], rtol=1e-13, atol=1e-300)


def test_all_equal_scores_give_one_over_c(eng):
    for C in (3, 10, 17, 40):
        dm = eng.load_linear(np.zeros((C, 5)), np.full(C, 2.5))
        p = eng.predict_proba_f64_host(dm, np.random.default_rng(C).standard_normal((300, 5)))[0]
        assert np.all(p == 1.0 / C), C


def test_binary_plus_minus_40():
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    est = make_est(np.array([[1.0]]), np.array([0.0]))
    X = np.array([[40.0], [-40.0], [36.7], [-36.7], [0.0]])
    got, want = linear_predict_proba(est, X, dtype=np.float64), est.predict_proba(X)
    assert got[0, 0] == want[0, 0] == 0.0 and got[0, 1] == 1.0  # 1 - p rounds to 0
    assert got[1, 0] == 1.0 and got[4, 0] == got[4, 1] == 0.5
    np.testing.assert_allclose(got, want, rtol=1e-15, atol=0)
    gl, wl = linear_predict_log_proba(est, X), est.predict_log_proba(X)
    assert gl[0, 0] == wl[0, 0] == -np.inf and gl[1, 0] == 0.0
    np.testing.assert_allclose(gl[1:], wl[1:], rtol=1e-13, atol=1e-300)


@pytest.mark.parametrize("binary", [False, True])
def test_finite_features_whose_scores_overflow_give_sklearns_nan_pattern(binary):
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    rng = np.random.default_rng(19)
    coef, intercept = rng.standard_normal((1 if binary else 3, 5)) * 1e10, rng.standard_normal(1 if binary else 3)
    est = make_est(coef, intercept)
    X = rng.standard_normal((200, 5))
    X[::4, 1] = 1e300
    X[1::4, 2] = -1e300
    X[2::8, 1:3] = [1e300, 1e300]  # inf - inf somewhere: NaN
    got = linear_predict_proba(est, X, dtype=np.float64)
    gl = linear_predict_log_proba(est, X)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        want = est.predict_proba(X)
        wl = est.predict_log_proba(X)
    assert (binary or np.any(np.isnan(want))) and np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(np.isnan(gl), np.isnan(wl)) and np.array_equal(np.isneginf(gl), np.isneginf(wl))
    exact01 = (want == 0) | (want == 1)
    assert np.array_equal(got[exact01], want[exact01])
    fin = ~np.isnan(want)
    np.testing.assert_allclose(got[fin], want[fin], rtol=0, atol=1e-9)


@pytest.mark.parametrize("C", [2, 10, 40])
def test_device_output_guards_and_8_byte_alignment(eng, C):
    rng = np.random.default_rng(13)
    coef, intercept = planted_model(rng, C, 64, C == 2)
    dm = eng.load_linear(coef, intercept)
    n = 1000 + 37
    b = eng.stage(rng.standard_normal((n, 64)), keep_f64=True)
    for log in (False, True):
        want = eng.predict_proba_f64(dm, b, log=log)[0].reshape(-1)
        assert want.size == n * C
        for off in (2, 1):  # 16-byte aligned, then 8 bytes off
            buf = torch.full((want.size + 4,), -7.25, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()  # the engine runs on its own stream
            _, st = eng.predict_proba_f64(dm, b, log=log, out_device_ptr=buf.data_ptr() + 8 * off, want_stats=True)
            h = buf.cpu().numpy()
            assert np.array_equal(h[off:off + want.size], want), (off, log)
            assert np.all(h[:off] == -7.25) and np.all(h[off + want.size:] == -7.25), (off, log)
            assert st["d2h_bytes"] == 0 and st["path"] == 7


def test_error_contract(eng):
    from sklearn.exceptions import NotFittedError
    from sklearn.linear_model import LinearRegression, LogisticRegression

    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    def f64(est, X):
        return linear_predict_proba(est, X, dtype=np.float64)

    rng = np.random.default_rng(17)
    est = make_est(rng.standard_normal((4, 6)), rng.standard_normal(4))
    X = rng.standard_normal((300, 6))
    for fn in (f64, linear_predict_log_proba):
        for bad in (np.nan, np.inf, -np.inf):
            Xb = X.copy()
            Xb[123, 4] = bad
            with pytest.raises(ValueError, match="NaN or infinity"):
                fn(est, Xb)
        with pytest.raises(ValueError, match="features"):
            fn(est, X[:, :5])
        with pytest.raises(ValueError, match="0 sample"):
            fn(est, X[:0])
        est2 = make_est(est.coef_, est.intercept_)
        est2.feature_names_in_ = np.array([f"f{i}" for i in range(6)], dtype=object)
        with pytest.raises(ValueError, match="feature names"):
            fn(est2, pd.DataFrame(X, columns=[f"g{i}" for i in range(6)]))
        reg = LinearRegression()
        reg.coef_, reg.intercept_ = np.ones(6), 0.0
        with pytest.raises(TypeError, match="classifier"):
            fn(reg, X)
        with pytest.raises(NotFittedError):
            fn(LogisticRegression(), X)
    for dtype in (np.float16, np.int64, "float128-ish", None):
        with pytest.raises(ValueError, match="float32 or float64"):
            linear_predict_proba(est, X, dtype=dtype)
    # NaN in rows wrapped in place on the device (no staging scan)
    dm = eng.load_linear(est.coef_, est.intercept_)
    t = torch.tensor(X, dtype=torch.float32, device="cuda")
    t[5, 0] = float("nan")
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="NaN or infinity"):
        eng.predict_proba_f64(dm, eng.wrap_device(t.data_ptr(), 300, 6, keepalive=t))
    with pytest.raises(ValueError, match="shape"):
        eng.predict_proba_f64_host(dm, X, out=np.empty((300, 5)))


# ---- 6. through the API -------------------------------------------------------------------------------------------
def test_model_predict_with_a_float64_proba_predictor_and_callback():
    from sklearn.datasets import load_digits
    from sklearn.linear_model import LogisticRegression

    from unionml_b200 import Dataset, Model
    from unionml_b200.predictors import linear_predict_log_proba, linear_predict_proba

    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="digits_classifier", init=LogisticRegression, dataset=dataset)
    seen = []

    @dataset.reader
    def reader(sample_frac: float = 1.0, random_state: int = 0) -> pd.DataFrame:
        return load_digits(as_frame=True).frame.sample(frac=sample_frac, random_state=random_state)

    @model.trainer
    def trainer(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> LogisticRegression:
        return estimator.fit(features, target.squeeze())

    def callback(estimator: LogisticRegression, features: pd.DataFrame, prediction: List[List[float]]) -> None:
        seen.append(prediction)

    @model.predictor(callbacks=[callback])
    def predictor(estimator: LogisticRegression, features: pd.DataFrame) -> List[List[float]]:
        return linear_predict_proba(estimator, features, dtype=np.float64).tolist()

    @model.evaluator
    def evaluator(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> float:
        return float((estimator.predict(features) == target.squeeze()).mean())

    est, _ = model.train(hyperparameters={"C": 1.0, "max_iter": 1000}, sample_frac=1.0, random_state=123)
    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]].sample(700, random_state=3)
    out = model.predict(features=feats)
    assert len(seen) == 1 and seen[0] is out
    assert len(out) == 700 and all(len(r) == 10 and all(isinstance(v, float) for v in r) for r in out)
    Xf = feats.to_numpy(dtype=np.float64)
    want = est.predict_proba(feats)
    assert_close_to_sklearn(np.array(out), want, Xf, est.coef_, est.intercept_)
    # predict_log_proba on a DataFrame with the fitted feature names
    assert list(est.feature_names_in_) == list(feats.columns)
    got_l = linear_predict_log_proba(est, feats)
    assert_close_to_sklearn(got_l, est.predict_log_proba(feats), Xf, est.coef_, est.intercept_, log=True, want_p=want)


# ---- 7. one full-size run -----------------------------------------------------------------------------------------
def test_full_size_host_10m_rows_against_numpy(eng, digits_model):
    from tests.conftest import digits_batch

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    dm = eng.load_linear(coef, intercept)
    N, C = 10_000_000, 10
    X = digits_batch(0, N, dtype=np.uint8)
    out, st = eng.predict_proba_f64_host(dm, X)
    assert st["path"] == 7 and st["n_nonfinite"] == 0 and out.shape == (N, C)
    step = 1_000_000
    for r0 in range(0, N, step):
        Xc = X[r0:r0 + step].astype(np.float64)
        s = Xc @ coef.T + intercept
        e = np.exp(s - s.max(axis=1, keepdims=True))
        want = e / e.sum(axis=1, keepdims=True)
        tol = sklearn_tolerance(Xc, coef, intercept, want)
        assert np.all(np.abs(out[r0:r0 + step] - want) <= tol), r0
