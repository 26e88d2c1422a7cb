"""Float64 decision_function scores (``uml_linear_decision_function*``, ``predictors.linear_decision_function``).

Contract (DESIGN.md 3.7): every score is within ``((F + 3) u + fold_rel) a_c + (F + 3) 2^-1074`` of the exact score
T_c of the caller's values, ``u = 2^-53``, ``a_c = sum_f |x_f w_cf| + bmag_c``.  Checked here with exact rational
arithmetic on planted batches, on every row source (raw host chunk, the keep_f64 copy, fp32 rows), against
scikit-learn's own BLAS result within that bound plus gamma_F a_c, and for bitwise agreement between the host layouts
and the resident route on the same values.
"""
from fractions import Fraction
from typing import List

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

U = Fraction(1, 2**53)
Q = Fraction(1, 2**1074)
FOLD_REL = 8 * U


@pytest.fixture(scope="module")
def eng():
    from unionml_b200.engine import get_engine

    return get_engine()


def _fr(v) -> Fraction:
    return Fraction(int(v)) if isinstance(v, (int, np.integer)) else Fraction(float(v))


def exact_check(got, X, W, b, bmag=None, fold=None, fold_rel=Fraction(0)):
    """Failures (strings) of the stated bound, with T and a_c in exact arithmetic.  W, b: the model the device scores
    (for a fold: w' and b' with the caller's scaler as fold = (mean_, scale_, w, b)); bmag: the bias magnitudes."""
    n, F = X.shape
    C = W.shape[0]
    got = np.asarray(got, dtype=np.float64).reshape(n, -1)
    c_first = C - got.shape[1]  # binary: only the score of class 1 of the expanded [0, s]
    Wf = [[_fr(W[c, f]) for f in range(F)] for c in range(C)]
    bm = [abs(_fr(v)) for v in b] if bmag is None else [_fr(v) for v in bmag]
    fails = []
    for r in range(n):
        xr = [_fr(X[r, f]) for f in range(F)]
        if fold is not None:
            mean, scale, w0, b0 = fold
            z = [(xr[f] - _fr(mean[f])) / _fr(scale[f]) for f in range(F)]
        for c in range(c_first, C):
            if fold is None:
                T = sum(xr[f] * Wf[c][f] for f in range(F)) + _fr(b[c])
            else:
                T = sum(z[f] * _fr(w0[c, f]) for f in range(F)) + _fr(b0[c])
            a = sum(abs(xr[f] * Wf[c][f]) for f in range(F)) + bm[c]
            bound = ((F + 3) * U + fold_rel) * a + (F + 3) * Q
            s = got[r, c - c_first]
            if not np.isfinite(s) or abs(Fraction(float(s)) - T) > bound:
                fails.append(f"row {r} class {c}: got {s!r}, exact {float(T)!r}, bound {float(bound):.3g}")
    return fails


def expanded(coef, intercept):
    """The model as the device stores it: a binary coef_ row becomes classes [0, s]."""
    coef = np.atleast_2d(np.asarray(coef, dtype=np.float64))
    intercept = np.atleast_1d(np.asarray(intercept, dtype=np.float64))
    if coef.shape[0] == 1:
        return np.vstack([np.zeros_like(coef), coef]), np.concatenate([[0.0], intercept])
    return coef, intercept


def spread_model(rng, C, F, binary=False):
    rows = 1 if binary else C
    coef = rng.standard_normal((rows, F)) * 2.0 ** rng.integers(-20, 20, size=(rows, F))
    return coef, rng.standard_normal(rows) * 2.0 ** rng.integers(-10, 10, size=rows)


def all_sources(eng, dm, X, X32_exact=True):
    """(name, scores) of every row source for the caller's values X: the raw host chunk, the keep_f64 copy, and (for
    values that are fp32 values) the fp32 rows."""
    out = [("raw", eng.decision_function_host(dm, X)[0])]
    b = eng.stage(X, keep_f64=True)
    out.append(("keep_f64" if not b.lossless else "fp32_rows_lossless", eng.decision_function(dm, b)[0]))
    if X32_exact:
        b32 = eng.stage(X.astype(np.float32), keep_f64=False)
        out.append(("fp32_rows", eng.decision_function(dm, b32)[0]))
    return out


# ---- 1. exact arithmetic ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("binary", [False, True])
def test_exact_lossy_float64_perturbed(eng, binary):
    rng = np.random.default_rng(1)
    F, C = 33, 10
    coef, intercept = spread_model(rng, C, F, binary)
    X = rng.integers(-50, 50, size=(150, F)).astype(np.float64) * 2.0 ** rng.integers(-8, 8, size=(150, F))
    X += rng.choice([-1e-9, 1e-9], size=X.shape)  # the fp32 copy is lossy
    dm = eng.load_linear(coef, intercept)
    W, b = expanded(coef, intercept)
    for name, got in all_sources(eng, dm, X, X32_exact=False):
        assert got.shape == ((150,) if binary else (150, C)), name
        fails = exact_check(got, X, W, b)
        assert not fails, (name, fails[:5])
    assert not eng.stage(X, keep_f64=False).lossless
    with pytest.raises(Exception, match="keep_f64|KEEP_F64|lossy"):  # fp32 rows that are not the caller's values
        eng.decision_function(dm, eng.stage(X, keep_f64=False))
    # the fp32 rows as the caller's values
    X32 = X.astype(np.float32)
    got = eng.decision_function(dm, eng.stage(X32, keep_f64=False))[0]
    assert not exact_check(got, X32, W, b)


def test_exact_int64_above_2_53(eng):
    rng = np.random.default_rng(2)
    F, C = 8, 3
    coef, intercept = spread_model(rng, C, F)
    X = rng.integers(2**53, 2**62, size=(100, F), dtype=np.int64) * rng.choice([-1, 1], size=(100, F))
    X[::7, 0] = 2**53 + 1  # not a float64 value
    dm = eng.load_linear(coef, intercept)
    for name, got in all_sources(eng, dm, X, X32_exact=False):
        fails = exact_check(got, X, coef, intercept)
        assert not fails, (name, fails[:5])
    for X2 in (np.asfortranarray(X), X.astype(np.int32) // 7):  # feature-major int64, int32
        got = eng.decision_function_host(dm, X2)[0]
        assert not exact_check(got, X2, coef, intercept)


def test_exact_float64_beyond_fp32_range(eng):
    rng = np.random.default_rng(3)
    F, C = 20, 4
    coef = rng.standard_normal((C, F)) * 1e-12
    intercept = rng.standard_normal(C)
    X = rng.standard_normal((120, F)) * 1e40
    X[::5] *= 1e200  # scores ~1e228, still finite
    dm = eng.load_linear(coef, intercept)
    for name, got in all_sources(eng, dm, X, X32_exact=False):
        fails = exact_check(got, X, coef, intercept)
        assert not fails, (name, fails[:5])


def test_exact_products_below_dbl_min(eng):
    F, C = 3, 2
    t = 2.0**-537
    coef = np.array([[0.6 * t, 0.6 * t, 0.0], [0.0, 0.0, 1.4 * t]])
    intercept = np.zeros(C)
    X = np.full((64, F), t)
    X[1::2] *= np.array([1.0, -1.0, 1.0])
    dm = eng.load_linear(coef, intercept)
    for name, got in all_sources(eng, dm, X, X32_exact=False):
        fails = exact_check(got, X, coef, intercept)
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


def test_exact_standard_scaler_fold_mean_much_larger_than_scale(eng):
    rng = np.random.default_rng(5)
    F, C = 16, 5
    coef, intercept = rng.standard_normal((C, F)), rng.standard_normal(C)
    mean = rng.uniform(1e5, 1e6, F)
    scale_ = rng.uniform(1e-3, 1e-2, F)
    X = mean + rng.standard_normal((100, F)) * scale_
    sc, w, bmag = fold_operands(mean, scale_, coef, intercept)
    dm = eng.load_linear(coef, intercept)
    dm.set_affine(shift=mean, scale=sc)
    for name, got in all_sources(eng, dm, X, X32_exact=False):
        fails = exact_check(got, X, w, intercept, bmag=bmag, fold=(mean, scale_, coef, intercept), fold_rel=FOLD_REL)
        assert not fails, (name, fails[:5])


# ---- 2. against scikit-learn --------------------------------------------------------------------------------------
def sklearn_tolerance(X, coef, intercept):
    """bound + gamma_F a_c per score, a_c in float64 (its own rounding is ~F u relative: the 1e-6 slack)."""
    F = X.shape[1]
    a = np.abs(X) @ np.abs(np.atleast_2d(coef)).T + np.abs(np.atleast_1d(intercept))
    u = 2.0**-53
    k = F + 3
    return ((k * u + F * u / (1 - F * u)) * a + k * 2.0**-1074) * (1 + 1e-6)


def assert_close_to_sklearn(got, want, X, coef, intercept):
    tol = sklearn_tolerance(X, coef, intercept).reshape(np.shape(want))
    assert got.shape == want.shape and got.dtype == np.float64
    err = np.abs(got - want)
    assert np.all(err <= tol), (float(np.max(err / np.maximum(tol, 1e-300))), int(np.sum(err > tol)))


def make_est(coef, intercept, cls=None):
    from sklearn.linear_model import LogisticRegression

    est = (cls or LogisticRegression)()
    est.coef_, est.intercept_ = np.asarray(coef), np.atleast_1d(np.asarray(intercept))
    est.classes_ = np.arange(max(est.coef_.shape[0], 2))
    est.n_features_in_ = est.coef_.shape[1]
    return est


def test_digits_logistic_regression_against_sklearn(digits_model, synthetic_digits):
    from unionml_b200.predictors import linear_decision_function

    est = make_est(digits_model["coef"], digits_model["intercept"])
    est.classes_ = digits_model["classes"]
    X = synthetic_digits["X"].astype(np.float64)
    got = linear_decision_function(est, X)
    assert_close_to_sklearn(got, est.decision_function(X), X, est.coef_, est.intercept_)
    Xp = pd.DataFrame(X)
    assert_close_to_sklearn(linear_decision_function(est, Xp), est.decision_function(Xp), X, est.coef_, est.intercept_)


def test_fitted_classifiers_without_predict_proba_against_sklearn():
    from sklearn.linear_model import LogisticRegression, RidgeClassifier
    from sklearn.svm import LinearSVC

    from unionml_b200.predictors import linear_decision_function

    rng = np.random.default_rng(7)
    X = rng.standard_normal((600, 20))
    y3 = rng.integers(0, 3, 600)
    Xq = rng.standard_normal((1000, 20)) * 3
    for est in (LinearSVC().fit(X, y3), RidgeClassifier().fit(X, y3),
                LogisticRegression().fit(X, (X[:, 0] > 0).astype(int)),
                LinearSVC().fit(X, np.where(X[:, 1] > 0, "yes", "no"))):  # binary, string classes_
        got = linear_decision_function(est, Xq)
        want = est.decision_function(Xq)
        assert got.shape == want.shape, type(est).__name__
        assert_close_to_sklearn(got, want, Xq, est.coef_, est.intercept_)


@pytest.mark.parametrize("F", [1, 32, 33, 64, 65, 784])
@pytest.mark.parametrize("C", [2, 3, 10, 16, 17, 40])
def test_shapes_against_sklearn(eng, F, C):
    from unionml_b200.predictors import linear_decision_function

    rng = np.random.default_rng(F * 100 + C)
    est = make_est(rng.standard_normal((C, F)), rng.standard_normal(C))
    X = rng.standard_normal((333, F))
    got = linear_decision_function(est, X)
    assert_close_to_sklearn(got, est.decision_function(X), X, est.coef_, est.intercept_)
    # the resident route agrees bitwise with the host route on the same values
    dm = eng.load_linear(est.coef_, est.intercept_)
    res, st = eng.decision_function(dm, eng.stage(X, keep_f64=True), want_stats=True)
    assert st["path"] == 6
    assert np.array_equal(res, got)


# ---- 3. host layouts ----------------------------------------------------------------------------------------------
def test_host_layouts_bitwise_equal_resident(eng, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    dm = eng.load_linear(coef, intercept)
    rng = np.random.default_rng(11)
    n = 5000
    base = rng.integers(-2**20, 2**20, size=(n, 64)) * 1.0
    base[::3] += 0.5 + 1e-7  # lossy in fp32 as float64
    for dt in (np.float32, np.float64, np.int32, np.int64):
        X = base.astype(dt)
        want = eng.decision_function(dm, eng.stage(X, keep_f64=True))[0]
        for order in ("C", "F"):
            Xo = np.asarray(X, order=order)
            for pinned in (False, True):
                if pinned:
                    P = eng.pinned_empty(Xo.T.shape if order == "F" else Xo.shape, dt)
                    P[...] = Xo.T if order == "F" else Xo
                    Xo = P.T if order == "F" else P
                for chunk in (0, 1300):  # 1300 -> 1408-row chunks: the last one ragged
                    got, st = eng.decision_function_host(dm, Xo, chunk_rows=chunk)
                    assert st["path"] == 6
                    assert np.array_equal(got, want), (dt, order, pinned, chunk)
        got = eng.decision_function_host(dm, pd.DataFrame(X))[0]  # a feature-major pandas block
        assert np.array_equal(got, want), dt


def test_lossless_float64_frame_narrowed_by_the_gather_threads(eng, digits_model):
    dm = eng.load_linear(digits_model["coef"], digits_model["intercept"])
    n = 40_000  # 20 MB pageable: bounce buffers and the fp32 wire
    X = np.random.default_rng(12).integers(0, 17, size=(n, 64)).astype(np.float64)
    got, st = eng.decision_function_host(dm, pd.DataFrame(X), chunk_rows=9000)
    assert st["h2d_bytes"] == n * 64 * 4, st  # crossed PCIe as fp32
    want = eng.decision_function(dm, eng.stage(X.astype(np.float32), keep_f64=False))[0]
    assert np.array_equal(got, want)


# ---- 4. device output ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("binary", [False, True])
def test_device_output_guards_and_8_byte_alignment(eng, binary):
    rng = np.random.default_rng(13)
    coef, intercept = spread_model(rng, 10, 64, binary)
    dm = eng.load_linear(coef, intercept)
    n = 1000 + 37
    b = eng.stage(rng.standard_normal((n, 64)), keep_f64=True)
    want = eng.decision_function(dm, b)[0].reshape(-1)
    for off in (2, 1):  # 16-byte aligned, then 8 bytes off
        buf = torch.full((want.size + 4,), -7.25, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()  # the engine runs on its own stream
        _, st = eng.decision_function(dm, b, out_device_ptr=buf.data_ptr() + 8 * off, want_stats=True)
        h = buf.cpu().numpy()
        assert np.array_equal(h[off:off + want.size], want), off
        assert np.all(h[:off] == -7.25) and np.all(h[off + want.size:] == -7.25), off
        assert st["d2h_bytes"] == 0 and st["path"] == 6


# ---- 5. consistency with the labels -------------------------------------------------------------------------------
@pytest.mark.parametrize("binary", [False, True])
def test_argmax_of_scores_matches_exact_labels(eng, digits_model, binary):
    from tests.conftest import digits_batch

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    if binary:
        coef, intercept = coef[:1], intercept[:1]
    dm = eng.load_linear(coef, intercept)
    X = digits_batch(21, 50_000)
    b = eng.stage(X)
    labels, st = eng.predict(dm, b, exact=True)
    scores = eng.decision_function(dm, b)[0]
    pred = (scores > 0).astype(np.int32) if binary else np.argmax(scores, axis=1).astype(np.int32)
    assert int(np.sum(pred != labels)) <= st["n_ambiguous"]


# ---- 6. error contract --------------------------------------------------------------------------------------------
def test_error_contract(eng):
    from sklearn.exceptions import NotFittedError
    from sklearn.linear_model import LinearRegression, LogisticRegression

    from unionml_b200.predictors import linear_decision_function

    rng = np.random.default_rng(17)
    est = make_est(rng.standard_normal((4, 6)), rng.standard_normal(4))
    X = rng.standard_normal((300, 6))
    for bad in (np.nan, np.inf, -np.inf):
        Xb = X.copy()
        Xb[123, 4] = bad
        with pytest.raises(ValueError, match="NaN or infinity"):
            linear_decision_function(est, Xb)
    # NaN in rows wrapped in place on the device (no staging scan)
    dm = eng.load_linear(est.coef_, est.intercept_)
    t = torch.tensor(X, dtype=torch.float32, device="cuda")
    t[5, 0] = float("nan")
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="NaN or infinity"):
        eng.decision_function(dm, eng.wrap_device(t.data_ptr(), 300, 6, keepalive=t))
    with pytest.raises(ValueError, match="features"):
        linear_decision_function(est, X[:, :5])
    with pytest.raises(ValueError, match="0 sample"):
        linear_decision_function(est, X[:0])
    est.feature_names_in_ = np.array([f"f{i}" for i in range(6)], dtype=object)
    with pytest.raises(ValueError, match="feature names"):
        linear_decision_function(est, pd.DataFrame(X, columns=[f"g{i}" for i in range(6)]))
    reg = LinearRegression()
    reg.coef_, reg.intercept_ = np.ones(6), 0.0
    with pytest.raises(TypeError, match="classifier"):
        linear_decision_function(reg, X)
    with pytest.raises(NotFittedError):
        linear_decision_function(LogisticRegression(), X)


def test_finite_features_whose_scores_overflow_match_numpy():
    from unionml_b200.predictors import linear_decision_function

    rng = np.random.default_rng(19)
    coef = rng.standard_normal((3, 5)) * 1e10
    est = make_est(coef, rng.standard_normal(3))
    X = rng.standard_normal((200, 5))
    X[::4, 1] = 1e300
    X[1::4, 2] = -1e300
    X[2::8, 1:3] = [1e300, 1e300]  # inf - inf somewhere: NaN
    got = linear_decision_function(est, X)
    with np.errstate(over="ignore", invalid="ignore"):
        want = est.decision_function(X)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[np.isinf(want)], want[np.isinf(want)])
    fin = np.isfinite(want) & np.isfinite(got)
    assert np.isinf(got).sum() == np.isinf(want).sum() and fin.sum() > 0
    with np.errstate(over="ignore", invalid="ignore"):  # the tolerance of the overflowing rows is not used
        tol = sklearn_tolerance(X, est.coef_, est.intercept_)
        err = np.abs(got - want)
    assert np.all(err[fin] <= tol[fin])


# ---- 7. through the API -------------------------------------------------------------------------------------------
def test_model_predict_with_a_decision_function_predictor_and_callback():
    from sklearn.datasets import load_digits
    from sklearn.linear_model import LogisticRegression

    from unionml_b200 import Dataset, Model
    from unionml_b200.predictors import linear_decision_function

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
        return linear_decision_function(estimator, features).tolist()

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
    assert_close_to_sklearn(np.array(out), est.decision_function(feats), Xf, est.coef_, est.intercept_)


# ---- 8. one full-size run -----------------------------------------------------------------------------------------
def test_full_size_resident_10m_rows_against_numpy(eng, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    dm = eng.load_linear(coef, intercept)
    N, F, C = 10_000_000, 64, 10
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 17, (N, F), generator=g, device="cuda", dtype=torch.int32).to(torch.float32)
    torch.cuda.synchronize()  # the rows are written on torch's stream, the engine scores on its own
    b = eng.wrap_device(x.data_ptr(), N, F, keepalive=x)
    out = torch.empty((N, C), dtype=torch.float64, device="cuda")
    _, st = eng.decision_function(dm, b, out_device_ptr=out.data_ptr(), want_stats=True)
    assert st["path"] == 6 and st["n_nonfinite"] == 0
    step = 1_000_000
    for r0 in range(0, N, step):
        Xc = x[r0:r0 + step].cpu().numpy().astype(np.float64)
        got = out[r0:r0 + step].cpu().numpy()
        want = Xc @ coef.T + intercept
        tol = sklearn_tolerance(Xc, coef, intercept)
        assert np.all(np.abs(got - want) <= tol), r0
