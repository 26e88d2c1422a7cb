"""GPU parity tests of the host-facing product path (round 2): ``linear_argmax`` / ``Engine.predict_host`` on the
dtypes and layouts the reference really feeds it.

* float64 frames whose values do NOT survive the fp32 down-cast (sklearn scores the float64 frame,
  ``sklearn/linear_model/_base.py:366-396``): flagged rows are re-scored from the caller's own values;
* the online shape (<= 64 rows): one float64 kernel replayed as a CUDA graph;
* ``predict_proba`` against ``LogisticRegression.predict_proba`` with the tolerance stated;
* the reader-kwargs route (``unionml:unionml/model.py:603-614``) and the BentoML runnable call site
  (``unionml:unionml/services/bentoml.py:201-211``) on the device predictor.
"""
from typing import List

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import linear as olin

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import get_engine

    return get_engine()  # the process-wide engine the predictors use


def _estimator(coef, intercept, classes=None):
    from sklearn.linear_model import LogisticRegression

    est = LogisticRegression()
    est.coef_, est.intercept_ = np.asarray(coef), np.asarray(intercept)
    n = max(2, est.coef_.shape[0])
    est.classes_ = np.arange(n) if classes is None else np.asarray(classes)
    est.n_features_in_ = est.coef_.shape[1]
    return est


def planted_near_ties(rng, coef, intercept, n_rows, eps=1e-9):
    """Rows whose float64 top-2 margin is +-eps (resolvable in float64, far inside the fp32 rounding of the features).

    Take a random row, move it along w_a - w_b until the two best classes tie, then step +-t*eps off the tie."""
    C, F = coef.shape
    X = rng.standard_normal((n_rows, F))
    s = X @ coef.T + intercept
    order = np.argsort(-s, axis=1)
    a, b = order[:, 0], order[:, 1]
    d = coef[a] - coef[b]
    gap = s[np.arange(n_rows), a] - s[np.arange(n_rows), b]
    lin = np.linspace(-1.0, 1.0, n_rows)
    t = np.where(lin < 0, -1.0, 1.0) * (0.1 + 0.9 * np.abs(lin))  # |margin| in [1e-10, 1e-9]: >> float64 rounding (1e-14)
    X = X - ((gap - t * eps) / (d * d).sum(axis=1))[:, None] * d
    return X


def test_lossy_float64_frame_through_linear_argmax(engine):
    """VERDICT r1 weak #1 / ADVICE: near-ties that only the float64 features resolve, through the product API."""
    from unionml_b200.predictors import linear_argmax

    rng = np.random.default_rng(5)
    coef, intercept = rng.standard_normal((5, 12)), rng.standard_normal(5)
    X = planted_near_ties(rng, coef, intercept, 120_000)
    est = _estimator(coef, intercept, classes=[3, 5, 8, 13, 21])
    frame = pd.DataFrame(X, columns=[f"f{i}" for i in range(12)])
    est.feature_names_in_ = np.asarray(frame.columns, dtype=object)
    want = [float(v) for v in est.predict(frame)]
    # the planted rows really are ties for fp32-rounded features: plain fp32 rounding of X changes many labels
    rounded = est.predict(pd.DataFrame(X.astype(np.float32).astype(np.float64), columns=frame.columns))
    assert (rounded != np.asarray(want)).sum() > 1000
    got = linear_argmax(est, frame)  # pandas block: feature-major float64, pageable -> bounce buffers
    assert got == want
    # the same through every host layout the staging layer takes, and the resident route
    m = engine.load_linear(coef, intercept)
    want_idx = olin.predict_indices(olin.decision_function(X, coef, intercept)).astype(np.int32)
    np.testing.assert_array_equal(np.asarray([3, 5, 8, 13, 21], dtype=np.float64)[want_idx], want)
    for name, arr in {"c_order": X, "f_order": np.asfortranarray(X), "strided": np.hstack([X, X])[:, :12]}.items():
        idx, st = engine.predict_host(m, arr, exact=True, chunk_rows=16_384)
        np.testing.assert_array_equal(idx, want_idx, err_msg=name)
        assert st["n_flagged"] > 1000  # the guard sent them to the float64 re-score
    pinned = engine.pinned_empty(X.shape, np.float64)
    pinned[:] = X
    idx, _ = engine.predict_host(m, pinned, exact=True)
    np.testing.assert_array_equal(idx, want_idx)
    idx, _ = engine.predict(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(idx, want_idx)


def test_lossy_integer_features_and_fp32_overflow(engine):
    rng = np.random.default_rng(9)
    coef, intercept = rng.standard_normal((4, 6)), rng.standard_normal(4)
    # int32 / int64 values above 2^24 are not representable in fp32
    Xi = rng.integers(2**24, 2**30, size=(50_000, 6))
    want = olin.predict_indices(olin.decision_function(Xi.astype(np.float64), coef, intercept)).astype(np.int32)
    m = engine.load_linear(coef, intercept)
    for arr in (Xi.astype(np.int64), Xi.astype(np.int32), np.asfortranarray(Xi.astype(np.int64))):
        idx, _ = engine.predict_host(m, arr, exact=True)
        np.testing.assert_array_equal(idx, want)
        idx, _ = engine.predict(m, engine.stage(arr), exact=True)
        np.testing.assert_array_equal(idx, want)
    # finite float64 beyond the fp32 range: Inf after the down-cast, but exact mode scores the float64 source - the
    # call must neither raise (sklearn does not) nor mislabel
    Xf = rng.standard_normal((20_000, 6))
    Xf[::7, 2] = 1e39
    Xf[3::11, 4] = -7e40
    want = olin.predict_indices(olin.decision_function(Xf, coef, intercept)).astype(np.int32)
    idx, st = engine.predict_host(m, Xf, exact=True)
    np.testing.assert_array_equal(idx, want)
    assert st["n_nonfinite"] == 0


def test_lossless_float64_frames_cross_the_link_as_fp32(engine, monkeypatch):
    """Integer-valued float64 frames (the digits / pixel domain) are narrowed to fp32 by the gather threads, every value
    checked; the first chunk with a value that does not survive the down-cast - and all chunks after it - travel as
    float64 and keep the float64 re-score from the caller's values.  Labels are the float64 labels either way."""
    rng = np.random.default_rng(21)
    coef, intercept = rng.standard_normal((5, 12)), rng.standard_normal(5)
    m = engine.load_linear(coef, intercept)
    N, chunk = 300_000, 65_536
    Xi = rng.integers(0, 17, size=(N, 12)).astype(np.float64)
    want = olin.predict_indices(olin.decision_function(Xi, coef, intercept)).astype(np.int32)
    for name, arr in {"c_order": Xi, "f_order": np.asfortranarray(Xi)}.items():
        idx, st = engine.predict_host(m, arr, exact=True, chunk_rows=chunk)
        np.testing.assert_array_equal(idx, want, err_msg=name)
        assert st["h2d_bytes"] == N * 12 * 4, name  # half the float64 bytes
    monkeypatch.setenv("UML_B200_NO_NARROW", "1")
    idx, st = engine.predict_host(m, np.asfortranarray(Xi), exact=True, chunk_rows=chunk)
    np.testing.assert_array_equal(idx, want)
    assert st["h2d_bytes"] == N * 12 * 8
    monkeypatch.delenv("UML_B200_NO_NARROW")
    # a strided row-major source (column slice of a wider array) is gathered row by row: not narrowed
    idx, st = engine.predict_host(m, np.hstack([Xi, Xi])[:, :12], exact=True, chunk_rows=chunk)
    np.testing.assert_array_equal(idx, want)
    assert st["h2d_bytes"] == N * 12 * 8
    # chunks 0-1 lossless, planted +-1e-9 near-ties from row 150 000 on: chunk 2 is detected lossy on the host, is sent
    # again as float64, and the rest of the call stays float64
    Xm = Xi.copy()
    Xm[150_000:] = planted_near_ties(rng, coef, intercept, N - 150_000)
    want = olin.predict_indices(olin.decision_function(Xm, coef, intercept)).astype(np.int32)
    rounded = olin.predict_indices(olin.decision_function(Xm.astype(np.float32).astype(np.float64), coef, intercept))
    assert (rounded != want).sum() > 1000
    for name, arr in {"c_order": Xm, "f_order": np.asfortranarray(Xm)}.items():
        idx, st = engine.predict_host(m, arr, exact=True, chunk_rows=chunk)
        np.testing.assert_array_equal(idx, want, err_msg=name)
        assert st["h2d_bytes"] == 2 * chunk * 12 * 4 + (N - 2 * chunk) * 12 * 8, name
    # a NaN is "not lossless" for the gather threads: the chunk travels as float64 and the staging kernel reports it
    Xn = Xi.copy()
    Xn[77, 3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        engine.predict_host(m, np.asfortranarray(Xn), exact=True, chunk_rows=chunk)


def test_mnist_scaled_float64_frame_one_million(engine):
    """cfg 3's real-world shape: pixels / 255 as float64 (not fp32-representable), 784 features, through linear_argmax."""
    from unionml_b200.predictors import linear_argmax

    rng = np.random.default_rng(1)
    coef = rng.standard_normal((10, 784)) * 0.05
    intercept = np.random.default_rng(2).standard_normal(10)
    N = 1_000_000
    X = np.empty((784, N), dtype=np.float64)  # feature-major, as a pandas block holds it
    for f0 in range(0, 784, 98):
        X[f0 : f0 + 98] = rng.integers(0, 256, size=(98, N)) / 255.0
    frame = pd.DataFrame(X.T, columns=[f"p{i}" for i in range(784)], copy=False)
    est = _estimator(coef, intercept)
    est.feature_names_in_ = np.asarray(frame.columns, dtype=object)
    want = est.predict(frame)
    got = linear_argmax(est, frame)
    assert len(got) == N and isinstance(got[0], float)
    np.testing.assert_array_equal(np.asarray(got), want.astype(np.float64))


def test_online_shape_small_batches(engine, digits_model):
    """<= 64 rows: path 4 (one float64 kernel, CUDA graph replay), every dtype / order, NaN contract kept."""
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    m = engine.load_linear(coef, intercept)
    rng = np.random.default_rng(3)
    for rows in (1, 2, 32, 64):
        base = rng.integers(0, 17, size=(rows, 64)).astype(np.float64)
        want = olin.predict_indices(olin.decision_function(base, coef, intercept)).astype(np.int32)
        frame = pd.DataFrame(base, columns=[f"pixel_{i}" for i in range(64)])
        for arr in (base, base.astype(np.float32), np.asfortranarray(base), base.astype(np.int64), base.astype(np.uint8), frame):
            for _ in range(3):  # first call captures the graph, the next ones replay it
                idx, st = engine.predict_host(m, arr, exact=True)
                np.testing.assert_array_equal(idx, want)
                assert st["path"] == 4 and st["kernel_launches"] == 1
        vals, _ = engine.predict_host_values(m, frame, np.arange(10, dtype=np.float64) * 1.5)
        np.testing.assert_array_equal(vals, want * 1.5)
    bad = rng.integers(0, 17, size=(32, 64)).astype(np.float64)
    bad[5, 7] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        engine.predict_host(m, bad, exact=True)
    idx, st = engine.predict_host(m, np.zeros((65, 64), dtype=np.float32))  # one row more: the tile route
    assert st["path"] == 1
    # a re-uploaded model (affine fold) must not replay a graph that points at the old operands
    X = rng.integers(0, 17, size=(32, 64)).astype(np.float64)
    before, _ = engine.predict_host(m, X)
    mu = X.mean(axis=0)
    m.set_affine(shift=mu, scale=np.full(64, 0.5))
    after, _ = engine.predict_host(m, X)
    want = olin.predict_indices(olin.decision_function((X - mu) * 0.5, coef, intercept)).astype(np.int32)
    np.testing.assert_array_equal(after, want)


def test_large_frames_build_the_list_while_the_batch_is_in_flight(engine, digits_model):
    """>= 1M rows: ``linear_argmax`` runs the pipeline on a library thread (``uml_linear_predict_host_begin``) and fills
    the finished prefix into the list meanwhile (one shared Python float per class, ``csrc_host/uml_pylist.c``).
    Same labels; NaN still raises; the engine is usable after."""
    from unionml_b200.predictors import linear_argmax

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    est = _estimator(coef, intercept, digits_model["classes"])
    N = 1_300_003
    X = np.random.default_rng(17).integers(0, 17, size=(64, N)).astype(np.float64)  # feature-major block
    frame = pd.DataFrame(X.T, columns=[f"pixel_{i}" for i in range(64)], copy=False)
    est.feature_names_in_ = np.asarray(frame.columns, dtype=object)
    want = est.predict(frame).astype(np.float64)
    for _ in range(2):
        got = linear_argmax(est, frame)
        assert isinstance(got, list) and len(got) == N and isinstance(got[0], float)
        np.testing.assert_array_equal(np.asarray(got), want)
    table = [float(c) * 2.0 for c in range(10)]
    for asynchronous in (True, False):
        out, st = engine.predict_host_list(engine.load_linear(coef, intercept), X.T, table, chunk_rows=8192, asynchronous=asynchronous)
        np.testing.assert_array_equal(np.asarray(out), want * 2.0)
        assert st["n_rows"] == N and all(type(v) is float for v in out[:100])
    bad = X.T.copy()
    bad[N // 2, 5] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        linear_argmax(est, pd.DataFrame(bad, columns=frame.columns))
    assert linear_argmax(est, frame.iloc[:1000]) == want[:1000].tolist()


def test_values_route_equals_take(engine, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    classes = np.array([3.0, 1.5, -2.0, 7.0, 9.0, 11.0, 0.0, 4.0, 5.0, 6.0])
    m = engine.load_linear(coef, intercept)
    X = np.random.default_rng(21).integers(0, 17, size=(300_001, 64)).astype(np.float64)
    want = classes[olin.predict_indices(olin.decision_function(X, coef, intercept))]
    vals, st = engine.predict_host_values(m, np.asfortranarray(X), classes, chunk_rows=50_000)
    np.testing.assert_array_equal(vals, want)
    assert st["d2h_bytes"] == 8 * X.shape[0]


def test_predict_proba_against_sklearn(engine, digits_model):
    """fp32 scores + fp32 softmax vs scikit-learn's float64: the error of a probability is at most the fp32 score
    error, (F+4) 2^-24 (|b| + sum |x w|) - stated per row below - plus ~1e-6 of fp32 exp/normalisation."""
    from unionml_b200.predictors import linear_predict_proba

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    est = _estimator(coef, intercept, digits_model["classes"])
    X = np.random.default_rng(4).integers(0, 17, size=(100_003, 64)).astype(np.float64)
    want = est.predict_proba(X)
    got = linear_predict_proba(est, X)
    assert got.shape == want.shape and got.dtype == np.float32
    A = np.abs(intercept).max() + np.abs(X) @ np.abs(coef).max(axis=0)
    bound = 2 * 68 * 2.0**-24 * A + 2e-6
    assert np.all(np.abs(got - want).max(axis=1) <= bound)
    np.testing.assert_allclose(got.sum(axis=1), 1.0, atol=1e-6)
    # well-scaled inputs: 2e-6 absolute
    Xs = X / 16.0
    np.testing.assert_allclose(linear_predict_proba(est, Xs), est.predict_proba(Xs), atol=2e-6, rtol=0)
    # binary model: columns [1 - p, p] of _predict_proba_lr
    rng = np.random.default_rng(8)
    est2 = _estimator(rng.standard_normal((1, 20)), rng.standard_normal(1), classes=[0, 1])
    Xb = rng.standard_normal((10_000, 20))
    np.testing.assert_allclose(linear_predict_proba(est2, Xb), est2.predict_proba(Xb), atol=2e-6, rtol=0)
    # more classes than the register-tiled kernel takes
    est3 = _estimator(rng.standard_normal((40, 20)), rng.standard_normal(40))
    np.testing.assert_allclose(linear_predict_proba(est3, Xb), est3.predict_proba(Xb), atol=2e-6, rtol=0)


def test_predictor_contract_errors():
    from sklearn.linear_model import LinearRegression

    from unionml_b200.predictors import linear_argmax

    reg = LinearRegression()
    reg.coef_, reg.intercept_ = np.ones(4), 0.0
    with pytest.raises(TypeError, match="classifier"):
        linear_argmax(reg, np.zeros((3, 4)))
    est = _estimator(np.ones((3, 4)), np.zeros(3))
    with pytest.raises(ValueError, match="0 sample"):
        linear_argmax(est, np.zeros((0, 4)))


def _digits_app(predictor_body):
    from sklearn.datasets import load_digits
    from sklearn.linear_model import LogisticRegression

    from unionml_b200 import Dataset, Model

    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="digits_classifier", init=LogisticRegression, dataset=dataset)

    @dataset.reader
    def reader(sample_frac: float = 1.0, random_state: int = 0) -> pd.DataFrame:
        return load_digits(as_frame=True).frame.sample(frac=sample_frac, random_state=random_state)

    @model.trainer
    def trainer(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> LogisticRegression:
        return estimator.fit(features, target.squeeze())

    @model.predictor
    def predictor(estimator: LogisticRegression, features: pd.DataFrame) -> List[float]:
        return predictor_body(estimator, features)

    @model.evaluator
    def evaluator(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> float:
        return float((estimator.predict(features) == target.squeeze()).mean())

    return dataset, model


def test_reader_kwargs_route_and_runnable_on_the_device_predictor():
    """SURVEY 8 rows a4 (predict(**reader_kwargs): reader -> parser -> transformer -> predictor, model.py:603-614 with
    the parser quirk of dataset.py:498-499) and a9 (UnionMLRunnable.predict, services/bentoml.py:208-211)."""
    from sklearn.datasets import load_digits

    from unionml_b200.predictors import linear_argmax
    from unionml_b200.services import PredictRunnable, create_runnable

    _, model = _digits_app(linear_argmax)
    est, _ = model.train(hyperparameters={"C": 1.0, "max_iter": 1000}, sample_frac=1.0, random_state=123)
    frame = load_digits(as_frame=True).frame
    feats = [c for c in frame if c != "target"]
    # a4: reader kwargs -> the whole (shuffled) frame through the device predictor
    from_reader = model.predict(sample_frac=0.5, random_state=7)
    sample = frame.sample(frac=0.5, random_state=7)
    assert from_reader == [float(v) for v in est.predict(sample[feats])]
    assert all(isinstance(v, float) for v in from_reader)
    # a9: the runnable call site (get_features twice, then Model.predict) on records and on a frame
    runnable = create_runnable()(model)
    assert isinstance(runnable, PredictRunnable)
    records = frame[feats].sample(32, random_state=11).to_dict(orient="records")
    assert runnable.predict(records) == [float(v) for v in est.predict(frame[feats].sample(32, random_state=11))]
    big = frame[feats].sample(1500, random_state=12)
    assert runnable.predict(big) == [float(v) for v in est.predict(big)]
