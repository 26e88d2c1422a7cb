"""Pin the oracle: reference known-answer vectors, committed fixtures, and scikit-learn itself (CPU only)."""
import numpy as np
import pandas as pd
import pytest
from sklearn.linear_model import LogisticRegression

from oracle import linear as olin
from oracle import unionml_path as opath


def _estimator(m, dtype=np.float64):
    est = LogisticRegression()
    est.coef_ = m["coef"].astype(dtype)
    est.intercept_ = m["intercept"].astype(dtype)
    est.classes_ = m["classes"]
    est.n_features_in_ = m["coef"].shape[1]
    return est


def test_known_answer_lambda_handler(digits_model, known_answer):
    # unionml:tests/unit/test_aws_lambda_handler.py:127,159
    ka = known_answer["sample3_random_state99"]
    frame = pd.DataFrame(ka["records"])[known_answer["feature_names"]]
    got = olin.canonical_predictor(_estimator(digits_model), frame)
    assert got == [8.0, 8.0, 0.0] == ka["expected"]
    assert all(isinstance(x, float) for x in got)


def test_known_answer_quickstart(digits_model, known_answer):
    ka = known_answer["sample5_random_state42"]
    frame = pd.DataFrame(ka["records"])[known_answer["feature_names"]]
    assert olin.canonical_predictor(_estimator(digits_model), frame) == [6.0, 9.0, 3.0, 7.0, 2.0]


def test_fixture_labels_f64(digits_model, synthetic_digits):
    X = synthetic_digits["X"].astype(np.float64)
    got = olin.predict(X, digits_model["coef"], digits_model["intercept"], digits_model["classes"])
    np.testing.assert_array_equal(got, synthetic_digits["labels_f64"])
    # exact rational arithmetic agrees with the float64 path on these rows (margins >> 1e-13)
    idx = olin.exact_predict_indices(X[:64], digits_model["coef"], digits_model["intercept"])
    np.testing.assert_array_equal(digits_model["classes"][idx], synthetic_digits["labels_f64"][:64])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_equals_sklearn(digits_model, dtype, seed):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 17, size=(20000, 64)).astype(dtype)
    est = _estimator(digits_model, dtype)
    want = est.predict(X)
    got = olin.predict(X, est.coef_, est.intercept_, est.classes_)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(olin.decision_function(X, est.coef_, est.intercept_), est.decision_function(X))


def test_binary_rule(binary_mock):
    got = olin.predict(binary_mock["X"], binary_mock["coef"], binary_mock["intercept"], binary_mock["classes"])
    np.testing.assert_array_equal(got, binary_mock["labels"])
    # scores exactly 0 -> class 0 (strict >), _base.py:416
    z = olin.predict(np.zeros((2, 1)), np.array([[1.0]]), np.array([0.0]), np.array([5, 7]))
    np.testing.assert_array_equal(z, [5, 5])


def test_tie_rule_first_max():
    coef = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0]])
    X = np.array([[2.0, 1.0], [1.0, 2.0], [1.0, 1.0]])
    np.testing.assert_array_equal(olin.predict(X, coef, np.zeros(3), np.arange(3)), [0, 2, 0])
    np.testing.assert_array_equal(olin.exact_predict_indices(X, coef, np.zeros(3)), [0, 2, 0])


def test_validation_errors(digits_model):
    m = digits_model
    bad = np.zeros((3, 64))
    bad[1, 5] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        olin.predict(bad, m["coef"], m["intercept"], m["classes"])
    bad[1, 5] = np.inf
    with pytest.raises(ValueError, match="infinity"):
        olin.predict(bad, m["coef"], m["intercept"], m["classes"])
    with pytest.raises(ValueError, match="63 features"):
        olin.predict(np.zeros((3, 63)), m["coef"], m["intercept"], m["classes"])
    # sklearn raises the same family
    est = _estimator(m)
    with pytest.raises(ValueError):
        est.predict(bad)
    with pytest.raises(ValueError):
        est.predict(np.zeros((3, 63)))


# ---------------------------------------------------------------------------------------------------------------
# wrapper restatement (dataset.py / model.py / fastapi.py semantics)
# ---------------------------------------------------------------------------------------------------------------
def _spec(digits_model, **kw):
    def reader() -> pd.DataFrame:  # annotation drives dataset_datatype (dataset.py:368-382)
        raise AssertionError("not called")

    return opath.PathSpec(
        reader=reader,
        targets=["target"],
        predictor=olin.canonical_predictor,
        model_object=_estimator(digits_model),
        **kw,
    )


def test_wrapper_predict_from_features(digits_model, known_answer):
    ka = known_answer["sample3_random_state99"]
    spec = _spec(digits_model)
    assert opath.predict(spec, features=ka["records"]) == [8.0, 8.0, 0.0]
    # FastAPI body: get_features twice is idempotent (fastapi.py:61 + model.py:740)
    assert opath.serving_predict(spec, features=ka["records"]) == [8.0, 8.0, 0.0]
    with pytest.raises(LookupError):
        opath.serving_predict(spec)


def test_wrapper_errors_and_callbacks(digits_model, known_answer, caplog):
    ka = known_answer["sample3_random_state99"]
    seen = []

    def good(model_object, features, predictions):
        seen.append((features.shape, list(predictions)))

    def bad(model_object, features, predictions):
        raise RuntimeError("boom")

    spec = _spec(digits_model, callbacks=(bad, good))
    assert opath.predict(spec, features=ka["records"]) == [8.0, 8.0, 0.0]
    assert seen == [((3, 64), [8.0, 8.0, 0.0])]
    assert "boom" in caplog.text
    with pytest.raises(ValueError):
        opath.predict(spec)
    spec.model_object = None
    with pytest.raises(RuntimeError):
        opath.predict(spec, features=ka["records"])


def test_parser_quirk():
    # dataset.py:498-499: explicit features are replaced by "all non-target columns" when targets is not None
    df = pd.DataFrame({"x": [1, 2], "x2": [3, 4], "y": [0, 1]})
    spec = opath.PathSpec(features=["x"], targets=["y"])
    feats, targ = opath.default_parser(spec, df, ["x"], ["y"])
    assert list(feats.columns) == ["x", "x2"] and list(targ.columns) == ["y"]

    def reader() -> pd.DataFrame:
        return df

    spec.reader = reader
    # ...while the feature loader honours the explicit list (dataset.py:515-518)
    assert list(opath.default_feature_loader(spec, df).columns) == ["x"]


def test_mlp_oracle_pinned_to_torch():
    """oracle.mlp against torch itself (the reference predictor as written) and the committed fixture."""
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    from oracle import mlp as omlp
    from tests.conftest import GOLDEN

    z = np.load(GOLDEN / "mlp_64_32_10.npz")
    w = (z["w1"], z["b1"], z["w2"], z["b2"])
    np.testing.assert_array_equal(omlp.predict_indices_f32(z["X"], *w), z["labels_torch"])
    np.testing.assert_array_equal(omlp.predict_indices_f64(z["X"], *w), z["labels_torch"])

    layers = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))
    with torch.no_grad():
        layers[0].weight.copy_(torch.from_numpy(z["w1"]))
        layers[0].bias.copy_(torch.from_numpy(z["b1"]))
        layers[2].weight.copy_(torch.from_numpy(z["w2"]))
        layers[2].bias.copy_(torch.from_numpy(z["b2"]))
        X = np.random.default_rng(11).integers(0, 17, size=(50_000, 64)).astype(np.float64)
        want = F.softmax(layers(torch.from_numpy(X).float()), dim=1).argmax(1).numpy()
    got = omlp.predict_indices_f64(X, *w)
    mism = np.flatnonzero(got != want)
    assert len(mism) <= 2 and np.all(omlp.logit_margin_f64(X, *w)[mism] < 1e-4)
    assert omlp.canonical_predictor({"w1": w[0], "b1": w[1], "w2": w[2], "b2": w[3]}, pd.DataFrame(X[:5])) == [
        float(v) for v in want[:5]
    ]


def test_c_restatement_matches_numpy_and_sklearn(digits_model, synthetic_digits, binary_mock):
    """oracle/linear_predict.c (plain C, float64) against the numpy restatement, sklearn's labels and the fixtures."""
    from oracle import c_port

    c_port.build()
    coef, intercept, classes = digits_model["coef"], digits_model["intercept"], digits_model["classes"]
    X = synthetic_digits["X"]
    for arr in (X.astype(np.float64), X.astype(np.float32)):
        idx = c_port.predict_indices(arr, coef, intercept)
        np.testing.assert_array_equal(classes[idx], synthetic_digits["labels_f64"])
    big = np.random.default_rng(5).integers(0, 17, size=(200_000, 64)).astype(np.float64)
    want = olin.predict_indices(olin.decision_function(big, coef, intercept))
    np.testing.assert_array_equal(c_port.predict_indices(big, coef, intercept), want)
    np.testing.assert_array_equal(_estimator(digits_model).predict(big[:5000]), classes[want[:5000]])
    got = c_port.predict_indices(binary_mock["X"], binary_mock["coef"], binary_mock["intercept"])
    np.testing.assert_array_equal(binary_mock["classes"][got], binary_mock["labels"])
    ties = c_port.predict_indices(np.array([[2.0, 1.0], [1.0, 1.0]]), np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0]]), np.zeros(3))
    np.testing.assert_array_equal(ties, [0, 0])
    assert c_port.num_threads() >= 1
