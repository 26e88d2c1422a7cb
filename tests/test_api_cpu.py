"""Host-side logic on CPU: the decorator API mirror behaves like the reference's (no GPU, no flytekit).

Modelled on unionml:tests/unit/{test_model.py,test_dataset.py,test_type_guards.py} and
unionml:tests/integration/test_fastapi.py.  The predictors registered here are the reference's CPU
predictors (sklearn called directly) - the device predictor has its own `-m gpu` tests.
"""
import io
import typing
from typing import Any, List

import numpy as np
import pandas as pd
import pytest
from sklearn.datasets import load_digits
from sklearn.linear_model import LogisticRegression
from sklearn.metrics import accuracy_score

from oracle import linear as olin
from oracle import unionml_path as opath
from unionml_b200 import Dataset, Model, ModelArtifact, type_guards


# fixtures shaped like unionml:tests/unit/model_fixtures.py:12-82
@pytest.fixture
def mock_data() -> pd.DataFrame:
    return pd.DataFrame({"x": [1, 2, 3, 4] * 25, "x2": [1, 2, 3, 4] * 25, "x3": [1, 2, 3, 4] * 25, "y": [0, 1, 0, 1] * 25})


@pytest.fixture(params=[True, False])
def model(request, mock_data) -> Model:
    dataset = Dataset(features=["x"], targets=["y"], test_size=0.2, shuffle=True, random_state=123)

    @dataset.reader
    def reader(sample_frac: float, random_state: int) -> pd.DataFrame:
        return mock_data.sample(frac=sample_frac, random_state=random_state)

    @dataset.loader
    def loader(raw_data: pd.DataFrame, head: typing.Optional[int] = None) -> pd.DataFrame:
        return raw_data if head is None else raw_data.head(head)

    m = Model(
        name="test_model",
        init=None if request.param else LogisticRegression,
        hyperparameter_config={"C": float, "max_iter": int},
        dataset=dataset,
    )
    if request.param:

        @m.init
        def init_fn(hyperparameters: dict) -> LogisticRegression:
            return LogisticRegression(**hyperparameters)

    @m.trainer
    def trainer(model: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> LogisticRegression:
        return model.fit(features, target.squeeze())

    @m.predictor
    def predictor(model: LogisticRegression, features: pd.DataFrame) -> List[float]:
        return [float(x) for x in model.predict(features)]

    @m.evaluator
    def evaluator(model: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> float:
        return float(accuracy_score(target, model.predict(features)))

    return m


def test_model_decorators(model):
    assert model._trainer.__name__ == "trainer" and model._predictor.__name__ == "predictor"
    assert model.model_type is LogisticRegression
    assert model.prediction_type == List[float]
    assert model._dataset.feature_type is pd.DataFrame


def test_model_train_and_predict(model, mock_data):
    model_object, metrics = model.train(hyperparameters={"C": 1.0, "max_iter": 1000}, sample_frac=1.0, random_state=123)
    assert isinstance(model_object, LogisticRegression)
    assert isinstance(metrics["train"], float) and isinstance(metrics["test"], float)
    # reader path and features path agree (ref. tests/unit/test_model.py:95-109)
    from_reader = model.predict(sample_frac=1.0, random_state=123)
    assert all(isinstance(x, float) for x in from_reader) and len(from_reader) == 100


def test_predict_from_features_matches_direct_call(model, mock_data):
    model_object = LogisticRegression().fit(mock_data[["x"]], mock_data["y"])
    model.artifact = ModelArtifact(model_object)
    predictions = model.predict(features=mock_data[["x"]])
    assert predictions == [float(x) for x in model_object.predict(mock_data[["x"]])]
    # the restated reference wrapper gives the same list
    spec = opath.PathSpec(
        reader=model._dataset._reader, features=["x"], targets=["y"], predictor=model._predictor, model_object=model_object
    )
    assert opath.predict(spec, features=mock_data[["x"]]) == predictions


def test_predict_errors(model, mock_data):
    with pytest.raises(RuntimeError, match="ModelArtifact not found"):
        model.predict(features=mock_data[["x"]])
    model.artifact = ModelArtifact(LogisticRegression().fit(mock_data[["x"]], mock_data["y"]))
    with pytest.raises(ValueError, match="At least one of features"):
        model.predict()


def test_callbacks_run_and_errors_are_swallowed(mock_data, caplog):
    dataset = Dataset(features=["x"], targets=["y"])

    @dataset.reader
    def reader() -> pd.DataFrame:
        return mock_data

    m = Model(init=LogisticRegression, dataset=dataset)
    seen = []

    def ok_cb(model_obj: LogisticRegression, features: pd.DataFrame, predictions: List[float]):
        seen.append(len(predictions))

    def bad_cb(model_obj: LogisticRegression, features: pd.DataFrame, predictions: List[float]) -> None:
        raise RuntimeError("boom")

    @m.predictor(callbacks=[bad_cb, ok_cb])
    def predictor(model_obj: LogisticRegression, features: pd.DataFrame) -> List[float]:
        return [float(x) for x in model_obj.predict(features)]

    m.artifact = ModelArtifact(LogisticRegression().fit(mock_data[["x"]], mock_data["y"]))
    out = m.predict(features=mock_data[["x"]])
    assert len(out) == 100 and seen == [100]
    assert "boom" in caplog.text

    with pytest.raises(TypeError):  # wrong arity (ref. type_guards.py:192-195)

        @m.predictor(callbacks=[lambda a, b: None])
        def p2(model_obj: LogisticRegression, features: pd.DataFrame) -> List[float]:
            return []

    with pytest.raises(ValueError):
        m.predictor(predictor, callbacks=["not callable"])


def test_type_guards():
    def reader_no_annotation():
        return 1

    with pytest.raises(TypeError):
        type_guards.guard_reader(reader_no_annotation)

    def pred_ok(m: LogisticRegression, f: pd.DataFrame) -> List[float]:
        return []

    type_guards.guard_predictor(pred_ok, LogisticRegression, pd.DataFrame)
    type_guards.guard_predictor(pred_ok, LogisticRegression, Any)

    def pred_two_args(m: LogisticRegression, f: pd.DataFrame, g: pd.DataFrame) -> List[float]:
        return []

    def pred_no_return(m: LogisticRegression, f: pd.DataFrame):
        return []

    def pred_wrong_model(m: int, f: pd.DataFrame) -> List[float]:
        return []

    for bad in (pred_two_args, pred_no_return, pred_wrong_model):
        with pytest.raises(TypeError):
            type_guards.guard_predictor(bad, LogisticRegression, pd.DataFrame)

    with pytest.raises(TypeError):
        type_guards.guard_feature_loader(lambda a, b: a, Any)
    with pytest.raises(TypeError):
        type_guards.guard_feature_transformer(lambda a, b: a, Any)

    def cb_returns(m: LogisticRegression, f: pd.DataFrame, p: List[float]) -> int:
        return 1

    with pytest.raises(TypeError):
        type_guards.guard_prediction_callback(cb_returns, pred_ok, LogisticRegression, pd.DataFrame)


def test_dataset_defaults_and_quirk(mock_data):
    ds = Dataset(features=["x"], targets=["y"])

    @ds.reader
    def reader() -> pd.DataFrame:
        return mock_data

    # feature loader honours the explicit list (ref. dataset.py:515-518) ...
    assert list(ds.get_features(mock_data.to_dict(orient="records")).columns) == ["x"]
    # ... the parser replaces it with all non-target columns (ref. dataset.py:498-499)
    feats, targ = ds._default_parser(mock_data, **ds.parser_kwargs)
    assert list(feats.columns) == ["x", "x2", "x3"] and list(targ.columns) == ["y"]
    data = ds.get_data(mock_data)
    assert set(data) == {"train", "test"} and len(data["test"][0]) == 20

    @ds.feature_transformer
    def scale(features: pd.DataFrame) -> pd.DataFrame:
        return features * 2.0

    assert ds.get_features(mock_data[["x"]])["x"].iloc[1] == 4.0
    assert ds.splitter_kwargs == {"test_size": 0.2, "shuffle": True, "random_state": 12345}


def test_feature_loader_from_json_path(tmp_path, mock_data):
    ds = Dataset(targets=["y"])

    @ds.reader
    def reader() -> pd.DataFrame:
        return mock_data

    p = tmp_path / "features.json"
    mock_data.head(3).to_json(p, orient="records")
    got = ds.get_features(p)
    assert list(got.columns) == ["x", "x2", "x3"] and len(got) == 3


def test_save_load_roundtrip(model, tmp_path):
    model_obj, _ = model.train(hyperparameters={"C": 1.0, "max_iter": 1000}, sample_frac=1.0, random_state=42)
    path = tmp_path / "model.joblib"
    out, *_ = model.save(path)
    assert out == str(path)
    assert model.load(path).get_params() == model_obj.get_params()
    buf = io.BytesIO()
    model.save(buf)
    buf.seek(0)
    assert model.load(buf).get_params() == model_obj.get_params()
    with pytest.raises(ValueError):
        model.resolve_model_artifact(model_object=1, model_file="x")


# ---- the README digits app (BASELINE.json configs[0]) through the API shell with a CPU predictor ----------------
def _digits_app():
    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="digits_classifier", init=LogisticRegression, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return load_digits(as_frame=True).frame

    @model.trainer
    def trainer(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> LogisticRegression:
        return estimator.fit(features, target.squeeze())

    @model.predictor
    def predictor(estimator: LogisticRegression, features: pd.DataFrame) -> List[float]:
        return [float(x) for x in estimator.predict(features)]

    @model.evaluator
    def evaluator(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> float:
        return float(accuracy_score(target.squeeze(), predictor(estimator, features)))

    return dataset, model


@pytest.fixture(scope="module")
def digits_app():
    dataset, model = _digits_app()
    model.train(hyperparameters={"C": 1.0, "max_iter": 1000})
    return dataset, model


def test_digits_app_known_answers(digits_app, digits_model):
    _, model = digits_app
    frame = load_digits(as_frame=True).frame
    feats = [c for c in frame if c != "target"]
    # unionml:tests/unit/test_aws_lambda_handler.py:127 and quickstart sample
    assert model.predict(features=frame[feats].sample(3, random_state=99)) == [8.0, 8.0, 0.0]
    assert model.predict(features=frame.sample(5, random_state=42)) == [6.0, 9.0, 3.0, 7.0, 2.0]
    # the app trains the very model stored in tests/golden/digits_lr.npz
    np.testing.assert_allclose(model.artifact.model_object.coef_, digits_model["coef"], rtol=0, atol=1e-12)
    assert model.artifact.metrics["train"] == 1.0 and abs(model.artifact.metrics["test"] - 0.9639) < 1e-3
    # no features and a reader without arguments: the reference refuses (model.py:727-728) - so does the mirror
    with pytest.raises(ValueError, match="At least one of features"):
        model.predict()


def test_fastapi_predict_and_health(digits_app, tmp_path, monkeypatch):
    from fastapi import FastAPI
    from fastapi.testclient import TestClient

    _, trained = digits_app
    path = tmp_path / "model.joblib"
    trained.save(path)

    _, fresh = _digits_app()
    app = FastAPI()
    fresh.serve(app)
    monkeypatch.setenv("UNIONML_MODEL_PATH", str(path))
    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    with TestClient(app) as client:
        assert client.get("/health").json()["message"] == "OK"
        r = client.post("/predict", json={"features": feats.sample(5, random_state=42).to_dict(orient="records")})
        assert r.status_code == 200 and r.json() == [6.0, 9.0, 3.0, 7.0, 2.0]
        assert client.post("/predict", json={}).status_code == 500  # ref. fastapi.py:55-56
        assert "unionml" in client.get("/").text


def test_fastapi_no_model_fails_startup(monkeypatch):
    from fastapi import FastAPI
    from fastapi.testclient import TestClient

    _, fresh = _digits_app()
    app = FastAPI()
    fresh.serve(app)
    monkeypatch.delenv("UNIONML_MODEL_PATH", raising=False)
    with pytest.raises(ValueError, match="Model artifact path not specified"):
        with TestClient(app):
            pass


def test_runnable_calls_get_features_then_predict(digits_app):
    from unionml_b200.services import PredictRunnable, create_runnable

    _, model = digits_app
    frame = load_digits(as_frame=True).frame
    r = create_runnable(supports_cpu_multi_threading=True)(model)
    assert isinstance(r, PredictRunnable) and r.SUPPORTS_CPU_MULTI_THREADING
    assert r.predict(frame.sample(5, random_state=42).to_dict(orient="records")) == [6.0, 9.0, 3.0, 7.0, 2.0]


def test_device_predictor_satisfies_the_guard_and_fails_loudly_without_gpu(digits_app):
    import torch

    from unionml_b200.predictors import linear_argmax

    dataset, _ = _digits_app()
    m = Model(name="gpu_digits", init=LogisticRegression, dataset=dataset)
    m.predictor(linear_argmax)  # guard_predictor accepts it (one features arg, return annotation)
    assert m.prediction_type == List[float]
    if not torch.cuda.is_available():
        _, trained = digits_app
        m.artifact = trained.artifact
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m.predict(features=load_digits(as_frame=True).frame.sample(3, random_state=99))


def test_feature_array_borrowing():
    from unionml_b200.engine import as_feature_array

    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    arr = as_feature_array(feats)
    assert arr.shape == (1797, 64) and arr.dtype == np.float64
    rs, cs = arr.strides
    assert cs == 8 or rs == 8  # contiguous along one axis: staged without a host copy
    assert as_feature_array(np.arange(12, dtype=np.int16).reshape(3, 4)).dtype == np.float64
    with pytest.raises(ValueError, match="Expected 2D array"):
        as_feature_array(np.arange(4.0))
    sliced = np.arange(64, dtype=np.float32).reshape(8, 8)[::2, ::2]
    assert as_feature_array(sliced).flags.c_contiguous
    assert olin.validate_features(as_feature_array(sliced), 4).shape == (4, 4)


def test_cli_serve_sets_model_path_and_starts_uvicorn(monkeypatch, tmp_path):
    """`serve` = uvicorn + --model-path exported as UNIONML_MODEL_PATH (ref. cli.py:285-320)."""
    import uvicorn

    from unionml_b200 import cli

    calls = {}
    monkeypatch.setattr(uvicorn, "run", lambda app, **kw: calls.update(app=app, **kw))
    model_file = tmp_path / "m.joblib"
    model_file.write_bytes(b"x")
    monkeypatch.delenv("UNIONML_MODEL_PATH", raising=False)
    assert cli.main(["serve", "app:app", "--model-path", str(model_file), "--port", "8123"]) == 0
    import os

    assert os.environ["UNIONML_MODEL_PATH"] == str(model_file)
    assert calls["app"] == "app:app" and calls["port"] == 8123
    with pytest.raises(SystemExit):
        cli.main(["serve", "app:app", "--model-path", str(tmp_path / "missing.joblib")])


def test_predictor_host_checks_without_a_gpu():
    """Validation that runs before the device is touched: fitted-ness, feature names, pipeline unwrapping."""
    from sklearn.exceptions import NotFittedError
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler, StandardScaler

    from unionml_b200 import predictors as P

    with pytest.raises(NotFittedError):
        P._check_fitted(LogisticRegression())
    frame = load_digits(as_frame=True).frame
    X, y = frame[[c for c in frame if c != "target"]], frame["target"]
    est = LogisticRegression(max_iter=200).fit(X.iloc[:300], y.iloc[:300])
    P._check_fitted(est)
    P._check_feature_names(est, X.iloc[:3])  # same names, same order: fine
    with pytest.raises(ValueError, match="feature names"):
        P._check_feature_names(est, X.iloc[:3, ::-1])
    with pytest.raises(ValueError, match="feature names"):
        P._check_feature_names(est, X.iloc[:3, :10])
    P._check_feature_names(est, X.iloc[:3].to_numpy())  # ndarray: nothing to check, like sklearn

    pipe = Pipeline([("scale", StandardScaler()), ("clf", LogisticRegression(max_iter=200))]).fit(X.iloc[:300], y.iloc[:300])
    clf, shift, scale = P.unwrap_pipeline(pipe)
    assert clf is pipe.named_steps["clf"]
    np.testing.assert_array_equal(shift, pipe.named_steps["scale"].mean_)
    np.testing.assert_allclose(scale, 1.0 / pipe.named_steps["scale"].scale_)
    # folding (x - shift) * scale into W, b reproduces the pipeline's decision function
    Xs = X.iloc[300:400].to_numpy()
    folded_w = clf.coef_ * scale
    folded_b = clf.intercept_ - folded_w @ shift
    np.testing.assert_allclose(Xs @ folded_w.T + folded_b, pipe.decision_function(X.iloc[300:400]), rtol=1e-10, atol=1e-10)
    assert P.unwrap_pipeline(est) == (est, None, None)
    no_mean = Pipeline([("s", StandardScaler(with_mean=False)), ("c", LogisticRegression(max_iter=50))]).fit(X.iloc[:200], y.iloc[:200])
    _, shift2, scale2 = P.unwrap_pipeline(no_mean)
    assert shift2 is None and scale2 is not None
    with pytest.raises(TypeError, match="StandardScaler"):
        P.unwrap_pipeline(Pipeline([("m", MinMaxScaler()), ("c", LogisticRegression())]))


def test_mlp_layer_extraction():
    import torch.nn as nn

    from unionml_b200.predictors import _mlp_layers

    class Net(nn.Module):  # the reference's PytorchModel layout (quickstart.py:14-24)
        def __init__(self):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))

    l1, l2 = _mlp_layers(Net())
    assert l1.weight.shape == (32, 64) and l2.weight.shape == (10, 32)
    with pytest.raises(TypeError, match="Linear -> ReLU -> Linear"):
        _mlp_layers(nn.Sequential(nn.Linear(4, 4), nn.Tanh(), nn.Linear(4, 2)))
    with pytest.raises(TypeError):
        _mlp_layers(nn.Linear(4, 2))


def test_predictor_contract_checks_and_bookkeeping_without_a_gpu():
    """Host-side guards of the drop-in predictor that never reach the device: classifier-only, dense weights, sklearn's
    empty-batch error, the weights cache key (identity + fingerprints, no hashing per request) and the counters the
    predictor publishes after a call."""
    import warnings

    from sklearn.linear_model import LinearRegression, Ridge

    from unionml_b200 import predictors as P

    X = np.random.default_rng(0).standard_normal((40, 5))
    y = (X[:, 0] > 0).astype(int)
    clf = LogisticRegression().fit(X, y)
    P._check_linear_classifier(clf)
    for reg in (LinearRegression().fit(X, X[:, 1]), Ridge().fit(X, X[:, 1])):
        with pytest.raises(TypeError, match="classifiers"):
            P._check_linear_classifier(reg)
    sparse = LogisticRegression().fit(X, y).sparsify()
    with pytest.raises(TypeError, match="dense"):
        P._check_linear_classifier(sparse)

    with pytest.raises(ValueError, match=r"0 sample\(s\)"):
        P._check_min_samples(np.empty((0, 5)))
    with pytest.raises(ValueError, match=r"0 sample\(s\)"):
        P._check_min_samples(pd.DataFrame(np.empty((0, 5))))
    P._check_min_samples(X)

    k1 = P._weights_key(clf, None, None)
    assert k1 == P._weights_key(clf, None, None)           # same arrays: same key, nothing hashed
    clf.coef_ = clf.coef_.copy()                            # what `fit` does: rebinding is seen
    assert P._weights_key(clf, None, None) != k1
    k2 = P._weights_key(clf, None, None)
    clf.coef_[0, 0] += 1.0                                  # in-place edit of a fingerprinted element is seen too
    assert P._weights_key(clf, None, None) != k2
    assert P._weights_key(clf, np.zeros(5), np.ones(5)) != P._weights_key(clf, np.zeros(5), 2 * np.ones(5))

    P._ambiguous.update(last=0, total=0, warned=False)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        P._note_ambiguous({"n_ambiguous": 3, "h2d_bytes": 10, "path": 1})
        P._note_ambiguous({"n_ambiguous": 2, "h2d_bytes": 20, "path": 1})
    assert [w.category for w in caught] == [RuntimeWarning]            # once per process
    assert P.last_ambiguous_rows() == 2 and P._ambiguous["total"] == 5
    assert P.last_call_stats() == {"n_ambiguous": 2, "h2d_bytes": 20, "path": 1}
    P._note_ambiguous({"n_ambiguous": 0})
    assert P.last_ambiguous_rows() == 0
    P._ambiguous.update(last=0, total=0, warned=False)
