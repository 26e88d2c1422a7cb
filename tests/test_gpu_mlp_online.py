"""GPU tests of the MLP predictor's online route: requests of <= 64 rows through ``uml_mlp_predict_host`` take one
float64 kernel (``mlp_small_kernel``, stats path 4) that reads the request from pinned host memory and is replayed as a
CUDA graph per (model, rows, features, dtype).  Its labels must be the float64 network's on the fp32-cast features
(what the exact-mode chunk pipeline gives for the same rows), its errors the pipeline's errors, and its graph cache
must never answer with another model's graph."""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import linear as olin
from oracle import mlp as omlp

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN  # noqa: E402

ROWS = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64]


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN / "mlp_64_32_10.npz")
    return {k: z[k] for k in z.files}


def _weights(g):
    return g["w1"], g["b1"], g["w2"], g["b2"]


def _pixels(rows, seed):
    """digits-like requests: integers 0..255, exact in every dtype the engine takes (uint8 included)"""
    return np.random.default_rng(seed).integers(0, 256, size=(rows, 64)).astype(np.float64)


def _digits(rows, seed):
    """the digits domain, 0..16: the golden network's logits stay within +-6 there"""
    return np.random.default_rng(seed).integers(0, 17, size=(rows, 64)).astype(np.float64)


def _online(engine, m, X, exact=True, calls=3):
    """the same request `calls` times (capture, then replays): every call on the online route with the same labels"""
    first = None
    for _ in range(calls):
        got, st = engine.predict_mlp_host(m, X, exact=exact)
        assert st["path"] == 4 and st["kernel_launches"] == 1 and st["n_ambiguous"] == 0, st
        assert st["n_rows"] == X.shape[0]
        if first is None:
            first = got.copy()
        np.testing.assert_array_equal(got, first)
    return first


def _quickstart_module():
    import torch.nn as nn
    import torch.nn.functional as F

    class PytorchModel(nn.Module):  # tests/integration/pytorch_app/quickstart.py:14-24
        def __init__(self, in_dims, hidden_dims, out_dims):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(in_dims, hidden_dims), nn.ReLU(), nn.Linear(hidden_dims, out_dims))

        def forward(self, features):
            return F.softmax(self.layers(features), dim=1)

    torch.manual_seed(0)
    return PytorchModel, PytorchModel(64, 32, 10)


# ---------------------------------------------------------------------------------------------------------------
# 1. parity on every dtype and layout
# ---------------------------------------------------------------------------------------------------------------
LAYOUTS = ["float64", "float32", "int64", "int32", "uint8", "fortran", "strided_slice", "frame"]


def _request(layout, X, n):
    """rows [0, n) of X (strided_slice: rows 0, 2, .., 2n-2) in the layout under test, and the row indices it holds"""
    if layout == "strided_slice":
        return X[0 : 2 * n : 2], np.arange(0, 2 * n, 2)
    idx = np.arange(n)
    if layout == "fortran":
        return np.asfortranarray(X[:n]), idx
    if layout == "frame":
        return pd.DataFrame(X[:n], columns=[f"pixel_{i}" for i in range(64)]), idx
    return np.ascontiguousarray(X[:n].astype(layout)), idx


@pytest.mark.parametrize("layout", LAYOUTS)
def test_parity_every_dtype_and_layout(engine, golden, layout):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = _pixels(200, 1)
    pipe, st = engine.predict_mlp_host(m, X)  # 200 rows: the chunk pipeline; rows are scored independently
    assert st["path"] == 5
    want = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    np.testing.assert_array_equal(pipe, want)
    for n in ROWS:
        req, idx = _request(layout, X, n)
        got = _online(engine, m, req)
        np.testing.assert_array_equal(got, want[idx], err_msg=f"{layout}, {n} rows")
        np.testing.assert_array_equal(got, pipe[idx])


def test_general_float_rows(engine, golden):
    """float64 values that are not fp32 values: cast to fp32 exactly as the staging kernels cast them"""
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = np.random.default_rng(2).standard_normal((200, 64)) * 4
    pipe, st = engine.predict_mlp_host(m, X)
    assert st["path"] == 3  # general floats: the CUDA-core kernel
    want = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    np.testing.assert_array_equal(pipe, want)
    for n in ROWS:
        for req in (X[:n], np.asfortranarray(X[:n]), X[:n].astype(np.float32)):
            np.testing.assert_array_equal(_online(engine, m, req), want[:n])


def test_int64_beyond_two_to_the_53(engine):
    """int64 -> double -> float as in the staging kernels: both routes see the same fp32 features"""
    rng = np.random.default_rng(3)
    w1, b1 = (rng.standard_normal((16, 8)) * 1e-18).astype(np.float32), rng.standard_normal(16).astype(np.float32)
    w2, b2 = rng.standard_normal((3, 16)).astype(np.float32), rng.standard_normal(3).astype(np.float32)
    m = engine.load_mlp(w1, b1, w2, b2)
    X = rng.integers(-(2**62), 2**62, size=(200, 8), dtype=np.int64) | 1  # odd: not a double
    pipe, _ = engine.predict_mlp_host(m, X)
    want = omlp.predict_indices_f64(X.astype(np.float64).astype(np.float32), w1, b1, w2, b2).astype(np.int32)
    np.testing.assert_array_equal(pipe, want)
    np.testing.assert_array_equal(_online(engine, m, X[:32]), want[:32])


def test_generic_shape(engine):
    """F = 13, H = 20, C = 7: a shape only the generic fp64 kernel takes in the pipeline"""
    rng = np.random.default_rng(0)
    w1, b1 = rng.standard_normal((20, 13)).astype(np.float32), rng.standard_normal(20).astype(np.float32)
    w2, b2 = rng.standard_normal((7, 20)).astype(np.float32), rng.standard_normal(7).astype(np.float32)
    m = engine.load_mlp(w1, b1, w2, b2)
    X = rng.standard_normal((200, 13))
    pipe, st = engine.predict_mlp_host(m, X)
    assert st["path"] == 2
    want = omlp.predict_indices_f64(X.astype(np.float32), w1, b1, w2, b2).astype(np.int32)
    np.testing.assert_array_equal(pipe, want)
    for n in ROWS:
        np.testing.assert_array_equal(_online(engine, m, X[:n]), want[:n])


def test_model_too_large_for_the_kernel_keeps_the_pipeline(engine):
    """the online kernel needs the fp64 weights plus eight strips of four rows and their fp32 features in shared
    memory; at F = 300, H = 48 that is ~244 KiB, beyond one SM, while the generic pipeline kernel (no fp32 rows)
    still fits: such a model is scored by the pipeline"""
    rng = np.random.default_rng(5)
    F, H, C = 300, 48, 10
    w1, b1 = (rng.standard_normal((H, F)) * 0.1).astype(np.float32), rng.standard_normal(H).astype(np.float32)
    w2, b2 = rng.standard_normal((C, H)).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    m = engine.load_mlp(w1, b1, w2, b2)
    X = rng.standard_normal((32, F))
    got, st = engine.predict_mlp_host(m, X)
    assert st["path"] == 2
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(X.astype(np.float32), w1, b1, w2, b2))


# ---------------------------------------------------------------------------------------------------------------
# 2. exactness at the edges
# ---------------------------------------------------------------------------------------------------------------
def _twin_classes(golden, gap):
    """classes 0 and 1 lead every row by ~50 and differ only by `gap` in b2 (fp32 cannot resolve a relative 1e-7)"""
    w1, b1, w2, b2 = (a.copy() for a in _weights(golden))
    w2[1] = w2[0]
    b2[0] = np.float32(50.0)
    b2[1] = np.nextafter(b2[0], np.float32(np.inf)) if gap else b2[0]
    return w1, b1, w2, b2


def test_planted_tiny_margin_gets_the_exact_label(engine, golden):
    w = _twin_classes(golden, gap=True)
    X = _digits(200, 6)
    margin = omlp.logit_margin_f64(X, *w)
    assert (margin > 0).all() and (margin < 1e-5).all()
    want = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    assert (want == 1).all()
    m = engine.load_mlp(*w)
    for exact in (True, False):  # FAST mode on <= 64 rows is the exact result too
        np.testing.assert_array_equal(_online(engine, m, X[:64], exact=exact), want[:64])
        np.testing.assert_array_equal(_online(engine, m, X[:7], exact=exact), want[:7])
    pipe, _ = engine.predict_mlp_host(m, X, exact=True)
    np.testing.assert_array_equal(pipe, want)


def test_fast_mode_returns_the_exact_labels(engine, golden):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = np.random.default_rng(7).standard_normal((64, 64)) * 4
    want = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    for n in ROWS:
        np.testing.assert_array_equal(_online(engine, m, X[:n], exact=False), want[:n])


def test_true_tie_first_index_wins_and_is_reported(engine, golden, monkeypatch):
    import warnings

    from unionml_b200 import predictors

    w = _twin_classes(golden, gap=False)
    X = _digits(32, 8)
    m = engine.load_mlp(*w)
    for _ in range(2):
        got, st = engine.predict_mlp_host(m, X)
        assert st["path"] == 4 and st["n_ambiguous"] == 32
        assert (got == 0).all()

    _, module = _quickstart_module()
    with torch.no_grad():
        for p, v in zip((module.layers[0].weight, module.layers[0].bias, module.layers[2].weight, module.layers[2].bias), w):
            p.copy_(torch.from_numpy(v))
    monkeypatch.setitem(predictors._ambiguous, "warned", False)
    with pytest.warns(RuntimeWarning, match="tied within rounding"):
        out = predictors.mlp_argmax(module, pd.DataFrame(X))
    assert out == [0.0] * 32
    assert predictors.last_ambiguous_rows() == 32 and predictors.last_call_stats()["path"] == 4
    with warnings.catch_warnings():
        warnings.simplefilter("error")  # one-time: no second warning
        predictors.mlp_argmax(module, pd.DataFrame(X))


# ---------------------------------------------------------------------------------------------------------------
# 3. errors match the pipeline
# ---------------------------------------------------------------------------------------------------------------
def _outcome(engine, m, X):
    try:
        got, st = engine.predict_mlp_host(m, X)
        return "labels", got, st["path"]
    except ValueError as ex:
        return "ValueError", str(ex), None


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf, 1e300])
def test_nonfinite_and_fp32_overflow_match_the_pipeline(engine, golden, bad):
    """NaN / Inf raise on both routes.  A finite float64 beyond the fp32 range becomes inf on the cast the reference
    predictor makes: the exact pipeline's fp64 re-score finds that row non-finite, and so does the online kernel."""
    m = engine.load_mlp(*_weights(golden))
    X = _pixels(200, 9)
    X[7, 3] = bad
    small = _outcome(engine, m, X[:32])
    pipe = _outcome(engine, m, X)
    assert small[0] == pipe[0] == "ValueError", (small, pipe)
    assert "NaN or infinity" in small[1] and "NaN or infinity" in pipe[1]
    # the engine is fine afterwards: a clean request on the same key replays its graph
    X[7, 3] = 0.0
    np.testing.assert_array_equal(_online(engine, m, X[:32]), omlp.predict_indices_f64(X[:32].astype(np.float32), *_weights(golden)))


def test_shape_and_empty_batch_errors(golden):
    from unionml_b200.predictors import mlp_argmax

    _, module = _quickstart_module()
    with pytest.raises(ValueError, match="X has 63 features"):
        mlp_argmax(module, np.ones((4, 63)))
    with pytest.raises(ValueError, match="0 sample"):
        mlp_argmax(module, pd.DataFrame(np.ones((0, 64))))


# ---------------------------------------------------------------------------------------------------------------
# 4. graph cache
# ---------------------------------------------------------------------------------------------------------------
def test_linear_and_mlp_with_equal_keys_alternate(engine, golden, digits_model):
    w = _weights(golden)
    mlp = engine.load_mlp(*w)
    lin = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    X = _pixels(32, 10) / 16.0
    want_mlp = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    want_lin = olin.predict_indices(olin.decision_function(X, digits_model["coef"], digits_model["intercept"]))
    assert (want_mlp != want_lin).any()
    for _ in range(3):
        got, st = engine.predict_host(lin, X)
        assert st["path"] == 4
        np.testing.assert_array_equal(got, want_lin)
        got, st = engine.predict_mlp_host(mlp, X)
        assert st["path"] == 4
        np.testing.assert_array_equal(got, want_mlp)


def test_more_keys_than_the_cache_holds(engine, golden):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = np.random.default_rng(11).standard_normal((64, 64))
    want = omlp.predict_indices_f64(X.astype(np.float32), *w).astype(np.int32)
    keys = [(n, dt) for n in range(1, 13) for dt in (np.float64, np.float32)]  # 24 keys > 16 cached graphs
    for _ in range(2):  # the second cycle re-captures evicted keys
        for n, dt in keys:
            got, st = engine.predict_mlp_host(m, X[:n].astype(dt))
            assert st["path"] == 4
            np.testing.assert_array_equal(got, want[:n])


def test_freed_and_reloaded_model_gets_its_own_graph(engine, golden):
    w1, b1, w2, b2 = _weights(golden)
    X = _pixels(32, 12)
    m = engine.load_mlp(w1, b1, w2, b2)
    np.testing.assert_array_equal(_online(engine, m, X), omlp.predict_indices_f64(X.astype(np.float32), w1, b1, w2, b2))
    m._fin()
    del m
    other = (w1, b1, w2[::-1].copy(), b2[::-1].copy())  # same shape, classes reversed
    want = omlp.predict_indices_f64(X.astype(np.float32), *other).astype(np.int32)
    m2 = engine.load_mlp(*other)
    np.testing.assert_array_equal(_online(engine, m2, X), want)


# ---------------------------------------------------------------------------------------------------------------
# 5. device_mlp cache
# ---------------------------------------------------------------------------------------------------------------
def test_device_mlp_cache_follows_the_weights(golden):
    import torch.nn as nn

    from unionml_b200.predictors import device_mlp, mlp_argmax

    _, module = _quickstart_module()
    X = pd.DataFrame(_pixels(32, 13))
    want = [float(v) for v in omlp.predict_indices_f64(X.values, *_weights(golden))]
    dm = device_mlp(module)
    assert device_mlp(module) is dm and mlp_argmax(module, X) == want and device_mlp(module) is dm
    saved = {k: v.clone() for k, v in module.state_dict().items()}
    out = module.layers[2]

    with torch.no_grad():
        out.bias[3] += 1000.0  # in place: torch bumps the parameter's version
    assert mlp_argmax(module, X) == [3.0] * 32
    assert device_mlp(module) is not dm

    module.load_state_dict(saved)  # in-place copy back
    assert mlp_argmax(module, X) == want

    bias = saved["layers.2.bias"].clone()
    bias[5] += 1000.0
    out.bias = nn.Parameter(bias)  # rebinding
    assert mlp_argmax(module, X) == [5.0] * 32


# ---------------------------------------------------------------------------------------------------------------
# 6. the served torch quickstart app
# ---------------------------------------------------------------------------------------------------------------
def test_served_quickstart_app(golden):
    from typing import List

    from fastapi import FastAPI
    from fastapi.testclient import TestClient
    from sklearn.datasets import load_digits

    from unionml_b200 import Dataset, Model, ModelArtifact, predictors

    PytorchModel, module = _quickstart_module()
    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="quickstart_mlp", init=PytorchModel, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return load_digits(as_frame=True).frame

    @model.predictor
    def predictor(module: PytorchModel, features: pd.DataFrame) -> List[float]:
        return predictors.mlp_argmax(module, features)

    model.artifact = ModelArtifact(module)
    app = FastAPI()
    model.serve(app)
    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    with TestClient(app) as client:
        for seed in (0, 1):
            sample = feats.sample(32, random_state=seed)
            r = client.post("/predict", json={"features": sample.to_dict(orient="records")})
            assert r.status_code == 200
            want = [float(v) for v in omlp.predict_indices_f64(sample.values, *_weights(golden))]
            assert r.json() == want
            assert predictors.last_call_stats()["path"] == 4
