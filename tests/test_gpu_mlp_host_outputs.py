"""GPU tests of the MLP predictor's class probabilities and top-k from HOST rows (``uml_mlp_predict_proba_host``,
``uml_mlp_predict_topk_host``, ``Engine.predict_mlp_proba_host`` / ``predict_mlp_topk_host`` and the predictors built
on them).

Above 64 rows they go through the chunk pipeline: bit-equal to the resident call on the same rows when every row, or
no row, is a tf32 value; in a mixed frame whose first rows are tf32 values, the rows that are not get the float64
route's values.  Up to 64 rows they take the online route (``mlp_small_kernel``, stats path 4): the float64 route's
values, which the resident call gives on path 2 (``k = C > kMlpTopkMax``: every row scored by ``mlp_topk_f64_kernel``)."""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import mlp as omlp

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN  # noqa: E402
from tests.test_gpu_mlp_proba import _assert_within_bound, _quickstart_module  # noqa: E402


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


def _small_mlp():
    """a random 50 -> 16 -> 3 network (tile shapes H = 16, C = 3; 50 features pad to 64)"""
    rng = np.random.default_rng(21)
    w1, b1 = (rng.standard_normal((16, 50)) * 0.2).astype(np.float32), rng.standard_normal(16).astype(np.float32)
    w2, b2 = rng.standard_normal((3, 16)).astype(np.float32), rng.standard_normal(3).astype(np.float32)
    return w1, b1, w2, b2


def _ints(rows, F, seed):
    return np.random.default_rng(seed).integers(0, 17, size=(rows, F)).astype(np.float64)


def _normals(rows, F, seed):
    return np.random.default_rng(seed).standard_normal((rows, F)) * 3


def _source(engine, X, dtype, order, pinned):
    a = X.astype(dtype)
    a = np.asfortranarray(a) if order == "F" else np.ascontiguousarray(a)
    if pinned:
        p = engine.pinned_empty(a.shape, a.dtype)
        if order == "F":
            p = p.reshape(a.shape[::-1]).T  # a feature-major view of the page-locked block
        p[...] = a
        return p
    return a


def _f64_route(engine, m, X):
    """the float64 route's probabilities and full ranks of every row: the resident top-k with k = C on path 2"""
    C = m.n_classes
    b = engine.stage(np.ascontiguousarray(X, dtype=np.float32))
    idx, proba, st = engine.predict_mlp_topk(m, b, C, exact=True)
    b.free()
    assert st["path"] == 2, st
    full = np.empty_like(proba)
    np.put_along_axis(full, idx.astype(np.int64), proba, axis=1)
    return full, idx, proba


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------
# 1. the pipeline is bit-equal to the resident call on frames that are all tf32 values or none
# ---------------------------------------------------------------------------------------------------------------
SOURCES = [("float32", "C", False), ("float64", "F", False), ("float64", "C", True), ("int64", "C", False),
           ("uint8", "F", True)]


@pytest.mark.parametrize("net", ["golden", "random"])
@pytest.mark.parametrize("dtype,order,pinned", SOURCES)
@pytest.mark.parametrize("domain", ["tf32", "normal"])
def test_pipeline_matches_the_resident_call(engine, golden, net, dtype, order, pinned, domain):
    if domain == "normal" and dtype not in ("float32", "float64"):
        pytest.skip("integer sources hold tf32 values only")
    w = _weights(golden) if net == "golden" else _small_mlp()
    F, C = w[0].shape[1], w[2].shape[0]
    m = engine.load_mlp(*w)
    X = _ints(3000, F, 1) if domain == "tf32" else _normals(3000, F, 1)
    src = _source(engine, X, dtype, order, pinned)
    b = engine.stage(np.ascontiguousarray(X.astype(dtype)))
    want, sw = engine.predict_mlp_proba(m, b, want_stats=True)
    got, st = engine.predict_mlp_proba_host(m, src, chunk_rows=640)  # 4 full chunks of 640 rows and a ragged 440
    assert st["path"] == sw["path"] == (5 if domain == "tf32" else 3), (st, sw)
    assert st["n_flagged"] == 0
    np.testing.assert_array_equal(_bits(got), _bits(want))
    for k in sorted({1, 3, 5, 7, C} & set(range(1, C + 1))):
        for exact in (True, False):
            wi, wp, ws = engine.predict_mlp_topk(m, b, k, exact=exact)
            gi, gp, gs = engine.predict_mlp_topk_host(m, src, k, exact=exact, chunk_rows=640)
            assert gs["path"] == ws["path"], (k, exact, gs, ws)
            np.testing.assert_array_equal(gi, wi, err_msg=f"k={k} exact={exact}")
            np.testing.assert_array_equal(_bits(gp), _bits(wp), err_msg=f"k={k} exact={exact}")
            assert gs["n_ambiguous"] == ws["n_ambiguous"]
    b.free()


# ---------------------------------------------------------------------------------------------------------------
# 2. a mixed frame: the first rows say "tf32", later chunks are not
# ---------------------------------------------------------------------------------------------------------------
def test_mixed_frame_rows_that_are_not_tf32_get_the_float64_values(engine, golden):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = np.concatenate([_ints(4096, 64, 2), _normals(6000, 64, 3)])
    X[5000:5100] = _ints(100, 64, 4)  # tf32 rows inside a later chunk too
    not_tf32 = np.any(X.astype(np.float32).view(np.uint32) & 0x1FFF, axis=1)
    assert not_tf32[4096:].sum() == 5900
    got, st = engine.predict_mlp_proba_host(m, X, chunk_rows=2048)
    assert st["path"] == 5 and st["n_flagged"] >= int(not_tf32.sum()), st
    full, ranks, _ = _f64_route(engine, m, X)
    np.testing.assert_array_equal(_bits(got[not_tf32]), _bits(full[not_tf32]))
    _assert_within_bound(got, X, w, 5)  # every row inside the path 5 bound of DESIGN.md 3.6
    b = engine.stage(X.astype(np.float32))
    for k in (1, 3, 5):
        want_idx, _, _ = engine.predict_mlp_topk(m, b, k, exact=True)
        gi, gp, gs = engine.predict_mlp_topk_host(m, X, k, exact=True, chunk_rows=2048)
        assert gs["path"] == 5 and gs["n_flagged"] >= int(not_tf32.sum())
        np.testing.assert_array_equal(gi, want_idx)
        # FAST: the rows that are not tf32 values take the float64 ranks and probabilities
        fi, fp, fs = engine.predict_mlp_topk_host(m, X, k, exact=False, chunk_rows=2048)
        assert fs["n_flagged"] >= int(not_tf32.sum())
        np.testing.assert_array_equal(fi[not_tf32], ranks[not_tf32, :k])
        np.testing.assert_array_equal(_bits(fp[not_tf32]), _bits(np.take_along_axis(full, fi.astype(np.int64), 1)[not_tf32]))
    b.free()


# ---------------------------------------------------------------------------------------------------------------
# 3. the online route
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 4, 5, 32, 64, 65])
def test_online_route_is_the_float64_route(engine, golden, rows):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = _normals(rows, 64, 5 + rows)
    full, ranks, rproba = _f64_route(engine, m, X)
    for frame in (X, np.asfortranarray(X), X.astype(np.float32)):
        for _ in range(2):  # capture, then replay
            got, st = engine.predict_mlp_proba_host(m, frame)
            assert (st["path"] == 4) == (rows <= 64), st
            if rows <= 64:
                assert st["kernel_launches"] == 1
                np.testing.assert_array_equal(_bits(got), _bits(full))
            for k in range(1, 11):
                gi, gp, gs = engine.predict_mlp_topk_host(m, frame, k, exact=False)
                assert (gs["path"] == 4) == (rows <= 64)
                if rows <= 64:
                    np.testing.assert_array_equal(gi, ranks[:, :k])
                    np.testing.assert_array_equal(_bits(gp), _bits(rproba[:, :k]))


def test_online_exact_tie_is_counted(engine, golden):
    w1, b1, w2, b2 = (a.copy() for a in _weights(golden))
    w2[1] = w2[0]
    b2[0] = b2[1] = np.float32(50.0)  # classes 0 and 1 tie on every row and lead it
    m = engine.load_mlp(w1, b1, w2, b2)
    X = _ints(16, 64, 6)
    for k in (1, 3):
        idx, _, st = engine.predict_mlp_topk_host(m, X, k)
        assert st["path"] == 4 and st["n_ambiguous"] == 16, st
        assert (idx[:, 0] == 0).all()
        if k > 1:
            assert (idx[:, 1] == 1).all()
    _, st = engine.predict_mlp_proba_host(m, X)
    assert st["n_ambiguous"] == 0


def test_online_graphs_of_each_output_stay_apart(engine, golden):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = _normals(32, 64, 7)
    full, ranks, rproba = _f64_route(engine, m, X)
    labels = omlp.predict_indices_f64(X.astype(np.float32), *w)
    for _ in range(3):
        got, st = engine.predict_mlp_host(m, X)
        assert st["path"] == 4
        np.testing.assert_array_equal(got, labels)
        got, st = engine.predict_mlp_proba_host(m, X)
        np.testing.assert_array_equal(_bits(got), _bits(full))
        for k in (3, 5):
            gi, gp, st = engine.predict_mlp_topk_host(m, X, k)
            assert st["path"] == 4
            np.testing.assert_array_equal(gi, ranks[:, :k])
            np.testing.assert_array_equal(_bits(gp), _bits(rproba[:, :k]))


def test_online_freed_and_reloaded_model(engine, golden):
    w1, b1, w2, b2 = _weights(golden)
    X = _ints(32, 64, 8)
    m = engine.load_mlp(w1, b1, w2, b2)
    engine.predict_mlp_proba_host(m, X)
    engine.predict_mlp_topk_host(m, X, 3)
    m._fin()
    del m
    other = (w1, b1, w2[::-1].copy(), b2[::-1].copy())
    m2 = engine.load_mlp(*other)
    full, ranks, rproba = _f64_route(engine, m2, X)
    got, _ = engine.predict_mlp_proba_host(m2, X)
    np.testing.assert_array_equal(_bits(got), _bits(full))
    gi, _, _ = engine.predict_mlp_topk_host(m2, X, 3)
    np.testing.assert_array_equal(gi, ranks[:, :3])


# ---------------------------------------------------------------------------------------------------------------
# 4. errors
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [np.nan, np.inf, 1e300])
@pytest.mark.parametrize("rows", [32, 3000])
def test_nonfinite_features(engine, golden, bad, rows):
    m = engine.load_mlp(*_weights(golden))
    X = _ints(rows, 64, 9)
    X[7, 3] = bad
    with pytest.raises(ValueError, match="NaN or infinity"):
        engine.predict_mlp_proba_host(m, X)
    for exact in (True, False):
        with pytest.raises(ValueError, match="NaN or infinity"):
            engine.predict_mlp_topk_host(m, X, 3, exact=exact)
    X[7, 3] = 0.0
    got, _ = engine.predict_mlp_proba_host(m, X)  # the engine is fine afterwards
    assert np.isfinite(got).all()


def test_shape_k_and_empty_errors(engine, golden):
    from unionml_b200.engine import EngineError
    from unionml_b200.predictors import mlp_predict_proba, mlp_predict_topk

    m = engine.load_mlp(*_weights(golden))
    for rows in (4, 3000):
        with pytest.raises(ValueError, match="63 features"):
            engine.predict_mlp_proba_host(m, np.ones((rows, 63)))
        with pytest.raises(ValueError, match="63 features"):
            engine.predict_mlp_topk_host(m, np.ones((rows, 63)), 3)
        for k in (0, 11):
            with pytest.raises(EngineError):
                engine.predict_mlp_topk_host(m, np.ones((rows, 64)), k)
    _, module = _quickstart_module(golden)
    with pytest.raises(ValueError, match="0 sample"):
        mlp_predict_proba(module, pd.DataFrame(np.ones((0, 64))))
    with pytest.raises(ValueError, match="0 sample"):
        mlp_predict_topk(module, pd.DataFrame(np.ones((0, 64))))


# ---------------------------------------------------------------------------------------------------------------
# 5. a frame of ten million rows
# ---------------------------------------------------------------------------------------------------------------
def test_ten_million_row_float64_frame(engine, golden):
    from bench import digits_rows

    w = _weights(golden)
    m = engine.load_mlp(*w)
    N = 10_000_000
    X8 = np.empty((N, 64), dtype=np.uint8)
    digits_rows(0, N, X8)
    frame = pd.DataFrame(X8.astype(np.float64), columns=[f"pixel_{i}" for i in range(64)])
    del X8
    proba, st = engine.predict_mlp_proba_host(m, frame)
    assert st["path"] == 5 and st["n_rows"] == N
    idx, tp, ts = engine.predict_mlp_topk_host(m, frame, 3, exact=True)
    bad = 0
    for lo in range(0, N, 1_000_000):
        Xc = frame.values[lo : lo + 1_000_000]
        _assert_within_bound(proba[lo : lo + 1_000_000], Xc, w, 5)
        z = omlp.logits(Xc, *w, dtype=np.float64)
        bad += int(np.any(idx[lo : lo + 1_000_000] != np.argsort(-z, kind="stable")[:, :3], axis=1).sum())
        at = np.take_along_axis(proba[lo : lo + 1_000_000], idx[lo : lo + 1_000_000].astype(np.int64), axis=1)
        assert np.abs(at - tp[lo : lo + 1_000_000]).max() <= 1e-6
    assert bad <= ts["n_ambiguous"]


# ---------------------------------------------------------------------------------------------------------------
# 6. the quickdraw template's predictor: one row, the top 3 as {name: probability}
# ---------------------------------------------------------------------------------------------------------------
def test_quickdraw_shaped_app(golden):
    from fastapi import FastAPI
    from fastapi.testclient import TestClient

    from unionml_b200 import Dataset, Model, ModelArtifact, predictors

    PytorchModel, module = _quickstart_module(golden)
    w = _weights(golden)
    names = [f"class_{i}" for i in range(10)]
    cols = [f"pixel_{i}" for i in range(64)]
    frame = pd.DataFrame(_ints(200, 64, 11), columns=cols)
    dataset = Dataset(name="quickdraw_shape", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="quickdraw_shape", init=PytorchModel, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return frame.assign(target=0)

    @model.predictor
    def predictor(module: PytorchModel, features: pd.DataFrame) -> dict:
        values, indices = predictors.mlp_predict_topk(module, features.iloc[:1], k=3)
        return {names[i]: float(v) for i, v in zip(indices[0], values[0])}

    model.artifact = ModelArtifact(module)

    def want(row):
        z = omlp.logits(frame.values[row : row + 1], *w, dtype=np.float64)
        return [names[i] for i in np.argsort(-z, kind="stable")[0, :3]]

    out = model.predict(features=frame.iloc[:1])
    assert list(out) == want(0)
    assert predictors.last_call_stats()["path"] == 4
    app = FastAPI()
    model.serve(app)
    with TestClient(app) as client:
        for row in (3, 4):
            r = client.post("/predict", json={"features": frame.iloc[row : row + 1].to_dict(orient="records")})
            assert r.status_code == 200
            got = r.json()
            assert list(got) == want(row)
            assert list(got.values()) == sorted(got.values(), reverse=True)
