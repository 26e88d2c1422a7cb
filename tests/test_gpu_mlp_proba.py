"""GPU tests of the MLP predictor's class probabilities (``uml_mlp_predict_proba``, ``Engine.predict_mlp_proba``,
``predictors.mlp_predict_proba``): softmax(W2 relu(W1 x + b1) + b2) per row, as ``PytorchModel.forward`` of the torch
quickstart returns it.

Paths 5 (tensor cores) and 3 (CUDA cores) are checked against the bound DESIGN.md 3.6 derives: with δ the route's own
bound on a logit's error (the EXACT guard's e1 A1 + e2 A2, DESIGN.md 3.3 / 3.4) and L = max_k |ẑ_k − max ẑ| on the
kernel's logits,
    |p̂_c − p_c| <= p_c (exp(2δ + 2uL) (1 + (C + 12) u) − 1) + FLT_MIN.
Path 2 (float64 logits and softmax) is checked within 1 ulp of fp32 plus FLT_MIN.  The reference is the float64
forward of the same fp32 weights on the fp32-cast features.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import mlp as omlp

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN  # noqa: E402

U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
HALF_SUBNORMAL = 2.0 ** -150


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


def _reference(X, w):
    z = omlp.logits(X, *w, dtype=np.float64)
    e = np.exp(z - z.max(axis=1, keepdims=True))
    return z, e / e.sum(axis=1, keepdims=True)


def _logit_bound(X, w, path):
    """δ per row: the bound on |ẑ_c − z_c| the route's EXACT guard uses (constants of mlp_tc_launch_one for path 5,
    launch_mlp_tma / uml_mlp_load for path 3; DESIGN.md 3.3 and 3.4)."""
    w1, b1, w2, b2 = (np.asarray(a, dtype=np.float64) for a in w)
    H, F = w1.shape
    Xd = np.asarray(X, dtype=np.float32).astype(np.float64)
    row_sum = np.abs(w2).sum(axis=1).max()
    w1max = np.abs(w1).max(axis=0)
    e2 = (H + 4) * U * 1.0001
    if path == 5:
        w1max = np.maximum(w1max, 2.0 ** -104)
        n_mma = (-(-F // 32) * 32) / 8
        e1 = (32 * n_mma + 12) * U * (1 + F * 2.0 ** -21) * 1.0001 * row_sum
        hidden_abs = (18 * n_mma + 3 + w1max.sum()) * FLT_MIN
    else:
        e1 = (F + 4) * U * (1 + F * 2.0 ** -21) * 1.0001 * row_sum
        hidden_abs = (F + 2) * HALF_SUBNORMAL
    k2 = (FLT_MIN + hidden_abs * row_sum + (H + 4) * HALF_SUBNORMAL) / e2 * (1 + 1 / 1024)
    a1 = np.abs(b1).max() + np.abs(Xd) @ w1max
    h = np.maximum(Xd @ w1.T + b1, 0)
    a2 = h @ np.abs(w2).max(axis=0) + np.abs(b2).max() + k2
    return e1 * a1 + e2 * a2


def _assert_within_bound(got, X, w, path):
    z, p = _reference(X, w)
    C = z.shape[1]
    assert got.shape == p.shape and got.dtype == np.float32
    assert np.isfinite(got).all() and (got >= 0).all()
    delta = _logit_bound(X, w, path)
    # L is taken on the kernel's logits, which lie within δ of the reference's: at most the reference's spread + 2δ
    L = z.max(axis=1) - z.min(axis=1) + 2 * delta
    rel = np.expm1(2 * delta + 2 * U * L) * (1 + (C + 12) * U) + (C + 12) * U
    err = np.abs(got.astype(np.float64) - p)
    excess = err - (p * rel[:, None] + FLT_MIN)
    assert (excess <= 0).all(), f"{int((excess > 0).sum())} entries outside the bound, worst excess {excess.max():.3g}"
    return err


def _assert_f64_route(got, X, w):
    _, p = _reference(X, w)
    ulp = np.spacing(p.astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - p)
    assert (err <= ulp + FLT_MIN).all(), f"worst {np.max(err / (ulp + FLT_MIN)):.3g} ulp"


def _assert_fast_label_is_row_max(engine, m, b, proba):
    labels, _ = engine.predict_mlp(m, b, exact=False)
    top = proba.max(axis=1)
    at_label = proba[np.arange(len(labels)), labels]
    assert (at_label >= top - np.spacing(top)).all()


def _int_rows(rows, F, seed):
    return np.random.default_rng(seed).integers(0, 17, size=(rows, F)).astype(np.float32)


def _normal_rows(rows, F, seed):
    return np.random.default_rng(seed).standard_normal((rows, F)).astype(np.float32)


def _random_mlp(F, H, C, seed):
    rng = np.random.default_rng(seed)
    w1, b1 = (rng.standard_normal((H, F)) * 0.2).astype(np.float32), rng.standard_normal(H).astype(np.float32)
    w2, b2 = rng.standard_normal((C, H)).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    return w1, b1, w2, b2


def _quickstart_module(golden):
    import torch.nn as nn
    import torch.nn.functional as F

    class PytorchModel(nn.Module):  # tests/integration/pytorch_app/quickstart.py:14-24
        def __init__(self, in_dims, hidden_dims, out_dims):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(in_dims, hidden_dims), nn.ReLU(), nn.Linear(hidden_dims, out_dims))

        def forward(self, features):
            return F.softmax(self.layers(features), dim=1)

    torch.manual_seed(0)
    module = PytorchModel(64, 32, 10)
    np.testing.assert_array_equal(module.layers[0].weight.detach().numpy(), golden["w1"])
    return PytorchModel, module


# ---------------------------------------------------------------------------------------------------------------
def test_golden_model_bound_row_sums_and_torch(engine, golden):
    w = _weights(golden)
    X = golden["X"].astype(np.float32)
    m = engine.load_mlp(*w)
    got, st = engine.predict_mlp_proba(m, engine.stage(X), want_stats=True)
    assert st["path"] == 5 and st["kernel_launches"] == 1 and st["n_rows"] == len(X)
    _assert_within_bound(got, X, w, 5)
    C = got.shape[1]
    assert np.abs(got.astype(np.float64).sum(axis=1) - 1).max() <= (C + 2) * 2.0 ** -23
    _, module = _quickstart_module(golden)
    with torch.no_grad():
        want = module(torch.from_numpy(X)).numpy()
    print(f"golden 4096 x 64: largest |p - torch CPU fp32 forward| = {np.abs(got - want).max():.3g}")


@pytest.mark.parametrize("case", ["tf32_rows", "tf32_rows_cuda_cores", "normal_rows", "normal_rows_forced_tc"])
def test_every_route_with_labels_consistent(engine, golden, case, monkeypatch):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = _int_rows(100_003, 64, 1) if case.startswith("tf32") else _normal_rows(100_003, 64, 2)
    if case == "tf32_rows_cuda_cores":
        monkeypatch.setenv("UML_B200_MLP_TC", "0")
    if case == "normal_rows_forced_tc":  # the probability kernels have no re-score: rows that are not tf32 stay off it
        monkeypatch.setenv("UML_B200_MLP_TC", "1")
    b = engine.stage(X)
    got, st = engine.predict_mlp_proba(m, b, want_stats=True)
    path = 5 if case == "tf32_rows" else 3
    assert st["path"] == path
    _assert_within_bound(got, X, w, path)
    if case != "normal_rows_forced_tc":  # the labels' forced route is the tensor-core kernel
        _assert_fast_label_is_row_max(engine, m, b, got)


def test_generic_shape_takes_the_float64_route(engine):
    w = _random_mlp(100, 64, 7, 3)
    m = engine.load_mlp(*w)
    for X in (_normal_rows(30_001, 100, 4), _int_rows(5_000, 100, 5)):
        got, st = engine.predict_mlp_proba(m, engine.stage(X), want_stats=True)
        assert st["path"] == 2
        _assert_f64_route(got, X, w)


@pytest.mark.parametrize("H", [16, 32])
@pytest.mark.parametrize("C", [2, 3, 10])
def test_tile_shapes(engine, H, C):
    F = {2: 32, 3: 50, 10: 128}[C]
    w = _random_mlp(F, H, C, 10 * H + C)
    m = engine.load_mlp(*w)
    for X, path in ((_int_rows(70_001, F, C) - 8, 5), (_normal_rows(70_001, F, H), 3)):
        b = engine.stage(X)
        got, st = engine.predict_mlp_proba(m, b, want_stats=True)
        assert st["path"] == path
        _assert_within_bound(got, X, w, path)
        _assert_fast_label_is_row_max(engine, m, b, got)


@pytest.mark.parametrize("rows", [1, 15, 16, 17, 127, 128, 129, 5000, 250_001])
@pytest.mark.parametrize("route", ["tensor_cores", "cuda_cores"])
def test_ragged_rows_and_device_output(engine, golden, rows, route):
    """Partial 16-row runs, the last tile, device buffers with guard words behind n_rows x C, a destination that is
    4- but not 16-byte aligned (bitwise the same result), and repeat calls (bitwise the same)."""
    w = _weights(golden)
    m = engine.load_mlp(*w)
    X = _int_rows(rows, 64, rows) if route == "tensor_cores" else _normal_rows(rows, 64, rows)
    path = 5 if route == "tensor_cores" else 3
    b = engine.stage(X)
    host, st = engine.predict_mlp_proba(m, b, want_stats=True)
    assert st["path"] == path
    _assert_within_bound(host, X, w, path)
    n = rows * 10
    guard = -7.0
    for offset in (0, 1):  # floats: 0 -> 16-byte aligned (torch allocations are), 1 -> 4 bytes past it
        buf = torch.full((n + 68,), guard, dtype=torch.float32, device="cuda")
        assert buf.data_ptr() % 16 == 0
        for _ in range(2):
            _, st = engine.predict_mlp_proba(m, b, out_device_ptr=buf.data_ptr() + 4 * offset, want_stats=True)
            assert st["path"] == path
            dev = buf.cpu().numpy()
            np.testing.assert_array_equal(dev[offset : offset + n].view(np.uint32), host.reshape(-1).view(np.uint32))
            assert (dev[:offset] == guard).all() and (dev[offset + n :] == guard).all()


@pytest.mark.parametrize("route", ["tensor_cores", "cuda_cores"])
def test_wide_and_equal_logits(engine, golden, route):
    w1, b1, w2, b2 = _weights(golden)
    X = _int_rows(20_000, 64, 7) if route == "tensor_cores" else _normal_rows(20_000, 64, 7) * 8
    path = 5 if route == "tensor_cores" else 3
    z = omlp.logits(X, w1, b1, w2, b2)
    scale = np.float32(100.0 / np.abs(z).max())
    wide = (w1, b1, (w2 * scale).astype(np.float32), (b2 * scale).astype(np.float32))
    zw = omlp.logits(X, *wide)
    assert np.abs(zw).max() > 90 and (zw.max(axis=1) - zw.min(axis=1)).max() > 100
    m = engine.load_mlp(*wide)
    got, st = engine.predict_mlp_proba(m, engine.stage(X), want_stats=True)
    assert st["path"] == path
    _assert_within_bound(got, X, wide, path)
    _, p = _reference(X, wide)
    assert (p < FLT_MIN).any()
    assert (got[p < FLT_MIN] < np.float32(FLT_MIN)).all()  # underflowing classes come out 0 or subnormal
    # all logits equal (W2 = 0, equal biases): every probability is 1 / C within the bound
    flat = (w1, b1, np.zeros_like(w2), np.full_like(b2, 0.5))
    m = engine.load_mlp(*flat)
    got, st = engine.predict_mlp_proba(m, engine.stage(X), want_stats=True)
    assert st["path"] == path
    _assert_within_bound(got, X, flat, path)
    assert np.abs(got.astype(np.float64) - 0.1).max() <= 0.1 * 23 * U


# ---------------------------------------------------------------------------------------------------------------
def test_public_predictor_and_model_predict(golden):
    from typing import List

    from unionml_b200 import Dataset, Model
    from unionml_b200.model import ModelArtifact
    from unionml_b200.predictors import mlp_predict_proba

    PytorchModel, module = _quickstart_module(golden)
    w = _weights(golden)
    cols = [f"pixel_{i}" for i in range(64)]
    frame = pd.DataFrame(np.random.default_rng(8).integers(0, 17, size=(30_000, 64)).astype(np.float64), columns=cols)
    got = mlp_predict_proba(module, frame)
    assert isinstance(got, np.ndarray) and got.shape == (30_000, 10) and got.dtype == np.float32
    _assert_within_bound(got, frame.values, w, 5)
    normal = pd.DataFrame(np.random.default_rng(9).standard_normal((10_000, 64)), columns=cols)
    _assert_within_bound(mlp_predict_proba(module, normal), normal.values, w, 3)

    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="quickstart_mlp", init=PytorchModel, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return frame.assign(target=0)

    seen = []

    def monitor(module: PytorchModel, features: pd.DataFrame, predictions: List[List[float]]):
        seen.append(predictions)

    @model.predictor(callbacks=[monitor])
    def predictor(module: PytorchModel, features: pd.DataFrame) -> List[List[float]]:
        return mlp_predict_proba(module, features).tolist()

    model.artifact = ModelArtifact(module)
    out = model.predict(features=frame.iloc[:500])
    assert isinstance(out, list) and len(out) == 500 and isinstance(out[0], list) and isinstance(out[0][0], float)
    np.testing.assert_array_equal(np.asarray(out, dtype=np.float32), got[:500])
    assert seen and seen[-1] is out


def test_errors(golden):
    import torch.nn as nn

    from unionml_b200.predictors import mlp_predict_proba

    _, module = _quickstart_module(golden)
    bad = np.ones((1000, 64))
    bad[5, 5] = np.nan
    with pytest.raises(ValueError):
        mlp_predict_proba(module, pd.DataFrame(bad))
    with pytest.raises(ValueError, match="63 features"):
        mlp_predict_proba(module, pd.DataFrame(np.ones((4, 63))))
    with pytest.raises(TypeError):
        mlp_predict_proba(nn.Sequential(nn.Linear(64, 32), nn.Tanh(), nn.Linear(32, 10)), pd.DataFrame(np.ones((4, 64))))
    with pytest.raises(ValueError, match="0 sample"):
        mlp_predict_proba(module, pd.DataFrame(np.ones((0, 64))))
