"""GPU parity of the 2-layer MLP predictor (BASELINE.json configs[4]) against the oracle and torch itself."""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import mlp as omlp

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN  # noqa: E402


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


@pytest.fixture(scope="module")
def mlp_golden():
    z = np.load(GOLDEN / "mlp_64_32_10.npz")
    return {k: z[k] for k in z.files}


def _weights(g):
    return g["w1"], g["b1"], g["w2"], g["b2"]


def test_golden_fixture_equals_torch_labels(engine, mlp_golden):
    m = engine.load_mlp(*_weights(mlp_golden))
    b = engine.stage(mlp_golden["X"])
    got, st = engine.predict_mlp(m, b, exact=True)
    np.testing.assert_array_equal(got, mlp_golden["labels_torch"])
    assert st["path"] == 5 and st["kernel_launches"] == 2  # integer pixel rows are tf32 values: tensor-core kernel + fp64 re-score


@pytest.mark.parametrize("rows", [1, 127, 128, 129, 5000, 250_001])
def test_exact_parity_against_float64_network(engine, mlp_golden, rows):
    w = _weights(mlp_golden)
    X = np.random.default_rng(rows).integers(0, 17, size=(rows, 64), dtype=np.uint8).astype(np.float32)
    want = omlp.predict_indices_f64(X, *w).astype(np.int32)
    m = engine.load_mlp(*w)
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, want)
    assert st["n_ambiguous"] == 0


def test_fast_mode_differs_only_inside_the_bound(engine, mlp_golden):
    w = _weights(mlp_golden)
    X = np.random.default_rng(9).standard_normal((1_000_000, 64)).astype(np.float32)
    m = engine.load_mlp(*w)
    b = engine.stage(X)
    exact, st = engine.predict_mlp(m, b, exact=True)
    want = omlp.predict_indices_f64(X, *w).astype(np.int32)
    np.testing.assert_array_equal(exact, want)
    assert 0 <= st["n_flagged"] < 20_000
    fast, stf = engine.predict_mlp(m, b, exact=False)
    assert stf["kernel_launches"] == 1
    diff = np.flatnonzero(fast != want)
    margin = omlp.logit_margin_f64(X, *w)
    assert len(diff) <= st["n_flagged"] and (len(diff) == 0 or margin[diff].max() < 1e-3)


def test_against_torch_cpu_module_and_predictor(mlp_golden):
    """The reference predictor as written vs the drop-in device predictor, on a DataFrame."""
    import torch.nn as nn
    import torch.nn.functional as F

    from unionml_b200.predictors import mlp_argmax

    class PytorchModel(nn.Module):  # tests/integration/pytorch_app/quickstart.py:14-24
        def __init__(self, in_dims, hidden_dims, out_dims):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(in_dims, hidden_dims), nn.ReLU(), nn.Linear(hidden_dims, out_dims))

        def forward(self, features):
            return F.softmax(self.layers(features), dim=1)

    torch.manual_seed(0)
    module = PytorchModel(64, 32, 10)
    np.testing.assert_array_equal(module.layers[0].weight.detach().numpy(), mlp_golden["w1"])
    frame = pd.DataFrame(np.random.default_rng(4).integers(0, 17, size=(20_000, 64)).astype(np.float64))
    with torch.no_grad():
        want = [float(x) for x in module(torch.from_numpy(frame.values).float()).argmax(1)]
    got = mlp_argmax(module, frame)
    assert all(isinstance(x, float) for x in got)
    mism = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    # torch's own fp32 forward is only trusted outside its rounding noise; inside it the float64 network decides
    margin = omlp.logit_margin_f64(frame.values, *_weights(mlp_golden))
    assert all(margin[i] < 1e-4 for i in mism) and len(mism) <= 2


# ---------------------------------------------------------------------------------------------------------------
# tensor-core (wgmma, tf32) kernel: stats path 5
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 127, 128, 129, 5000, 250_001])
def test_tensor_core_path_parity_and_dispatch(engine, mlp_golden, rows, monkeypatch):
    """Integer / pixel rows are tf32 values -> layer 1 on the tensor cores; general floats -> the CUDA-core kernel.
    Both equal the float64 network on every row."""
    w = _weights(mlp_golden)
    m = engine.load_mlp(*w)
    Xi = np.random.default_rng(rows).integers(0, 256, size=(rows, 64)).astype(np.float32)  # MNIST pixel domain
    got, st = engine.predict_mlp(m, engine.stage(Xi), exact=True)
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(Xi, *w).astype(np.int32))
    assert st["path"] == 5
    Xf = np.random.default_rng(rows).standard_normal((rows, 64)).astype(np.float32)
    got, st = engine.predict_mlp(m, engine.stage(Xf), exact=True)
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(Xf, *w).astype(np.int32))
    assert st["path"] == 3
    # forcing the CUDA-core kernel on the integer rows gives the same labels
    monkeypatch.setenv("UML_B200_MLP_TC", "0")
    got0, st0 = engine.predict_mlp(m, engine.stage(Xi), exact=True)
    assert st0["path"] == 3
    np.testing.assert_array_equal(got0, omlp.predict_indices_f64(Xi, *w).astype(np.int32))


def test_tensor_core_kernel_is_safe_on_rows_that_are_not_tf32(engine, mlp_golden, monkeypatch):
    """Forced onto general floats the kernel scores truncated inputs - and knows it: every such row gets A1 = +inf,
    is flagged and re-scored in fp64, so the labels are still the float64 network's."""
    w = _weights(mlp_golden)
    m = engine.load_mlp(*w)
    rng = np.random.default_rng(12)
    X = rng.integers(0, 17, size=(200_000, 64)).astype(np.float32)
    dirty = rng.choice(200_000, size=5_000, replace=False)
    X[dirty, rng.integers(0, 64, size=5_000)] += np.float32(1.0 / 3.0)  # not representable in 10 mantissa bits
    want = omlp.predict_indices_f64(X, *w).astype(np.int32)
    monkeypatch.setenv("UML_B200_MLP_TC", "1")
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    assert st["path"] == 5 and st["n_flagged"] >= 5_000
    np.testing.assert_array_equal(got, want)
    Xf = rng.standard_normal((50_000, 64)).astype(np.float32)
    got, st = engine.predict_mlp(m, engine.stage(Xf), exact=True)
    assert st["path"] == 5 and st["n_flagged"] == 50_000
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(Xf, *w).astype(np.int32))


def test_tensor_core_flagged_rows_rescored_in_float64(engine, mlp_golden, monkeypatch):
    """The flag list + mlp_rescore_f64_kernel behind the tensor-core kernel: a second launch that gives every flagged
    row the float64 network's label, also when every row of the batch is flagged."""
    w = _weights(mlp_golden)
    m = engine.load_mlp(*w)
    monkeypatch.setenv("UML_B200_MLP_TC", "1")
    X = np.random.default_rng(41).integers(0, 17, size=(1_200_000, 64), dtype=np.uint8).astype(np.float32)
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    assert st["path"] == 5 and st["kernel_launches"] == 2 and st["n_flagged"] > 0
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(X, *w).astype(np.int32))
    Xf = np.random.default_rng(42).standard_normal((150_000, 64)).astype(np.float32)  # forced onto the tensor cores
    got, st = engine.predict_mlp(m, engine.stage(Xf), exact=True)
    assert st["path"] == 5 and st["n_flagged"] == 150_000
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(Xf, *w).astype(np.int32))


@pytest.mark.parametrize("shape", [(64, 32, 10), (64, 16, 10), (50, 32, 3), (32, 16, 2), (128, 32, 10), (100, 16, 3)])
def test_tensor_core_shapes(engine, shape):
    F, H, C = shape
    rng = np.random.default_rng(F * 1000 + H * 10 + C)
    w1, b1 = (rng.standard_normal((H, F)) * 0.2).astype(np.float32), rng.standard_normal(H).astype(np.float32)
    w2, b2 = rng.standard_normal((C, H)).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    X = rng.integers(-8, 9, size=(70_001, F)).astype(np.float32)
    m = engine.load_mlp(w1, b1, w2, b2)
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(X, w1, b1, w2, b2).astype(np.int32))
    assert st["path"] == 5, st
    fast, stf = engine.predict_mlp(m, engine.stage(X), exact=False)
    assert stf["path"] == 5 and (fast != got).sum() <= st["n_flagged"]


def test_tensor_core_full_size_ten_million(engine, mlp_golden):
    """cfg 5 at BASELINE size: all 10M labels against the float64 network, streamed in 1M-row chunks."""
    w = _weights(mlp_golden)
    m = engine.load_mlp(*w)
    N = 10_000_000
    X = engine.pinned_empty((N, 64), np.float32)
    for k in range(10):
        X[k * 1_000_000 : (k + 1) * 1_000_000] = np.random.default_rng(k).integers(0, 17, size=(1_000_000, 64), dtype=np.uint8)
    b = engine.stage(X)
    labels, st = engine.predict_mlp(m, b, exact=True)
    assert st["path"] == 5 and st["n_rows"] == N and st["n_ambiguous"] == 0 and st["n_flagged"] < N // 50
    for k in range(10):
        sl = slice(k * 1_000_000, (k + 1) * 1_000_000)
        np.testing.assert_array_equal(labels[sl], omlp.predict_indices_f64(X[sl], *w).astype(np.int32))
    fast, _ = engine.predict_mlp(m, b, exact=False)
    assert (fast != labels).sum() <= st["n_flagged"]
    print(f"mlp tensor-core 10M x 64: kernel {st['kernel_ms']:.3f} ms, re-score {st['recheck_ms']:.3f} ms, flagged {st['n_flagged']}")


def test_mlp_peer_label_vectors(engine, mlp_golden, monkeypatch):
    """uml_mlp_predict_peers: labels land in every target vector (uint8 and int32 wire), both kernels."""
    w = _weights(mlp_golden)
    m = engine.load_mlp(*w)
    rows = 100_003
    X = np.random.default_rng(2).integers(0, 17, size=(rows, 64)).astype(np.float32)
    want = omlp.predict_indices_f64(X, *w).astype(np.int32)
    b = engine.stage(X)
    for force in ("1", "0"):
        monkeypatch.setenv("UML_B200_MLP_TC", force)
        for lb, dt in ((1, torch.uint8), (4, torch.int32)):
            v0 = torch.full((rows + 64,), 77, dtype=dt, device="cuda")
            v1 = torch.full((rows + 64,), 77, dtype=dt, device="cuda")
            st = engine.predict_mlp_peers(m, b, [v0.data_ptr(), v1.data_ptr()], 32, exact=True, want_stats=True, label_bytes=lb)
            assert st["path"] == (5 if force == "1" else 3)
            for v in (v0, v1):
                host = v.cpu().numpy().astype(np.int32)
                np.testing.assert_array_equal(host[32 : 32 + rows], want)
                assert (host[:32] == 77).all() and (host[32 + rows :] == 77).all()


def test_mlp_host_pipeline_and_async_list(mlp_golden):
    """mlp_argmax on host frames: the chunk pipeline of the linear predictor (uml_mlp_predict_host), and from 1M rows on
    the asynchronous form that fills the list while the batch is in flight.  Integer frames take the
    tensor-core kernel, general floats the CUDA-core kernel; both equal the float64 network."""
    import torch.nn as nn

    from unionml_b200.engine import get_engine
    from unionml_b200.predictors import device_mlp, mlp_argmax

    w = _weights(mlp_golden)
    module = nn.Sequential(nn.Linear(64, 32), nn.ReLU(), nn.Linear(32, 10))
    with torch.no_grad():
        module[0].weight.copy_(torch.from_numpy(w[0])); module[0].bias.copy_(torch.from_numpy(w[1]))
        module[2].weight.copy_(torch.from_numpy(w[2])); module[2].bias.copy_(torch.from_numpy(w[3]))
    N = 1_100_001
    Xi = np.random.default_rng(5).integers(0, 17, size=(64, N)).astype(np.float64)  # feature-major float64 block
    frame = pd.DataFrame(Xi.T, columns=[f"pixel_{i}" for i in range(64)], copy=False)
    want = omlp.predict_indices_f64(Xi.T.astype(np.float32), *w).astype(np.float64)
    got = mlp_argmax(module, frame)  # >= 1M rows: asynchronous list building
    assert isinstance(got, list) and len(got) == N and isinstance(got[0], float)
    np.testing.assert_array_equal(np.asarray(got), want)
    np.testing.assert_array_equal(np.asarray(mlp_argmax(module, frame.iloc[:300_000])), want[:300_000])  # synchronous form
    eng = get_engine()
    vals, st = eng.predict_mlp_host(device_mlp(module, eng), Xi.T[:500_000], chunk_rows=8192)
    assert st["path"] == 5 and vals.dtype == np.int32
    np.testing.assert_array_equal(vals, want[:500_000])
    Xf = np.random.default_rng(6).standard_normal((200_000, 64))  # float64 general values: cast to fp32 like the reference
    vals, st = eng.predict_mlp_host(device_mlp(module, eng), Xf)
    assert st["path"] == 3
    np.testing.assert_array_equal(vals, omlp.predict_indices_f64(Xf.astype(np.float32), *w).astype(np.float64))
    with pytest.raises(ValueError):
        bad = Xf.copy(); bad[777, 3] = np.inf
        mlp_argmax(module, bad)


def test_generic_shapes_take_the_fp64_kernel(engine):
    rng = np.random.default_rng(0)
    w1, b1 = rng.standard_normal((20, 13)).astype(np.float32), rng.standard_normal(20).astype(np.float32)
    w2, b2 = rng.standard_normal((7, 20)).astype(np.float32), rng.standard_normal(7).astype(np.float32)
    X = rng.standard_normal((30_000, 13)).astype(np.float32)
    m = engine.load_mlp(w1, b1, w2, b2)
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, omlp.predict_indices_f64(X, w1, b1, w2, b2))
    assert st["path"] == 2


def test_mlp_nonfinite_and_shape_errors(engine, mlp_golden):
    m = engine.load_mlp(*_weights(mlp_golden))
    X = np.ones((1000, 64), dtype=np.float32)
    X[5, 5] = np.nan
    with pytest.raises(ValueError):
        engine.predict_mlp(m, engine.stage(X, check_finite=False), exact=True)
    with pytest.raises(ValueError, match="63 features"):
        engine.predict_mlp(m, engine.stage(np.ones((4, 63), dtype=np.float32)))
