"""GPU tests of the MLP predictor's top-k classes (``uml_mlp_predict_topk``, ``uml_topk_count_hits``,
``Engine.predict_mlp_topk``, ``predictors.mlp_predict_topk`` / ``mlp_accuracy`` / ``mlp_topk_accuracy``).

EXACT indices are checked against ``np.argsort(-z64, kind="stable")[:, :k]`` of the float64 network on the fp32-cast
features (rows that differ must have a float64 gap among the ranks they rank within the float64 stage's bound, and
be no more than ``n_ambiguous``), probabilities bitwise against ``uml_mlp_predict_proba`` on rows the rank
guard did not send to the float64 re-score, and all of them against the bound of DESIGN.md 3.6 (3.8).
"""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import mlp as omlp
from tests import f64_stage_cases as K

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN  # noqa: E402
from tests.test_gpu_mlp_proba import (  # noqa: E402
    U,
    FLT_MIN,
    _int_rows,
    _logit_bound,
    _normal_rows,
    _quickstart_module,
    _random_mlp,
)


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


def _ranks64(X, w, k):
    z = omlp.logits(X, *w, dtype=np.float64)
    return np.argsort(-z, kind="stable")[:, :k], z


def _assert_exact(idx, X, w, k, st):
    """Rows that differ from the float64 ranks are rows the float64 rank rule may count as ambiguous: their float64
    gap among ranks 1 .. min(k, C - 1) + 1 lies within the stage's bound beta (tests/f64_stage_cases.mlp_beta); and
    there are no more of them than n_ambiguous."""
    want, z = _ranks64(X, w, k)
    assert idx.shape == want.shape and idx.dtype == np.int32
    bad = np.any(idx != want, axis=1)
    if bad.any():
        kk = min(k, z.shape[1] - 1)
        zs = -np.sort(-z[bad], axis=1)
        gap = (zs[:, :kk] - zs[:, 1 : kk + 1]).min(axis=1)
        beta = K.mlp_beta(np.asarray(X)[bad], *w)
        far = np.flatnonzero(gap > beta)
        assert far.size == 0, (f"rows {np.flatnonzero(bad)[far][:6].tolist()} differ with float64 gaps "
                               f"{(gap / beta)[far][:6].tolist()} x beta")
    assert int(bad.sum()) <= st["n_ambiguous"], f"{int(bad.sum())} rows differ, {st['n_ambiguous']} ambiguous"


def _assert_proba_bound(proba, idx, X, w, path):
    """|p̂ − p| <= p (exp(2δ + 2uL)(1 + (C + 12)u) − 1) + FLT_MIN per selected entry (DESIGN.md 3.6, 3.8); path 2 and
    re-scored rows are float64 rounded once, well inside it."""
    z = omlp.logits(X, *w, dtype=np.float64)
    e = np.exp(z - z.max(axis=1, keepdims=True))
    p = e / e.sum(axis=1, keepdims=True)
    C = z.shape[1]
    delta = _logit_bound(X, w, 5 if path == 5 else 3)
    L = z.max(axis=1) - z.min(axis=1) + 2 * delta
    rel = np.expm1(2 * delta + 2 * U * L) * (1 + (C + 12) * U) + (C + 12) * U
    ps = np.take_along_axis(p, idx.astype(np.int64), axis=1)
    excess = np.abs(proba.astype(np.float64) - ps) - (ps * rel[:, None] + FLT_MIN)
    assert (excess <= 0).all(), f"{int((excess > 0).sum())} entries outside the bound"


def _assert_consistent(engine, m, b, k, exact, idx, proba, st):
    """column 0 = the labels of the same mode; probabilities bit-equal to the probability kernel except re-scored rows"""
    labels, _ = engine.predict_mlp(m, b, exact=exact)
    np.testing.assert_array_equal(idx[:, 0], labels)
    full, sp = engine.predict_mlp_proba(m, b, want_stats=True)
    if st["path"] == 2 or sp["path"] != st["path"]:  # the float64 kernel, or a route the probabilities do not take
        return
    at = np.take_along_axis(full, idx.astype(np.int64), axis=1)
    differs = np.any(at.view(np.uint32) != proba.view(np.uint32), axis=1)
    assert int(differs.sum()) <= (st["n_flagged"] if exact else 0)


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2, 3, 5, 10])
def test_golden_exact_ranks_and_consistency(engine, golden, k):
    w = _weights(golden)
    X = golden["X"].astype(np.float32)
    m = engine.load_mlp(*w)
    b = engine.stage(X)
    idx, proba, st = engine.predict_mlp_topk(m, b, k, exact=True)
    assert st["path"] == (5 if k <= 5 else 2) and st["n_rows"] == len(X)
    assert st["kernel_launches"] == (2 if k <= 5 else 1)
    _assert_exact(idx, X, w, k, st)
    _assert_proba_bound(proba, idx, X, w, st["path"])
    _assert_consistent(engine, m, b, k, True, idx, proba, st)


@pytest.mark.parametrize("H", [16, 32])
@pytest.mark.parametrize("C", [2, 3, 10])
@pytest.mark.parametrize("route", ["tensor_cores", "cuda_cores", "tf32_rows_cuda_cores"])
def test_tile_shapes_ragged_rows(engine, H, C, route, monkeypatch):
    F = {2: 32, 3: 50, 10: 128}[C]
    w = _random_mlp(F, H, C, 10 * H + C)
    m = engine.load_mlp(*w)
    if route == "tf32_rows_cuda_cores":
        monkeypatch.setenv("UML_B200_MLP_TC", "0")
    ks = sorted({k for k in (1, 2, 3, 5) if k <= C} | {C})
    for rows in (1, 127, 129, 30_001):
        X = _normal_rows(rows, F, rows + C) if route == "cuda_cores" else _int_rows(rows, F, rows + C) - 8
        b = engine.stage(X)
        for k in ks:
            tile = 5 if route == "tensor_cores" else 3
            for exact in (True, False):
                idx, proba, st = engine.predict_mlp_topk(m, b, k, exact=exact)
                assert st["path"] == (tile if k <= 5 else 2), (rows, k, st)
                if exact or st["path"] == 2:
                    _assert_exact(idx, X, w, k, st)
                _assert_proba_bound(proba, idx, X, w, st["path"])
                _assert_consistent(engine, m, b, k, exact, idx, proba, st)
                if not exact:  # FAST: descending probabilities
                    assert (np.diff(proba.astype(np.float64), axis=1) <= 0).all()


def test_device_outputs_guard_words_alignment_and_no_proba(engine, golden):
    w = _weights(golden)
    m = engine.load_mlp(*w)
    for rows, X in ((129, _int_rows(129, 64, 3)), (5_000, _normal_rows(5_000, 64, 4))):
        b = engine.stage(X)
        for k in (1, 3, 5, 7):
            idx, proba, st = engine.predict_mlp_topk(m, b, k, exact=True)
            n = rows * k
            for offset in (0, 1):  # 4-byte words: 16-byte aligned, then 4 bytes past it
                ib = torch.full((n + 68,), -7, dtype=torch.int32, device="cuda")
                pb = torch.full((n + 68,), -7.0, dtype=torch.float32, device="cuda")
                _, _, _ = engine.predict_mlp_topk(m, b, k, exact=True, idx_device_ptr=ib.data_ptr() + 4 * offset,
                                                  proba_device_ptr=pb.data_ptr() + 4 * offset)
                torch.cuda.synchronize()
                di, dp = ib.cpu().numpy(), pb.cpu().numpy()
                np.testing.assert_array_equal(di[offset : offset + n], idx.reshape(-1))
                np.testing.assert_array_equal(dp[offset : offset + n].view(np.uint32), proba.reshape(-1).view(np.uint32))
                assert (di[:offset] == -7).all() and (di[offset + n :] == -7).all()
                assert (dp[:offset] == -7).all() and (dp[offset + n :] == -7).all()
            # indices only: host and device
            only, none, _ = engine.predict_mlp_topk(m, b, k, exact=True, want_proba=False)
            assert none is None
            np.testing.assert_array_equal(only, idx)
            ib = torch.full((n + 68,), -7, dtype=torch.int32, device="cuda")
            engine.predict_mlp_topk(m, b, k, exact=True, want_proba=False, idx_device_ptr=ib.data_ptr())
            di = ib.cpu().numpy()
            np.testing.assert_array_equal(di[:n], idx.reshape(-1))
            assert (di[n:] == -7).all()


def test_errors(engine, golden):
    from unionml_b200.engine import EngineError
    from unionml_b200.predictors import mlp_predict_topk

    w = _weights(golden)
    m = engine.load_mlp(*w)
    b = engine.stage(_int_rows(100, 64, 1))
    for k in (0, 11):
        with pytest.raises(EngineError):
            engine.predict_mlp_topk(m, b, k)
    with pytest.raises(ValueError, match="63 features"):
        engine.predict_mlp_topk(m, engine.stage(_int_rows(100, 63, 1)), 3)
    _, module = _quickstart_module(golden)
    bad = np.ones((1000, 64))
    bad[5, 5] = np.inf
    with pytest.raises(ValueError):
        mlp_predict_topk(module, pd.DataFrame(bad))
    with pytest.raises(ValueError, match="0 sample"):
        mlp_predict_topk(module, pd.DataFrame(np.ones((0, 64))))
    for k in (0, 11):
        with pytest.raises(ValueError, match="out of range"):
            mlp_predict_topk(module, pd.DataFrame(np.ones((4, 64))), k=k)
    # NaN in device rows that no staging scan saw: the EXACT guard flags them and the re-score reports them
    x = torch.from_numpy(_int_rows(1000, 64, 2)).cuda()
    x[7, 3] = float("nan")
    wrapped = engine.wrap_device(x.data_ptr(), 1000, 64, keepalive=x)
    with pytest.raises(ValueError):
        engine.predict_mlp_topk(m, wrapped, 3, exact=True)


# ---------------------------------------------------------------------------------------------------------------
def _quickdraw_accuracy(output, target, topk):
    """numpy restatement of the quickdraw template's accuracy helper (as fractions instead of percent)"""
    maxk = min(max(topk), output.shape[1])
    pred = np.argsort(-output, kind="stable")[:, :maxk].T
    correct = pred == target.reshape(1, -1)
    return [correct[: min(k, maxk)].reshape(-1).sum() / len(target) for k in topk]


def test_public_api_against_torch_and_the_metrics(golden):
    from typing import List

    from sklearn.metrics import accuracy_score

    from unionml_b200 import Dataset, Model
    from unionml_b200.model import ModelArtifact
    from unionml_b200.predictors import mlp_accuracy, mlp_predict_proba, mlp_predict_topk, mlp_topk_accuracy

    PytorchModel, module = _quickstart_module(golden)
    w = _weights(golden)
    cols = [f"pixel_{i}" for i in range(64)]
    for frame in (pd.DataFrame(np.random.default_rng(8).integers(0, 17, size=(30_000, 64)).astype(np.float64), columns=cols),
                  pd.DataFrame(np.random.default_rng(9).standard_normal((10_000, 64)), columns=cols)):
        x = torch.from_numpy(frame.values).float()
        with torch.no_grad():
            tv, ti = torch.topk(module(x), 3)
        values, indices = mlp_predict_topk(module, frame, k=3)
        assert values.shape == (len(frame), 3) and values.dtype == np.float32 and indices.dtype == np.int64
        ref, z = _ranks64(frame.values, w, 3)
        agree = np.all(ti.numpy() == ref, axis=1)
        assert agree.mean() > 0.99
        np.testing.assert_array_equal(indices[agree], ti.numpy()[agree])
        assert np.abs(values[agree] - tv.numpy()[agree]).max() < 1e-5
        full = mlp_predict_proba(module, frame)
        assert np.abs(values - np.take_along_axis(full, indices, axis=1)).max() < 1e-5

        target = np.random.default_rng(10).integers(0, 10, size=len(frame))
        target[::3] = ref[::3, 0]  # some hits at rank 1, some further down
        target[1::7] = ref[1::7, 2]
        with torch.no_grad():
            evaluator = accuracy_score(target, [float(c) for c in module(x).argmax(1)])
        got = mlp_accuracy(module, frame, pd.Series(target))
        assert got == accuracy_score(target, omlp.predict_indices_f64(frame.values, *w).astype(float))
        assert abs(got - evaluator) <= (~agree).mean() + 1e-12
        acc = mlp_topk_accuracy(module, frame, target, topk=(1, 5))
        assert acc == pytest.approx(_quickdraw_accuracy(z, target, (1, 5)), abs=0)
        assert mlp_topk_accuracy(module, frame, target, topk=(1, 3, 20))[2] == 1.0  # k beyond n_out: every class

    # the quickdraw template's predictor shape: {class name: probability} of the top 3, through Model.predict
    names = [f"class_{i}" for i in range(10)]
    frame = pd.DataFrame(np.random.default_rng(13).integers(0, 17, size=(200, 64)).astype(np.float64), columns=cols)
    dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
    model = Model(name="quickdraw_shape", init=PytorchModel, dataset=dataset)

    @dataset.reader
    def reader() -> pd.DataFrame:
        return frame.assign(target=0)

    seen = []

    def monitor(module: PytorchModel, features: pd.DataFrame, predictions: dict):
        seen.append(predictions)

    @model.predictor(callbacks=[monitor])
    def predictor(module: PytorchModel, features: pd.DataFrame) -> dict:
        values, indices = mlp_predict_topk(module, features.iloc[:1], k=3)
        return {names[i]: float(v) for i, v in zip(indices[0], values[0])}

    model.artifact = ModelArtifact(module)
    out = model.predict(features=frame.iloc[:1])
    ref, _ = _ranks64(frame.values[:1], w, 3)
    assert list(out) == [names[i] for i in ref[0]]
    assert list(out.values()) == sorted(out.values(), reverse=True)
    assert seen and seen[-1] is out


def test_ten_million_rows_cfg5_shape(engine, golden):
    from bench import digits_rows

    w = _weights(golden)
    m = engine.load_mlp(*w)
    N, k = 10_000_000, 3
    X = np.empty((N, 64), dtype=np.uint8)
    digits_rows(0, N, X)
    b = engine.stage(X)
    idx, proba, st = engine.predict_mlp_topk(m, b, k, exact=True)
    assert st["path"] == 5 and st["n_rows"] == N
    labels, _ = engine.predict_mlp(m, b, exact=True)
    np.testing.assert_array_equal(idx[:, 0], labels)
    full, _ = engine.predict_mlp_proba(m, b)
    at = np.take_along_axis(full, idx.astype(np.int64), axis=1)
    del full
    assert int(np.any(at.view(np.uint32) != proba.view(np.uint32), axis=1).sum()) <= st["n_flagged"]
    bad = 0
    step = 1_000_000
    for lo in range(0, N, step):
        Xc = X[lo : lo + step].astype(np.float32)
        want, _ = _ranks64(Xc, w, k)
        bad += int(np.any(idx[lo : lo + step] != want, axis=1).sum())
        _assert_proba_bound(proba[lo : lo + step], idx[lo : lo + step], Xc, w, 5)
    assert bad <= st["n_ambiguous"]
    print(f"10M x 64 top-3: {st['n_flagged']} rows re-scored in float64, {st['n_ambiguous']} ambiguous, "
          f"kernel {st['kernel_ms']:.3f} ms + re-score {st['recheck_ms']:.3f} ms")
