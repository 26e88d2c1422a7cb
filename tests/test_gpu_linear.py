"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on the same seeded inputs.

Bar: labels are index work -> bit-exact.  In EXACT mode the engine's labels must equal the float64 oracle
(= scikit-learn's float64 path) on every row.  In FAST mode (plain fp32) differences are only allowed on rows whose
float64 top-2 margin is below the fp32 error bound, and the test states that bound.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from oracle import linear as olin

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there (the -m gpu run happens on an H100)
    pytest.skip("needs a CUDA device", allow_module_level=True)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def digits_rows(seed, rows, dtype=np.float32):
    return np.random.default_rng(seed).integers(0, 17, size=(rows, 64), dtype=np.uint8).astype(dtype)


def oracle_idx(X, coef, intercept):
    return olin.predict_indices(olin.decision_function(np.asarray(X, dtype=np.float64), coef, intercept)).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# golden vectors
# ---------------------------------------------------------------------------------------------------------------
def test_known_answer_through_predictor(digits_model, known_answer):
    """[8.0, 8.0, 0.0]: unionml:tests/unit/test_aws_lambda_handler.py:127,159 - now on the GPU."""
    from sklearn.linear_model import LogisticRegression

    from unionml_b200.predictors import linear_argmax

    est = LogisticRegression()
    est.coef_, est.intercept_, est.classes_ = digits_model["coef"], digits_model["intercept"], digits_model["classes"]
    est.n_features_in_ = 64
    for key, want in (("sample3_random_state99", [8.0, 8.0, 0.0]), ("sample5_random_state42", [6.0, 9.0, 3.0, 7.0, 2.0])):
        frame = pd.DataFrame(known_answer[key]["records"])[known_answer["feature_names"]]
        got = linear_argmax(est, frame)
        assert got == want
        assert all(isinstance(x, float) for x in got)


def test_committed_fixture(engine, digits_model, synthetic_digits):
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"], digits_model["classes"])
    X = synthetic_digits["X"]
    for arr in (X.astype(np.float32), X.astype(np.float64), X, np.asfortranarray(X.astype(np.float64))):
        idx, stats = engine.predict_host(m, arr, exact=True)
        np.testing.assert_array_equal(digits_model["classes"][idx], synthetic_digits["labels_f64"])
        b = engine.stage(arr)
        idx2, st2 = engine.predict(m, b, exact=True)
        np.testing.assert_array_equal(idx2, idx)
        assert st2["path"] == 1 and st2["kernel_launches"] == 1  # flagged rows are re-scored by a warp of the same launch


# ---------------------------------------------------------------------------------------------------------------
# seeded parity at sizes the oracle finishes in seconds
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 31, 127, 128, 129, 1000, 4097, 300_001])
def test_exact_parity_ragged_sizes(engine, digits_model, rows):
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    X = digits_rows(rows, rows)
    want = oracle_idx(X, digits_model["coef"], digits_model["intercept"])
    got, stats = engine.predict(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, want)
    assert stats["n_rows"] == rows and stats["n_nonfinite"] == 0
    got_h, _ = engine.predict_host(m, X, exact=True, chunk_rows=1024)
    np.testing.assert_array_equal(got_h, want)


def test_empty_batch(engine, digits_model):
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    X = np.zeros((0, 64), dtype=np.float32)
    got, _ = engine.predict_host(m, X)
    assert got.shape == (0,)
    got, _ = engine.predict(m, engine.stage(X))
    assert got.shape == (0,)


def test_exact_vs_fast_two_million(engine, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    m = engine.load_linear(coef, intercept)
    X = np.concatenate([digits_rows(k, 500_000) for k in range(4)])
    scores = olin.decision_function(X.astype(np.float64), coef, intercept)
    want = olin.predict_indices(scores).astype(np.int32)
    b = engine.stage(X)
    exact, st = engine.predict(m, b, exact=True)
    np.testing.assert_array_equal(exact, want)
    # the guard flags few rows (< 0.1 %) and re-scores them; none is a genuine float64 tie on this data
    assert 0 < st["n_flagged"] < 2000, st
    assert st["n_ambiguous"] == 0
    fast, stf = engine.predict(m, b, exact=False)
    assert stf["kernel_launches"] == 1
    diff = np.flatnonzero(fast != want)
    # fp32 error bound of a 64-term FMA chain: (F+4) 2^-24 * (|b| + sum |x w|)  <=  68 * 6e-8 * A
    A = np.abs(intercept).max() + np.abs(X.astype(np.float64)) @ np.abs(coef).max(axis=0)
    margin = olin.top2_margin(scores)
    assert np.all(margin[diff] <= 2 * 68 * 2.0**-24 * A[diff])
    assert len(diff) < 50


def test_layouts_and_dtypes(engine, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    m = engine.load_linear(coef, intercept)
    base = digits_rows(7, 50_000, np.float64)
    want = oracle_idx(base, coef, intercept)
    frame = pd.DataFrame(base, columns=[f"pixel_{i}" for i in range(64)])  # pandas block: feature-major
    wide = np.zeros((50_000, 80), dtype=np.float32)
    wide[:, :64] = base
    variants = {
        "f64_c": base,
        "f64_f": np.asfortranarray(base),
        "f32_c": base.astype(np.float32),
        "f32_f": np.asfortranarray(base.astype(np.float32)),
        "i64": base.astype(np.int64),
        "i32_f": np.asfortranarray(base.astype(np.int32)),
        "u8": base.astype(np.uint8),
        "frame": frame,
        "row_strided": wide[:, :64],
        "noncontig": base[::2],
    }
    for name, arr in variants.items():
        w = want[::2] if name == "noncontig" else want
        got, _ = engine.predict_host(m, arr, exact=True)
        np.testing.assert_array_equal(got, w, err_msg=name)
        got2, _ = engine.predict(m, engine.stage(arr), exact=True)
        np.testing.assert_array_equal(got2, w, err_msg=name)


def test_queue_and_kernel_rescore_agree(engine, digits_model):
    """UML_B200_RESCORE_MODE=queue: flagged rows go through a shared-memory queue to a re-score warp of the tile kernel
    (one launch); =kernel: flag list + rescore_f64_kernel (two launches).  Same labels, same counters - also when most
    rows are near-ties and the queue backs up (the scoring warps then re-score their own rows)."""
    import os
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parent.parent
    code = (
        "import sys, numpy as np; sys.path.insert(0, %r)\n"
        "from unionml_b200.engine import Engine\n"
        "z = np.load(%r); e = Engine(0); m = e.load_linear(z['coef'], z['intercept'])\n"
        "X = np.random.default_rng(31).integers(0, 17, size=(1_500_000, 64), dtype=np.uint8).astype(np.float32)\n"
        "idx, st = e.predict(m, e.stage(X), exact=True)\n"
        "print(st['kernel_launches'], st['n_flagged'], int(idx.astype(np.int64).sum()), int((idx * np.arange(idx.size) %% 1000003).sum()))\n"
        "m0 = e.load_linear(np.zeros((5, 64)), np.zeros(5))   # every row is a five-way tie: all rows flagged\n"
        "idx0, st0 = e.predict(m0, e.stage(X[:300_000]), exact=True)\n"
        "print(st0['n_flagged'], st0['n_ambiguous'], int(idx0.sum()))\n"
        "u8 = e.device_alloc(300_000); e.predict_peers(m0, e.stage(X[:300_000]), [u8.ptr], 0, exact=True, want_stats=True, label_bytes=1)\n"
        "print(int(e.take_labels(u8.ptr, 300_000, np.arange(5.0), label_bytes=1).sum()))\n"
    ) % (str(root), str(root / "tests" / "golden" / "digits_lr.npz"))
    outs = []
    for mode in ("queue", "kernel"):
        env = dict(os.environ, UML_B200_RESCORE_MODE=mode)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append([ln.split() for ln in r.stdout.strip().splitlines()])
    assert outs[0][0][0] == "1" and outs[1][0][0] == "2"   # one launch with the queue, two with the flag list
    assert outs[0][0][1:] == outs[1][0][1:] and int(outs[0][0][1]) > 0
    assert outs[0][1] == outs[1][1] == ["300000", "300000", "0"]   # all flagged, all ambiguous, first index wins
    assert outs[0][2] == outs[1][2] == ["0"]


def test_lossy_float64_features_use_the_f64_copy(engine):
    """Features that do not survive the fp32 down-cast: exact mode re-scores flagged rows from the float64 copy."""
    rng = np.random.default_rng(5)
    coef = rng.standard_normal((5, 12))
    intercept = rng.standard_normal(5)
    X = rng.standard_normal((100_000, 12))
    # plant near-ties that only float64 features resolve
    X[:1000] = X[0]
    X[:1000, 3] += np.linspace(-1e-9, 1e-9, 1000)
    want = oracle_idx(X, coef, intercept)
    m = engine.load_linear(coef, intercept)
    b = engine.stage(X, keep_f64=True)
    assert not b.lossless
    got, st = engine.predict(m, b, exact=True)
    np.testing.assert_array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------
# tie / edge semantics
# ---------------------------------------------------------------------------------------------------------------
def test_ties_first_maximum_wins(engine):
    coef = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0], [0.0, 1.0]])
    intercept = np.zeros(4)
    X = np.array([[2.0, 1.0], [1.0, 2.0], [1.0, 1.0], [0.0, 0.0]], dtype=np.float32)
    m = engine.load_linear(coef, intercept)
    for exact in (True, False):
        got, st = engine.predict(m, engine.stage(X), exact=exact)
        np.testing.assert_array_equal(got, [0, 2, 0, 0])
    np.testing.assert_array_equal(olin.exact_predict_indices(X, coef, intercept), [0, 2, 0, 0])


def test_binary_model(engine, binary_mock):
    m = engine.load_linear(binary_mock["coef"], binary_mock["intercept"], binary_mock["classes"])
    got, _ = engine.predict_host(m, binary_mock["X"], exact=True)
    np.testing.assert_array_equal(binary_mock["classes"][got], binary_mock["labels"])
    # score exactly zero -> class 0 (strict '>' of _base.py:416)
    m0 = engine.load_linear(np.array([[1.0]]), np.array([0.0]))
    got, _ = engine.predict_host(m0, np.array([[0.0], [1e-30], [-1.0]]), exact=True)
    np.testing.assert_array_equal(got, [0, 1, 0])


@pytest.mark.parametrize("n_classes", [2, 3, 7, 10, 16, 17, 40])
@pytest.mark.parametrize("n_features", [1, 3, 33, 64, 100])
def test_shapes(engine, n_classes, n_features):
    rng = np.random.default_rng(n_classes * 1000 + n_features)
    coef = rng.standard_normal((n_classes, n_features))
    intercept = rng.standard_normal(n_classes)
    X = rng.integers(-8, 9, size=(20_011, n_features)).astype(np.float32)
    want = oracle_idx(X, coef, intercept)
    m = engine.load_linear(coef, intercept)
    got, st = engine.predict(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, want)
    assert st["path"] == (1 if n_classes <= 16 else 2)


def test_mnist_shape_784(engine):
    rng = np.random.default_rng(1)
    coef = (rng.standard_normal((10, 784)) * 0.05).astype(np.float32)
    intercept = np.random.default_rng(2).standard_normal(10).astype(np.float32)
    X = (rng.integers(0, 256, size=(100_000, 784)).astype(np.float32)) / np.float32(255.0)
    want = oracle_idx(X, coef.astype(np.float64), intercept.astype(np.float64))
    m = engine.load_linear(coef, intercept)
    got, st = engine.predict(m, engine.stage(X), exact=True)
    np.testing.assert_array_equal(got, want)
    assert st["path"] == 1


def test_affine_fold_matches_scaler_pipeline(engine, digits_model):
    """Pipeline(StandardScaler, LogisticRegression) of docs/tutorials/mnist.md:116-124, scaler folded into W, b."""
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    X = digits_rows(11, 100_000, np.float64)
    mu, sd = X.mean(axis=0), X.std(axis=0) + 0.5
    want = oracle_idx((X - mu) / sd, coef, intercept)
    m = engine.load_linear(coef, intercept)
    m.set_affine(shift=mu, scale=1.0 / sd)
    got, _ = engine.predict_host(m, X, exact=True)
    assert (got != want).sum() == 0


# ---------------------------------------------------------------------------------------------------------------
# errors at the boundary
# ---------------------------------------------------------------------------------------------------------------
def test_nonfinite_raises_value_error(engine, digits_model):
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    for bad_value in (np.nan, np.inf, -np.inf):
        X = digits_rows(3, 5000)
        X[4321, 17] = bad_value
        with pytest.raises(ValueError):
            engine.predict_host(m, X, exact=True)
        with pytest.raises(ValueError):
            engine.predict_host(m, X, exact=False)
        with pytest.raises(ValueError):
            engine.stage(X)
        # device-resident rows that never went through staging: exact mode still catches it
        b = engine.stage(X, check_finite=False)
        with pytest.raises(ValueError):
            engine.predict(m, b, exact=True)


def test_wrong_feature_count(engine, digits_model):
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    with pytest.raises(ValueError, match="63 features"):
        engine.predict_host(m, np.zeros((4, 63), dtype=np.float32))


# ---------------------------------------------------------------------------------------------------------------
# full BASELINE size (10M x 64): size-independent properties + streamed oracle comparison
# ---------------------------------------------------------------------------------------------------------------
def test_full_size_ten_million(engine, digits_model):
    coef, intercept = digits_model["coef"], digits_model["intercept"]
    m = engine.load_linear(coef, intercept)
    N = 10_000_000
    X = engine.pinned_empty((N, 64), np.float32)
    for k in range(10):
        X[k * 1_000_000 : (k + 1) * 1_000_000] = digits_rows(k, 1_000_000)
    b = engine.stage(X)
    labels, st = engine.predict(m, b, exact=True)
    assert st["n_rows"] == N and st["n_ambiguous"] == 0 and 0 < st["n_flagged"] < N // 1000
    # (1) every row against the float64 oracle, streamed in 1M-row chunks
    for k in range(10):
        sl = slice(k * 1_000_000, (k + 1) * 1_000_000)
        np.testing.assert_array_equal(labels[sl], oracle_idx(X[sl], coef, intercept))
    # (2) chunking invariance: host-streamed path == resident path
    streamed, _ = engine.predict_host(m, X, exact=True)
    np.testing.assert_array_equal(streamed, labels)
    # (3) permutation equivariance on a shuffled million
    perm = np.random.default_rng(0).permutation(1_000_000)
    sub, _ = engine.predict_host(m, X[:1_000_000][perm], exact=True)
    np.testing.assert_array_equal(sub, labels[:1_000_000][perm])
    # (4) label histogram is a checksum that must agree between modes except on flagged rows
    fast, _ = engine.predict(m, b, exact=False)
    assert (fast != labels).sum() <= st["n_flagged"]


# ---------------------------------------------------------------------------------------------------------------
# ring-protocol regression: foreign kernels between launches perturb TMA completion order (cold TLB / L2).  A first
# version of the kernel let a consumer warp run one barrier phase ahead of a stage's previous occupant and faulted
# or hung within a few launches in exactly this setting; UML_B200_STAGES=8 is the shallowest legal ring.
# ---------------------------------------------------------------------------------------------------------------
_RING_WORKER = r'''
import os, sys
import numpy as np, torch
sys.path.insert(0, os.environ["UML_ROOT"])
from oracle import linear as olin
from unionml_b200.engine import Engine
z = np.load(os.path.join(os.environ["UML_ROOT"], "tests", "golden", "digits_lr.npz"))
dev = torch.device("cuda", 0)
eng = Engine(0); s = torch.cuda.Stream(device=dev); torch.cuda.set_stream(s); eng.set_stream(s.cuda_stream)
m = eng.load_linear(z["coef"], z["intercept"])
X = np.random.default_rng(3).integers(0, 17, size=(3_000_000, 64), dtype=np.uint8).astype(np.float32)
want = olin.predict_indices(olin.decision_function(X.astype(np.float64), z["coef"], z["intercept"])).astype(np.int32)
b = eng.stage(X)
out = torch.empty(X.shape[0], dtype=torch.int32, device=dev)
a = torch.randn(2048, 2048, device=dev, dtype=torch.bfloat16); c = torch.empty_like(a); d = torch.zeros(1 << 22, device=dev)
for i in range(60):
    out.fill_(-1)
    eng.predict(m, b, exact=(i % 2 == 0), out_device_ptr=out.data_ptr(), want_stats=False)
    if i % 3 == 0: torch.matmul(a, a, out=c)
    elif i % 3 == 1: d.add_(1)
    else: torch.cuda._sleep(500_000)
    if i % 10 == 0:
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert (got != want).sum() <= (0 if i % 2 == 0 else 5), i
torch.cuda.synchronize()
print("ring ok")
'''


@pytest.mark.parametrize("stages", ["", "8"])
def test_ring_protocol_with_foreign_kernels_between_launches(tmp_path, stages):
    import os
    import subprocess
    import sys
    from pathlib import Path

    script = tmp_path / "ring_worker.py"
    script.write_text(_RING_WORKER)
    env = dict(os.environ, UML_ROOT=str(Path(__file__).resolve().parent.parent))
    if stages:
        env["UML_B200_STAGES"] = stages
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ring ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------
# the README digits app end to end on the device path (BASELINE.json configs[0] and [3])
# ---------------------------------------------------------------------------------------------------------------
def test_digits_app_and_fastapi_on_the_device_path(tmp_path, monkeypatch):
    from typing import List

    from fastapi import FastAPI
    from fastapi.testclient import TestClient
    from sklearn.datasets import load_digits
    from sklearn.linear_model import LogisticRegression
    from sklearn.metrics import accuracy_score

    from unionml_b200 import Dataset, Model
    from unionml_b200.predictors import linear_argmax

    def make_app():
        dataset = Dataset(name="digits_dataset", test_size=0.2, shuffle=True, targets=["target"])
        model = Model(name="digits_classifier", init=LogisticRegression, dataset=dataset)

        @dataset.reader
        def reader() -> pd.DataFrame:
            return load_digits(as_frame=True).frame

        @model.trainer
        def trainer(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> LogisticRegression:
            return estimator.fit(features, target.squeeze())

        seen = []

        def monitor(estimator: LogisticRegression, features: pd.DataFrame, predictions: List[float]):
            seen.append(len(predictions))

        @model.predictor(callbacks=[monitor])
        def predictor(estimator: LogisticRegression, features: pd.DataFrame) -> List[float]:
            return linear_argmax(estimator, features)  # the one changed line of the README app

        @model.evaluator
        def evaluator(estimator: LogisticRegression, features: pd.DataFrame, target: pd.DataFrame) -> float:
            return float(accuracy_score(target.squeeze(), predictor(estimator, features)))

        return model, seen

    model, seen = make_app()
    est, metrics = model.train(hyperparameters={"C": 1.0, "max_iter": 1000})
    # evaluator ran the GPU predictor on both splits: same metrics as the CPU pipeline (SURVEY.md 8d cfg 1)
    assert metrics["train"] == 1.0 and abs(metrics["test"] - 0.9639) < 1e-3
    frame = load_digits(as_frame=True).frame
    feats = frame[[c for c in frame if c != "target"]]
    assert model.predict(features=feats.sample(3, random_state=99)) == [8.0, 8.0, 0.0]
    assert model.predict(features=frame.sample(5, random_state=42)) == [6.0, 9.0, 3.0, 7.0, 2.0]
    with pytest.raises(ValueError, match="At least one of features"):  # no-arg reader: same guard as ref. model.py:727
        model.predict()
    whole = model.predict(features=frame)  # the feature loader drops the target column (dataset.py:515-518)
    assert whole == [float(x) for x in est.predict(feats)] and seen[-1] == len(frame)

    path = tmp_path / "model.joblib"
    model.save(path)
    served, _ = make_app()
    app = FastAPI()
    served.serve(app)
    monkeypatch.setenv("UNIONML_MODEL_PATH", str(path))
    with TestClient(app) as client:
        assert client.get("/health").status_code == 200
        r = client.post("/predict", json={"features": feats.sample(32, random_state=7).to_dict(orient="records")})
        assert r.status_code == 200
        assert r.json() == [float(x) for x in est.predict(feats.sample(32, random_state=7))]
        # reordered columns: the default feature loader keeps the request's order, and the predictor raises the same
        # ValueError sklearn raises (utils/validation.py:2769); TestClient re-raises server exceptions
        bad = feats.sample(2, random_state=1).iloc[:, ::-1].to_dict(orient="records")
        with pytest.raises(ValueError, match="feature names"):
            client.post("/predict", json={"features": bad})
    with pytest.raises(ValueError, match="feature names"):
        linear_argmax(est, feats.iloc[:4, ::-1])


def test_device_side_take_and_accuracy(engine, digits_model):
    """SURVEY.md 8(f)4: classes_.take + float conversion and the evaluator's match count on the device."""
    from sklearn.linear_model import LogisticRegression

    from unionml_b200.predictors import linear_accuracy

    coef, intercept = digits_model["coef"], digits_model["intercept"]
    classes = np.array([3.0, 1.5, -2.0, 7.0, 9.0, 11.0, 0.0, 4.0, 5.0, 6.0])  # not the identity map
    m = engine.load_linear(coef, intercept)
    X = digits_rows(21, 200_001)
    idx = oracle_idx(X, coef, intercept)
    b = engine.stage(X)
    buf = engine.device_alloc(4 * b.n_rows)
    engine.predict(m, b, exact=True, out_device_ptr=buf.ptr, want_stats=True)
    got = engine.take_labels(buf.ptr, b.n_rows, classes)
    np.testing.assert_array_equal(got, classes[idx])
    target = classes[idx].copy()
    target[::7] += 100.0  # 1/7 of the rows are "wrong"
    hits = engine.count_equal(buf.ptr, b.n_rows, classes, target)
    assert hits == int((classes[idx] == target).sum())
    est = LogisticRegression()
    est.coef_, est.intercept_, est.classes_, est.n_features_in_ = coef, intercept, classes, 64
    assert linear_accuracy(est, X, target) == hits / b.n_rows
    # uint8 label vectors go through the same kernels
    u8 = engine.device_alloc(b.n_rows)
    engine.predict_peers(m, b, [u8.ptr], 0, exact=True, want_stats=True, label_bytes=1)
    np.testing.assert_array_equal(engine.take_labels(u8.ptr, b.n_rows, classes, label_bytes=1), classes[idx])
