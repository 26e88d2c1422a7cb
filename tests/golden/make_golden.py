"""Generate the golden fixtures under tests/golden/ (run once in the build container, outputs committed).

The reference (``unionml``) cannot be imported here (flytekit absent), so the fixtures are produced by running the
reference's *arithmetic dependency* - scikit-learn, the library its canonical predictor calls - through a hand
restatement of the default ``Dataset`` pipeline:

* ``unionml:unionml/dataset.py:44-53``  defaults ``test_size=0.2, shuffle=True, random_state=12345``
* ``dataset.py:477-487``  default splitter = ``train_test_split(data, test_size, random_state, shuffle)``
* ``dataset.py:489-504``  default parser   = all non-target columns / ``data[targets]``
* trainer = ``estimator.fit(features, target.squeeze())`` (``unionml:README.md:80-85``)

Known answers reproduced: ``[8.0, 8.0, 0.0]`` (``unionml:tests/unit/test_aws_lambda_handler.py:117-127``) and
the quickstart sample (``unionml:tests/integration/sklearn_app/quickstart.py:34-40``).

    python tests/golden/make_golden.py
"""
import json
from pathlib import Path

import numpy as np
from sklearn.datasets import load_digits
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import train_test_split

HERE = Path(__file__).parent


def train_digits(max_iter: int):
    frame = load_digits(as_frame=True).frame
    train, _test = train_test_split(frame, test_size=0.2, random_state=12345, shuffle=True)
    feats = [c for c in frame if c not in ["target"]]
    est = LogisticRegression(C=1.0, max_iter=max_iter).fit(train[feats], train[["target"]].squeeze())
    return frame, feats, est


def main():
    frame, feats, est = train_digits(1000)

    # ---- known answers ------------------------------------------------------------------------------------------
    s3 = frame[feats].sample(3, random_state=99)
    ka3 = [float(x) for x in est.predict(s3)]
    assert ka3 == [8.0, 8.0, 0.0], ka3
    s5 = frame.sample(5, random_state=42)[feats]
    ka5 = [float(x) for x in est.predict(s5)]
    assert ka5 == [6.0, 9.0, 3.0, 7.0, 2.0], ka5
    (HERE / "known_answer.json").write_text(
        json.dumps(
            {
                "source": "tests/unit/test_aws_lambda_handler.py:117-127 ([8,8,0]); "
                "tests/integration/sklearn_app/quickstart.py:34-40 ([6,9,3,7,2])",
                "feature_names": feats,
                "sample3_random_state99": {"records": s3.to_dict(orient="records"), "expected": ka3},
                "sample5_random_state42": {"records": s5.to_dict(orient="records"), "expected": ka5},
            },
            indent=1,
        )
    )

    # ---- the trained digits model (cfg 2 uses exactly these W, b) -----------------------------------------------
    np.savez_compressed(
        HERE / "digits_lr.npz",
        coef=est.coef_,
        intercept=est.intercept_,
        classes=est.classes_,
        n_iter=est.n_iter_,
    )

    # ---- seeded synthetic batch in the digits pixel domain, with scikit-learn's labels --------------------------
    rng = np.random.default_rng(2024)
    X = rng.integers(0, 17, size=(4096, 64), dtype=np.uint8)
    y64 = est.predict(X.astype(np.float64))
    est32 = LogisticRegression(C=1.0, max_iter=1000)
    est32.coef_ = est.coef_.astype(np.float32)
    est32.intercept_ = est.intercept_.astype(np.float32)
    est32.classes_ = est.classes_
    est32.n_features_in_ = 64
    y32 = est32.predict(X.astype(np.float32))
    np.savez_compressed(HERE / "synthetic_digits_4096.npz", X=X, labels_f64=y64, labels_f32=y32)

    # ---- binary model on the reference's mock_data fixture (tests/unit/model_fixtures.py:12-20) -----------------
    x = np.array([1, 2, 3, 4] * 25, dtype=np.float64)[:, None]
    y = np.array([0, 1, 0, 1] * 25)
    b = LogisticRegression().fit(x, y)
    np.savez_compressed(
        HERE / "binary_mock.npz", coef=b.coef_, intercept=b.intercept_, classes=b.classes_, X=x, labels=b.predict(x)
    )
    print("wrote fixtures:", sorted(p.name for p in HERE.glob("*.np*")), "known_answer.json")


if __name__ == "__main__":
    main()


def make_mlp_golden():
    """PytorchModel(64, 32, 10) of tests/integration/pytorch_app/quickstart.py:14-24,80 with torch.manual_seed(0),
    and torch's own labels on a seeded digits-domain batch (the reference predictor run as written)."""
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    class PytorchModel(nn.Module):
        def __init__(self, in_dims: int, hidden_dims: int, out_dims: int):
            super().__init__()
            self.layers = nn.Sequential(nn.Linear(in_dims, hidden_dims), nn.ReLU(), nn.Linear(hidden_dims, out_dims))

        def forward(self, features):
            return F.softmax(self.layers(features), dim=1)

    torch.manual_seed(0)
    module = PytorchModel(64, 32, 10)
    X = np.random.default_rng(2025).integers(0, 17, size=(4096, 64), dtype=np.uint8)
    with torch.no_grad():
        labels = module(torch.from_numpy(X.astype(np.float64)).float()).argmax(1).numpy()
    sd = module.state_dict()
    np.savez_compressed(
        HERE / "mlp_64_32_10.npz",
        w1=sd["layers.0.weight"].numpy(), b1=sd["layers.0.bias"].numpy(),
        w2=sd["layers.2.weight"].numpy(), b2=sd["layers.2.bias"].numpy(),
        X=X, labels_torch=labels,
    )
    print("wrote mlp_64_32_10.npz; label histogram", np.bincount(labels, minlength=10))


if __name__ == "__main__" and "--mlp" in __import__("sys").argv:
    make_mlp_golden()
