"""Oracle (test infrastructure only): the PyTorch quickstart predictor, restated in numpy.

Reference: ``unionml:tests/integration/pytorch_app/quickstart.py``

* ``PytorchModel`` (14-24): ``Sequential(Linear(in, hidden), ReLU(), Linear(hidden, out))`` then ``softmax(dim=1)``;
* ``process_features`` (31-32): ``torch.from_numpy(features.values).float()`` - features are cast to float32;
* ``predictor`` (68-70): ``[float(x) for x in module(process_features(features)).argmax(1)]``.

``torch.nn.Linear`` computes ``x @ W.T + b`` with ``W`` of shape (out, in).  softmax is strictly monotone, so the
argmax of the probabilities is the argmax of the logits unless float32 rounding collapses two near-equal logits to the
same probability (then torch returns the first index).  ``predict_indices_f64`` is the exact-arithmetic-grade label
(float64 network on the float32-cast features); ``forward_f32`` mirrors the reference's float32 pipeline.  Pinned
against torch itself in ``tests/test_oracle_golden.py`` / ``tests/golden/mlp_64_32_10.npz``.
"""
from __future__ import annotations

import numpy as np


def logits(X, w1, b1, w2, b2, dtype=np.float64) -> np.ndarray:
    X = np.asarray(X, dtype=np.float32).astype(dtype)  # process_features(): .float()
    h = np.maximum(X @ np.asarray(w1, dtype).T + np.asarray(b1, dtype), 0)
    return h @ np.asarray(w2, dtype).T + np.asarray(b2, dtype)


def forward_f32(X, w1, b1, w2, b2) -> np.ndarray:
    """softmax(logits) in float32, as ``PytorchModel.forward`` returns it."""
    z = logits(X, w1, b1, w2, b2, np.float32)
    z = z - z.max(axis=1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=1, keepdims=True)


def predict_indices_f32(X, w1, b1, w2, b2) -> np.ndarray:
    return forward_f32(X, w1, b1, w2, b2).argmax(axis=1)


def predict_indices_f64(X, w1, b1, w2, b2) -> np.ndarray:
    return logits(X, w1, b1, w2, b2, np.float64).argmax(axis=1)


def logit_margin_f64(X, w1, b1, w2, b2) -> np.ndarray:
    z = logits(X, w1, b1, w2, b2, np.float64)
    part = np.partition(z, z.shape[1] - 2, axis=1)
    return part[:, -1] - part[:, -2]


def canonical_predictor(module_weights: dict, features) -> list:
    """``[float(x) for x in module(process_features(features)).argmax(1)]`` with the float32 pipeline."""
    feats = features.to_numpy() if hasattr(features, "to_numpy") else np.asarray(features)
    idx = predict_indices_f32(feats, module_weights["w1"], module_weights["b1"], module_weights["w2"], module_weights["b2"])
    return [float(x) for x in idx]
