"""Oracle (test infrastructure only): numpy restatement of scikit-learn's linear-classifier predict.

Follows ``sklearn/linear_model/_base.py`` (scikit-learn 1.9.0, the third-party dependency that holds
the arithmetic of the reference's hot path; reference call sites: ``unionml:README.md:92``,
``unionml:tests/integration/sklearn_app/quickstart.py:26``,
``unionml:tests/unit/model_fixtures.py:71``):

* ``decision_function`` (``_base.py:366-396``): ``scores = X @ coef_.T + intercept_``; a single-row
  ``coef_`` (binary problem) is flattened to 1-D.
* ``predict`` (``_base.py:398-427``): 1-D scores -> ``(scores > 0)``; 2-D -> ``argmax(axis=1)``
  (numpy: first maximum wins); then ``classes_.take(indices)``.
* input validation (``sklearn/utils/validation.py:107`` ``_assert_all_finite``, ``:2868`` feature
  count): NaN/Inf and a wrong number of features raise ``ValueError``.

Parity status: pinned against scikit-learn in-process and against the reference's known-answer vector
(``tests/test_oracle_golden.py``).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np


def validate_features(X, n_features_in: int) -> np.ndarray:
    """``validate_data(reset=False)`` as far as this path needs it.

    dtype rule of ``check_array(dtype="numeric")``: float32/float64 (and ints) are kept, ``object`` becomes
    float64; the matmul against a float64 ``coef_`` then promotes.  NaN/Inf raise the same ``ValueError``
    family scikit-learn raises (``validation.py:107-171``).
    """
    X = np.asarray(X)
    if X.dtype == object:
        X = X.astype(np.float64)
    if X.ndim != 2:
        raise ValueError(f"Expected 2D array, got {X.ndim}D array instead")
    if X.shape[1] != n_features_in:
        raise ValueError(
            f"X has {X.shape[1]} features, but the estimator is expecting {n_features_in} features as input."
        )
    if X.dtype.kind == "f" and not np.isfinite(X).all():
        has_nan = bool(np.isnan(X).any())
        raise ValueError("Input X contains NaN." if has_nan else "Input X contains infinity or a value too large")
    return X


def decision_function(X: np.ndarray, coef: np.ndarray, intercept: np.ndarray) -> np.ndarray:
    """``_base.py:388-396``: ``safe_sparse_dot(X, coef_.T) + intercept_`` (dense case = ``a @ b``)."""
    coef = np.asarray(coef)
    coef_T = coef.T if coef.ndim == 2 else coef
    scores = X @ coef_T + np.asarray(intercept)
    if scores.ndim > 1 and scores.shape[1] == 1:
        return scores.reshape(-1)
    return scores


def predict_indices(scores: np.ndarray) -> np.ndarray:
    """``_base.py:415-418``."""
    if scores.ndim == 1:
        return (scores > 0).astype(np.int64)
    return np.argmax(scores, axis=1)


def predict(X, coef, intercept, classes) -> np.ndarray:
    """``LinearClassifierMixin.predict`` (``_base.py:398-427``)."""
    coef = np.asarray(coef)
    n_features = coef.shape[-1]
    X = validate_features(X, n_features)
    idx = predict_indices(decision_function(X, coef, intercept))
    return np.asarray(classes).take(idx, axis=0)


def canonical_predictor(estimator, features) -> list:
    """The reference's canonical user predictor (``unionml:README.md:87-92``):
    ``[float(x) for x in estimator.predict(features)]`` with ``estimator.predict`` restated above."""
    feats = features.to_numpy() if hasattr(features, "to_numpy") else np.asarray(features)
    labels = predict(feats, estimator.coef_, estimator.intercept_, estimator.classes_)
    return [float(x) for x in labels]


# ----------------------------------------------------------------------------------------------------------------------
# exact arithmetic (small cases only): what "the argmax of the real-valued scores" is, independent of summation order
# ----------------------------------------------------------------------------------------------------------------------
def exact_scores(x_row, coef, intercept) -> list:
    """Scores of one row in exact rational arithmetic (every float is a dyadic rational)."""
    coef = np.asarray(coef, dtype=np.float64)
    intercept = np.asarray(intercept, dtype=np.float64)
    if coef.ndim == 1:
        coef = coef[None, :]
    xs = [Fraction(float(v)) for v in np.asarray(x_row, dtype=np.float64)]
    out = []
    for c in range(coef.shape[0]):
        s = Fraction(float(intercept[c] if intercept.ndim else intercept))
        for xi, wi in zip(xs, coef[c]):
            s += xi * Fraction(float(wi))
        out.append(s)
    return out


def exact_predict_indices(X, coef, intercept) -> np.ndarray:
    """Exact-arithmetic labels with numpy's tie rule (first maximum; binary: strictly positive -> 1)."""
    X = np.asarray(X)
    coef = np.asarray(coef)
    binary = coef.ndim == 1 or coef.shape[0] == 1
    out = np.empty(X.shape[0], dtype=np.int64)
    for r in range(X.shape[0]):
        s = exact_scores(X[r], coef, intercept)
        if binary:
            out[r] = 1 if s[0] > 0 else 0
        else:
            best = 0
            for c in range(1, len(s)):
                if s[c] > s[best]:
                    best = c
            out[r] = best
    return out


def top2_margin(scores: np.ndarray) -> np.ndarray:
    """Gap between the best and second-best score per row (0-margin rows are exact ties)."""
    if scores.ndim == 1:
        return np.abs(scores)
    part = np.partition(scores, scores.shape[1] - 2, axis=1)
    return part[:, -1] - part[:, -2]
