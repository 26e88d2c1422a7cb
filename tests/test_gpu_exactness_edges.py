"""EXACT mode against exact arithmetic where the margin guards are weakest: below FLT_MIN and on near-ties.

The linear tile kernel and both MLP kernels certify a row when its fp32 margin exceeds twice an error bound, and
re-score the others in float64 (DESIGN.md 3.2-3.4).  A bound that is too small gives wrong labels with no flag and
no counter.  These tests plant rows where a relative-only bound fails (underflow of weights, features, products and
biases; the tf32 split of tiny W1 weights; tensor-core flushes), and sweep near-ties whose margins span 0.01x..100x
(MLP: 1e-4x..100x) the kernels' own bounds on data with exponents spread over 2^+-20.  The reference is exact
arithmetic (Fractions) on planted and float64-ambiguous rows, the float64 oracle elsewhere.
"""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import linear as olin
from oracle import mlp as omlp
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

Q = 2.0**-149  # smallest fp32 subnormal
U = 2.0**-24
E = 2.0**-74


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def linear_thr(F):
    """p.thr of the tile kernel (linear_margin_thr): certain iff margin > thr * A."""
    return float(np.float32(2.0 * (F + 4.0) * U * (1.0 + F * 2.0**-21) * 1.0001))


# ---------------------------------------------------------------------------------------------------------------
# linear: planted underflow rows (classes 0 and 1, the first k features); each exact label differs from what a
# relative-only guard lets the fp32 chain certify
# ---------------------------------------------------------------------------------------------------------------
LINEAR_CONSTRUCTIONS = {
    # (float)4e-46 == 0 on upload, so wmax = 0 and A does not see the true score 4e-46 * 3e38 = 1.2e-7
    "weight_underflows_on_upload": ([[4e-46], [0.0]], [0.0, 1e-8], [3e38]),
    # x0 = 0.49 q becomes 0 in the staging cast; the class-0 score 6.9e-16 is invisible to A
    "float64_feature_underflows": ([[1e30, 0.0], [0.0, 1e-16]], [0.0, 0.0], [0.49 * Q, 1.0]),
    # the same cast against weights +W and -W: the two scores err in opposite directions, so the margin carries twice
    # one score's absolute error (exact 6.87e-16 vs 5.13e-16; computed 0 vs 1.2e-15)
    "float64_feature_underflows_two_sided": ([[1e30], [-1e30]], [0.0, 1.2e-15], [0.49 * Q]),
    # normal operands, subnormal products: class 1 (40.47 q) rounds up to 41 q, class 0 (40.49 q) down to 40 q
    "subnormal_products": ([[40.49 * E, 0, 0, 0], [0, 13.51 * E, 13.51 * E, 13.45 * E]], [0.0, 0.0], [2.0**-75] * 4),
    # the bias 2.6 q rounds to 3 q, above class 1's 1.4 q + 1.4 q (computed as 2 q)
    "bias_rounds_in_subnormals": ([[0.0, 0.0], [1.4 * E, 1.4 * E]], [2.6 * Q, 0.0], [2.0**-75] * 2),
    # a subnormal weight 1.3 q rounds to q: 23 % of the score is lost, far above any relative bound
    "subnormal_weight": ([[1.3 * Q], [0.0]], [0.0, 1.15 * 2.0**-29], [2.0**120]),
    # weights at FLT_MIN (+-): rounding stays relative; the planted margin (1e-6) sits inside the guard
    "weight_just_below_flt_min": ([[2.0**-126 * (1 - 1.3 * 2.0**-23)], [0.0]], [0.0, None], [2.0**100]),
    "weight_just_above_flt_min": ([[2.0**-126 * (1 + 1.3 * 2.0**-23)], [0.0]], [0.0, None], [2.0**100]),
}
PLANT_AT = (0, 37, 4_099, 8_191, 10_006)  # among 10 007 rows


def linear_case(name, F, C=4, binary=False, seed=0):
    """Model (C classes or the binary form w1 - w0, b1 - b0) and float64 rows with the construction planted."""
    w, b, x = LINEAR_CONSTRUCTIONS[name]
    w = np.array(w, dtype=np.float64)
    k = w.shape[1]
    b = list(b)
    if b[1] is None:  # just under the class-0 score: a near-tie the guard must catch
        b[1] = float(Fraction(w[0, 0]) * Fraction(x[0]) * (1 - Fraction(1, 10**6)))
    rng = np.random.default_rng(seed + F)
    coef = np.zeros((C, F))
    coef[:2, :k] = w
    coef[:, k:] = rng.standard_normal((C, F - k))
    intercept = np.zeros(C)
    intercept[:2] = b
    X = np.zeros((10_007, F))
    X[:, k:] = rng.integers(-8, 9, size=(10_007, F - k))
    X[list(PLANT_AT)] = 0.0
    X[list(PLANT_AT), :k] = x
    if binary:
        coef, intercept = (coef[1] - coef[0])[None, :], intercept[1:2] - intercept[0:1]
    return coef, intercept, X


def linear_reference(X, coef, intercept):
    """Exact labels: Fractions on the planted rows, float64 on the ordinary rows (asserted unambiguous)."""
    scores = olin.decision_function(X, coef, intercept)
    want = olin.predict_indices(scores).astype(np.int32)
    ordinary = np.setdiff1d(np.arange(X.shape[0]), PLANT_AT)
    assert olin.top2_margin(scores)[ordinary].min() > 1e-6
    exact = olin.exact_predict_indices(X[list(PLANT_AT)], coef, intercept)
    assert np.array_equal(exact, want[list(PLANT_AT)]), "planted row with an ambiguous float64 label"
    return want


def linear_edges_report(F_values=(32, 100, 33, 64, 784)):
    """Every construction x F x entry point; returns the failures (name, F, entry, planted labels got / want)."""
    from sklearn.linear_model import LogisticRegression

    from unionml_b200.engine import Engine
    from unionml_b200.predictors import linear_argmax

    eng = Engine(0)
    failures = []
    for F in F_values:
        for name in LINEAR_CONSTRUCTIONS:
            for binary in (False, True):
                coef, intercept, X = linear_case(name, F, binary=binary)
                want = linear_reference(X, coef, intercept)
                m = eng.load_linear(coef, intercept)
                est = LogisticRegression()
                est.coef_, est.intercept_, est.n_features_in_ = coef, intercept, F
                est.classes_ = np.arange(max(2, coef.shape[0]), dtype=np.float64)
                got = {
                    "predict(stage)": eng.predict(m, eng.stage(X), exact=True)[0],
                    "predict_host(C)": eng.predict_host(m, X, exact=True)[0],
                    "predict_host(F)": eng.predict_host(m, np.asfortranarray(X), exact=True)[0],
                    "linear_argmax(DataFrame)": np.asarray(linear_argmax(est, pd.DataFrame(X))).astype(np.int32),
                }
                for entry, labels in got.items():
                    if not np.array_equal(labels, want):
                        bad = np.flatnonzero(labels != want)
                        failures.append(f"{name}{' (binary)' if binary else ''} F={F} {entry}: rows {bad.tolist()[:6]} "
                                        f"got {labels[bad].tolist()[:6]} want {want[bad].tolist()[:6]}")
    return failures


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_linear_underflow_constructions(mode):
    """UML_B200_RESCORE_MODE is read once per process, so each mode runs in its own interpreter.  F = 32 and 100 take
    the chunked schedule, 33 and 64 whole rows, 784 the separate re-score kernel under programmatic dependent launch
    (in both modes)."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from tests.test_gpu_exactness_edges import linear_edges_report\n"
        "fails = linear_edges_report()\n"
        "print('\\n'.join(fails)); print('failures', len(fails))\n"
    ) % str(ROOT)
    env = dict(os.environ, UML_B200_RESCORE_MODE=mode)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    print(r.stdout)
    assert r.stdout.strip().endswith("failures 0"), r.stdout[-6000:]


# ---------------------------------------------------------------------------------------------------------------
# MLP: planted underflow rows.  Features are tf32 values (the tensor-core kernel takes them, path 5); the same rows
# through the CUDA-core kernel (path 3) with UML_B200_MLP_TC=0.
# ---------------------------------------------------------------------------------------------------------------
def mlp_construction(name, F, H, C, rng):
    """(w1, b1, w2, b2, planted x): the construction on features / hidden units 0..3, classes 0 and 1; the other
    units see only the other features, which are zero in the planted row."""
    w1 = np.zeros((H, F), np.float32)
    w1[4:, 4:] = rng.standard_normal((H - 4, F - 4)) * 0.25
    b1 = np.zeros(H, np.float32)
    b2 = np.zeros(C, np.float32)
    x = np.zeros(F, np.float32)
    w2_scale = 2.0**-10
    w2 = np.zeros((C, H), np.float32)
    if name == "layer2_subnormal_products":  # W1 passes x = 2^-75 through; class 1 rounds up to 41 q, class 0 down to 40 q
        w1[np.arange(4), np.arange(4)] = 1.0
        x[:4] = 2.0**-75
        w2[0, 0] = 40.49 * E
        w2[1, 1:4] = [13.51 * E, 13.51 * E, 13.45 * E]
        w2_scale = E
    elif name == "w1_subnormal_weight":  # 665 q: its tf32 hi and lo are both 0
        w1[0, 0], w1[1, 1] = 665 * Q, 1.0
        x[0], x[1] = 2.0**100, 300 * 2.0**-49
        w2[0, 0], w2[1, 1] = 1.0, 1.0
    elif name == "w1_split_remainder_subnormal":  # w = 2^-115 + 2^-127: hi = 2^-115, lo = 2^-127 is subnormal
        w1[0, 0], w1[1, 1] = 2.0**-115 + 2.0**-127, 2.0**-15 + 2.0**-28
        x[0], x[1] = 2.0**100, 1.0
        w2[0, 0], w2[1, 1] = 1.0, 1.0
    elif name == "product_below_flt_min":  # 2^-60 * 1.5 2^-70 = 1.5 2^-130 in layer 1, magnified by 2^100
        w1[0, 0] = 1.5 * 2.0**-70
        x[0] = 2.0**-60
        w2[0, 0] = 2.0**100
        b2[1] = 1.25 * 2.0**-30
    elif name == "subnormal_feature":  # x0 = 0.75 FLT_MIN is a tf32 value; flushed, class 1 (0.7 2^-26) would win
        w1[0, 0], w1[1, 1] = 2.0**100, 0.7 * 2.0**-26
        x[0], x[1] = 0.75 * 2.0**-126, 1.0
        w2[0, 0], w2[1, 1] = 1.0, 1.0
    elif name == "tiny_b1":
        b1[0] = 3 * Q
        w2[0, 0] = 2.0**100
        b2[1] = 2.5 * 2.0**-49
    elif name == "tiny_b2":
        b2[0], b2[1] = 2 * Q, Q
    else:
        raise KeyError(name)
    w2[:, 4:] = rng.standard_normal((C, H - 4)) * w2_scale
    return w1, b1, w2, b2, x


def exact_mlp_labels(X, w1, b1, w2, b2):
    """The float64 network restated in Fractions (ReLU is exact); first maximum wins."""
    out = []
    for row in X:
        xs = [(f, Fraction(float(v))) for f, v in enumerate(row) if v != 0]
        h = []
        for n in range(w1.shape[0]):
            s = Fraction(float(b1[n])) + sum((v * Fraction(float(w1[n, f])) for f, v in xs), Fraction(0))
            h.append(max(s, Fraction(0)))
        z = [Fraction(float(b2[c])) + sum((h[n] * Fraction(float(w2[c, n])) for n in range(len(h)) if h[n]), Fraction(0))
             for c in range(w2.shape[0])]
        out.append(max(range(len(z)), key=lambda c: (z[c], -c)))
    return np.array(out, dtype=np.int32)


MLP_CONSTRUCTIONS = ["layer2_subnormal_products", "w1_subnormal_weight", "w1_split_remainder_subnormal",
                     "product_below_flt_min", "subnormal_feature", "tiny_b1", "tiny_b2"]
MLP_TC_SHAPES = [(64, 32, 10), (32, 16, 2), (128, 16, 3)]


@pytest.mark.parametrize("kernel", ["tensor_core", "cuda_core"])
@pytest.mark.parametrize("shape", MLP_TC_SHAPES)
@pytest.mark.parametrize("name", MLP_CONSTRUCTIONS)
def test_mlp_underflow_constructions(engine, monkeypatch, name, shape, kernel):
    F, H, C = shape
    rng = np.random.default_rng(F + H + C)
    w1, b1, w2, b2, x = mlp_construction(name, F, H, C, rng)
    assert not (x.view(np.uint32) & np.uint32(0x1FFF)).any()  # tf32 values: the tensor-core kernel scores them itself
    X = np.zeros((10_007, F), np.float32)
    X[:, 4:] = rng.integers(0, 9, size=(10_007, F - 4))
    X[list(PLANT_AT)] = x
    want = omlp.predict_indices_f64(X, w1, b1, w2, b2).astype(np.int32)
    exact = exact_mlp_labels(X[list(PLANT_AT)], w1, b1, w2, b2)
    assert np.array_equal(exact, want[list(PLANT_AT)]), "planted row with an ambiguous float64 label"
    ordinary = np.setdiff1d(np.arange(X.shape[0]), PLANT_AT)
    assert omlp.logit_margin_f64(X[ordinary], w1, b1, w2, b2).min() > 0
    monkeypatch.setenv("UML_B200_MLP_TC", "1" if kernel == "tensor_core" else "0")
    m = engine.load_mlp(w1, b1, w2, b2)
    got, st = engine.predict_mlp(m, engine.stage(X), exact=True)
    assert st["path"] == (5 if kernel == "tensor_core" else 3), st
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"rows {bad.tolist()[:8]}: got {got[bad].tolist()[:8]} want {want[bad].tolist()[:8]}"


# ---------------------------------------------------------------------------------------------------------------
# near-tie sweep: w_c = w_0 (1 + eps r_c), margins eps-scaled over 0.01x .. 100x the kernel's bound
# ---------------------------------------------------------------------------------------------------------------
EPS_FACTORS = (0.01, 0.1, 1.0, 10.0, 100.0)
# the MLP bounds sit far above the errors the kernels make (the tensor-core one budgets 32u per MMA step, the hardware
# loses about 3u, tests/test_gpu_wgmma_accum.py), so plain fp32 is wrong only well inside them: reach down to 1e-4x
MLP_EPS_FACTORS = (1e-4, 1e-3) + EPS_FACTORS


def spread(rng, shape, lo=-20, hi=20, tf32=False):
    """Values with random signs, mantissas and exponents in [lo, hi]; tf32 values (low 13 bits zero) on request."""
    v = (rng.uniform(1.0, 2.0, size=shape) * rng.choice([-1.0, 1.0], size=shape) *
         np.exp2(rng.integers(lo, hi + 1, size=shape))).astype(np.float32)
    if tf32:
        v = (v.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return v


def top2(z):
    part = np.partition(z, z.shape[1] - 2, axis=1)
    return part[:, -1] - part[:, -2]


def exact_linear_labels(X, coef, intercept):
    """float64 labels where the float64 margin is far outside float64's own error, Fractions elsewhere."""
    s = olin.decision_function(X, coef, intercept)
    want = olin.predict_indices(s).astype(np.int32)
    a64 = np.abs(intercept).max() + np.abs(X) @ np.abs(coef).max(axis=0)
    unsure = np.flatnonzero(top2(s) <= 4 * (X.shape[1] + 2) * 2.0**-53 * a64)
    if unsure.size:
        want[unsure] = olin.exact_predict_indices(X[unsure], coef, intercept)
    exact_margin = top2(s)  # within float64 error of the exact margin (far below the fp32 bounds compared with it)
    return want, exact_margin, unsure.size


@pytest.mark.parametrize("C", [2, 10, 16])
@pytest.mark.parametrize("F", [1, 32, 33, 64, 65, 784])
def test_linear_near_tie_sweep(engine, F, C):
    rng = np.random.default_rng(100 * F + C)
    N = 8_000 if F == 784 else 20_000
    X = spread(rng, (N, F)).astype(np.float64)
    w0, b0 = spread(rng, F).astype(np.float64), float(spread(rng, 1)[0])
    r, rb = rng.standard_normal((C - 1, F)), rng.standard_normal(C - 1)
    thr = linear_thr(F)
    # eps = 1 gives margins D; scale eps so that eps * D spans 0.01x .. 100x the guard's margin threshold thr * A
    d1 = X @ np.vstack([np.zeros(F), w0 * r]).T + np.concatenate([[0.0], b0 * rb])
    base = np.median(thr * (abs(b0) + np.abs(X) @ np.abs(w0)) / np.maximum(top2(d1), 1e-300))
    n_fast_wrong = n_flagged = n_within = 0
    for k in EPS_FACTORS:
        eps = k * base
        coef = np.vstack([w0, w0 * (1 + eps * r)])
        intercept = np.concatenate([[b0], b0 * (1 + eps * rb)])
        want, margin, _ = exact_linear_labels(X, coef, intercept)
        m = engine.load_linear(coef, intercept)
        b = engine.stage(X)
        got, st = engine.predict(m, b, exact=True)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"eps {k}x: EXACT wrong on rows {bad.tolist()[:8]} (flagged {st['n_flagged']})"
        fast, _ = engine.predict(m, b, exact=False)
        c32, b32 = coef.astype(np.float32).astype(np.float64), intercept.astype(np.float32).astype(np.float64)
        A = np.abs(b32).max() + np.abs(X) @ np.abs(c32).max(axis=0)
        n_fast_wrong += int((fast != want).sum())
        n_flagged += st["n_flagged"]
        within = int((margin <= 2.02 * thr * A).sum())
        n_within += within
        # a flagged row has |exact margin| <= thr A + 2 err <= 2 thr A: a guard flagging more is vacuous (or thr too big)
        assert st["n_flagged"] <= within, (k, st["n_flagged"], within)
    print(f"\nlinear F={F} C={C}: FAST wrong {n_fast_wrong}, EXACT wrong 0, flagged {n_flagged} <= {n_within} rows "
          f"within 2.02 thr A, of {N * len(EPS_FACTORS)}")
    assert n_fast_wrong >= 20  # the data has teeth: plain fp32 gets many of these rows wrong


@pytest.mark.parametrize("kernel", ["tensor_core", "cuda_core"])
@pytest.mark.parametrize("shape", MLP_TC_SHAPES)
def test_mlp_near_tie_sweep(engine, monkeypatch, shape, kernel):
    F, H, C = shape
    rng = np.random.default_rng(F * 7 + H * 3 + C)
    N = 20_000
    X = spread(rng, (N, F), -10, 10, tf32=True)
    w1, b1 = spread(rng, (H, F), -10, 10), spread(rng, H, -10, 10)
    w20, b20 = spread(rng, H, -10, 10).astype(np.float64), float(spread(rng, 1, -10, 10)[0])
    r, rb = rng.standard_normal((C - 1, H)), rng.standard_normal(C - 1)
    u = U
    n_mma = ((F + 31) // 32 * 32) / 8
    e1_factor = ((32 * n_mma + 12) if kernel == "tensor_core" else (F + 4)) * u * (1 + F * 2.0**-21) * 1.0001
    e2 = float(np.float32((H + 4) * u * 1.0001))
    x64 = X.astype(np.float64)
    h = np.maximum(x64 @ w1.astype(np.float64).T + b1, 0)
    A1 = np.abs(b1).max() + np.abs(x64) @ np.abs(w1.astype(np.float64)).max(axis=0)
    d1 = h @ np.vstack([np.zeros(H), w20 * r]).T + np.concatenate([[0.0], b20 * rb])
    monkeypatch.setenv("UML_B200_MLP_TC", "1" if kernel == "tensor_core" else "0")
    b = engine.stage(X)
    n_fast_wrong = n_flagged = n_within = 0
    base = None
    for k in MLP_EPS_FACTORS:
        eps = 1.0 if base is None else k * base
        w2 = np.vstack([w20, w20 * (1 + eps * r)]).astype(np.float32)
        b2 = np.concatenate([[b20], b20 * (1 + eps * rb)]).astype(np.float32)
        rowsum = np.abs(w2.astype(np.float64)).sum(axis=1).max()
        A2 = np.abs(b2).max() + h @ np.abs(w2.astype(np.float64)).max(axis=0)
        err = float(np.float32(e1_factor * rowsum)) * A1 + e2 * A2
        if base is None:  # eps from the bound at this scale: eps * D spans 0.01x .. 100x of 2 err
            base = np.median(2 * err / np.maximum(top2(d1), 1e-300))
            eps = k * base
            w2 = np.vstack([w20, w20 * (1 + eps * r)]).astype(np.float32)
            b2 = np.concatenate([[b20], b20 * (1 + eps * rb)]).astype(np.float32)
        z = omlp.logits(X, w1, b1, w2, b2)
        want = z.argmax(axis=1).astype(np.int32)
        zbound = (F + H + 4) * 2.0**-53 * (A1 * np.abs(w2.astype(np.float64)).sum(axis=1).max() + A2)
        unsure = np.flatnonzero(top2(z) <= 4 * zbound)
        if unsure.size:
            want[unsure] = exact_mlp_labels(X[unsure], w1, b1, w2, b2)
        m = engine.load_mlp(w1, b1, w2, b2)
        got, st = engine.predict_mlp(m, b, exact=True)
        assert st["path"] == (5 if kernel == "tensor_core" else 3), st
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"eps {k}x: EXACT wrong on rows {bad.tolist()[:8]} (flagged {st['n_flagged']})"
        fast, _ = engine.predict_mlp(m, b, exact=False)
        n_fast_wrong += int((fast != want).sum())
        n_flagged += st["n_flagged"]
        within = int((top2(z) <= 2.02 * err).sum())
        n_within += within
        assert st["n_flagged"] <= within, (k, st["n_flagged"], within)
    print(f"\nmlp {kernel} {F}->{H}->{C}: FAST wrong {n_fast_wrong}, EXACT wrong 0, flagged {n_flagged} <= {n_within} "
          f"rows within 2.02 err, of {N * len(MLP_EPS_FACTORS)}")
    assert n_fast_wrong >= 20
