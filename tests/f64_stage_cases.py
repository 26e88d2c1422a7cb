"""Constructions for the float64 re-score stage tests (tests/test_gpu_f64_stage_edges.py), importable without a GPU.

The stage's contract: a row's label is the argmax of its exact scores (numpy's first-maximum rule), or the row is
counted in ``n_ambiguous``.  Rows are planted at exact margins measured against the stage's own bound beta (twice the
per-score error bound of ``score_row_f64`` in linear_tile.cuh, or of ``mlp_rs_rows`` in mlp_rescore.cuh), and split
into batches by that margin: certain (>= 4 beta), inside (<= beta / 4, exact ties included) and straddle (between).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

U = 2.0**-53
Q64 = 2.0**-1074  # float64 subnormal spacing


# ---------------------------------------------------------------------------------------------------------------
# bounds, restated from the kernels
# ---------------------------------------------------------------------------------------------------------------
def linear_beta(X, coef, intercept, bmag=None, fold_rel=0.0):
    """beta = 2 err of score_row_f64 per row: err = (n u + fold_rel) a + n 2^-1074, n = F/32 + 8,
    a = max_c (sum_f |x_f w_cf| + bmag_c).  coef / intercept are the caller's (one row for a binary model)."""
    coef = np.atleast_2d(np.asarray(coef, np.float64))
    intercept = np.atleast_1d(np.asarray(intercept, np.float64))
    bmag = np.abs(intercept) if bmag is None else np.asarray(bmag, np.float64)
    X = np.asarray(X, np.float64)
    n = X.shape[1] / 32.0 + 8.0
    a = (np.abs(X) @ np.abs(coef).T + bmag).max(axis=1)
    if coef.shape[0] == 1:  # expanded binary layout [0, s]: class 0 contributes 0
        a = np.maximum(a, 0.0)
    return 2.0 * ((n * U + fold_rel) * a + n * Q64)


def mlp_beta(X, w1, b1, w2, b2):
    """beta = 2 err of mlp_rs_rows: herr = (F + 6) u a1, err = herr w2sum + (H + 16) u (a2 + herr w2sum + b2max)."""
    x = np.asarray(X, np.float32).astype(np.float64)
    w1, b1, w2, b2 = (np.asarray(a, np.float32).astype(np.float64) for a in (w1, b1, w2, b2))
    F, H = x.shape[1], w1.shape[0]
    a1 = np.abs(x) @ np.abs(w1).max(axis=0) + np.abs(b1).max()
    herr = (F + 6.0) * U * a1
    h = np.maximum(x @ w1.T + b1, 0.0)
    w2m = np.abs(w2).max(axis=0)
    w2sum = w2m.sum()
    amax = h @ w2m + herr * w2sum + np.abs(b2).max()
    return 2.0 * (herr * w2sum + (H + 16.0) * U * amax)


# ---------------------------------------------------------------------------------------------------------------
# exact arithmetic
# ---------------------------------------------------------------------------------------------------------------
# Every float64 is an integer multiple of 2^-1074, so a product of two is one of 2^-2148: scores are summed exactly as
# Python integers in units of 2^-2148 (much faster than Fractions), and ints divide with correct rounding.
SHIFT = 1074
ONE2 = 1 << (2 * SHIFT)  # 1.0 in units of 2^-2148


def fixed(v):
    """float64 v as an integer in units of 2^-1074 (exact)."""
    n, d = float(v).as_integer_ratio()
    return n << (SHIFT - (d.bit_length() - 1))


def _fixed_rows(a):
    return [[fixed(v) for v in row] for row in np.atleast_2d(np.asarray(a, np.float64))]


def _int_scores(xs, wq, bq):
    """Exact scores in units of 2^-2148: xs = [(feature, fixed x)] of the nonzero features, wq / bq fixed weights."""
    return [(bq[c] << SHIFT) + sum(v * wq[c][f] for f, v in xs) for c in range(len(wq))]


def exact_linear_scores(x, coef, intercept):
    """Exact scores of one float64 row; a binary model gives [0, s] (sklearn: class 1 iff s > 0)."""
    wq, bq = _fixed_rows(coef), [fixed(v) for v in np.atleast_1d(intercept)]
    xs = [(f, fixed(v)) for f, v in enumerate(np.asarray(x, np.float64)) if v != 0]
    s = [Fraction(v, ONE2) for v in _int_scores(xs, wq, bq)]
    return [Fraction(0)] + s if len(s) == 1 else s


def label_margin(scores):
    """(first-maximum argmax, top-2 margin) of exact scores."""
    best = max(range(len(scores)), key=lambda c: (scores[c], -c))
    second = max(s for c, s in enumerate(scores) if c != best)
    return best, scores[best] - second


def exact_linear(X, coef, intercept):
    """Exact labels and top-2 margins (as float64) of float64 rows."""
    wq, bq = _fixed_rows(coef), [fixed(v) for v in np.atleast_1d(intercept)]
    labels, margins = [], []
    for x in np.asarray(X, np.float64):
        s = _int_scores([(f, fixed(v)) for f, v in enumerate(x) if v != 0], wq, bq)
        if len(s) == 1:
            s = [0] + s
        lab, m = label_margin(s)
        labels.append(lab)
        margins.append(m / ONE2)
    return np.array(labels, np.int32), np.array(margins)


def _exact_mlp_logits(row, w1, b1, w2, b2):
    """Exact logits of one fp32 row, in Fractions (ReLU is exact); zero features and zero weights are skipped."""
    xs = [(f, Fraction(float(v))) for f, v in enumerate(row) if v != 0]
    h = [max(Fraction(float(b1[n])) + sum((v * Fraction(float(w1[n, f])) for f, v in xs if w1[n, f]), Fraction(0)),
             Fraction(0)) for n in range(w1.shape[0])]
    return [Fraction(float(b2[c])) + sum((h[n] * Fraction(float(w2[c, n])) for n in range(len(h)) if h[n]), Fraction(0))
            for c in range(w2.shape[0])]


def exact_mlp(X, w1, b1, w2, b2):
    """The float64 network on fp32 x and weights, in Fractions (ReLU is exact)."""
    w1, b1, w2, b2 = (np.asarray(a, np.float32) for a in (w1, b1, w2, b2))
    labels, margins = [], []
    for row in np.asarray(X, np.float32):
        lab, m = label_margin(_exact_mlp_logits(row, w1, b1, w2, b2))
        labels.append(lab)
        margins.append(float(m))
    return np.array(labels, np.int32), np.array(margins)


def topk_gap(z, k):
    """(stable descending top k, smallest consecutive gap among ranks 1 .. min(k, C - 1) + 1) of one row's logits: ties
    go to the lower class index, as np.argsort(-z, kind="stable") orders them."""
    order = sorted(range(len(z)), key=lambda c: (-z[c], c))
    kk = min(k, len(z) - 1)
    return order[:k], min(z[order[r]] - z[order[r + 1]] for r in range(kk))


def mlp_f64_bound(X, w1, b1, w2, b2):
    """Per row, a bound on the error of any float64 evaluation of any one logit (any summation order): a dot product of
    n terms errs by at most (n + 1) u times its absolute sum; each hidden unit's error is carried through |W2| (ReLU is
    1-Lipschitz).  Per unit and class rather than through the largest weights, so that a huge weight on a unit a row
    leaves at zero does not send every row to Fractions."""
    x = np.asarray(X, np.float32).astype(np.float64)
    w1, b1, w2, b2 = (np.asarray(a, np.float32).astype(np.float64) for a in (w1, b1, w2, b2))
    F, H = x.shape[1], w1.shape[0]
    e1 = (F + 4) * U * (np.abs(x) @ np.abs(w1).T + np.abs(b1))  # (n, H)
    carried = e1 @ np.abs(w2).T  # (n, C)
    h = np.maximum(x @ w1.T + b1, 0.0)
    a2 = h @ np.abs(w2).T + np.abs(b2) + carried
    return (carried + (H + 4) * U * a2).max(axis=1) * (1 + 2.0**-20)


def exact_mlp_topk(X, w1, b1, w2, b2, k):
    """Exact top-k of the float64 network on fp32 x and weights: (indices (n, k) int32, gaps (n,) float64), the gap
    being the smallest exact consecutive gap among ranks 1 .. min(k, C - 1) + 1.  Rows whose float64 gaps all sit
    beyond four times float64's own error bound keep the float64 order (their gap is the float64 one, within that
    bound of the exact gap); the others, exact ties included, are recomputed in Fractions."""
    X = np.asarray(X, np.float32)
    w1, b1, w2, b2 = (np.asarray(a, np.float32) for a in (w1, b1, w2, b2))
    C = w2.shape[0]
    kk = min(k, C - 1)
    x = X.astype(np.float64)
    z = np.maximum(x @ w1.T.astype(np.float64) + b1, 0.0) @ w2.T.astype(np.float64) + b2
    order = np.argsort(-z, axis=1, kind="stable")
    zs = np.take_along_axis(z, order, axis=1)
    gap = (zs[:, :kk] - zs[:, 1 : kk + 1]).min(axis=1)
    idx = order[:, :k].astype(np.int32)
    for i in np.flatnonzero(~(gap > 4 * mlp_f64_bound(X, w1, b1, w2, b2))):
        top, g = topk_gap(_exact_mlp_logits(X[i], w1, b1, w2, b2), k)
        idx[i], gap[i] = top, float(g)
    return idx, gap


def tf32(v):
    """fp32 values with the low 13 mantissa bits cleared (tf32 values: the tensor-core kernel scores them itself)."""
    return (np.asarray(v, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


RANK_LADDER = (0.6, 0.75, 0.9, 1.3, 1.6, 3.0)  # float64 is exact on these rows: below beta counted, above certified
RANK_TIE_LADDER = (0.0, 0.1, 0.5, 3.0, 10.0)


def mlp_rank_case(F, H, C, r, tie=False, big=False, seed=0):
    """A network and rows whose logits are D = 64 c0 apart but for one planted pair at ranks r, r + 1 (1-based), set
    on the ladder of beta (mlp_beta).  Hidden unit 0 = x0 - x1 + x2 with x0 = x1 = 2^20 (big: 2^50, integer rows); it
    cancels, so herr w2sum dominates beta while float64 is exact.  Class a gets logit h0 = x2, class b the bias c0 =
    16 beta (rounded to a power of 2); the classes above the pair c0 + j D, those below c0 - j D.  x2 = c0 +- f beta,
    so a sits above b (+) or below it (-).  tie: class t copies a (weights and bias), so a and t tie exactly on every
    row and the group a, t, b takes ranks r .. r + 2.  Returns (w1, b1, w2, b2), X (fp32, tf32 values), the factors f
    (signed), beta and (a, b, t)."""
    rng = np.random.default_rng(seed)
    n_pair = 3 if tie else 2
    assert r + n_pair - 1 <= C and F >= 3 and H >= 1
    perm = rng.permutation(C)
    above, group, below = perm[: r - 1], perm[r - 1 : r - 1 + n_pair], perm[r - 1 + n_pair :]
    a, b = int(group[0]), int(group[-1])
    t = int(group[1]) if tie else -1
    w1 = np.zeros((H, F), np.float32)
    w1[0, :3] = [1.0, -1.0, 1.0]
    b1 = np.zeros(H, np.float32)
    w2 = np.zeros((C, H), np.float32)
    w2[a, 0] = 1.0
    if tie:
        w2[t, 0] = 1.0
    x0 = np.zeros(F, np.float32)
    x0[:2] = 2.0**50 if big else 2.0**20
    b2 = np.zeros(C, np.float32)
    beta = float(mlp_beta(x0[None, :], w1, b1, w2, b2)[0])
    c0 = 2.0 ** np.ceil(np.log2(16 * beta))
    D = 64 * c0
    b2[b] = c0
    for j, c in enumerate(above[::-1], 1):
        b2[c] = c0 + j * D
    for j, c in enumerate(below, 1):
        b2[c] = c0 - j * D
    rows, fs = [], []
    for f in RANK_TIE_LADDER if tie else RANK_LADDER:
        for sign in (1, -1) if f else (1,):
            x = x0.copy()
            v = c0 + sign * f * beta
            x[2] = tf32(np.rint(v) if big else v)
            rows.append(x)
            fs.append(sign * f)
    return (w1, b1, w2, b2), np.array(rows, np.float32), np.array(fs), beta, (a, b, t)


def rungs(margin, beta):
    """Row indices of the certain, inside and straddle batches."""
    certain = np.flatnonzero(margin >= 4 * beta)
    inside = np.flatnonzero(margin <= beta / 4)
    straddle = np.setdiff1d(np.arange(margin.size), np.concatenate([certain, inside]))
    return certain, inside, straddle


# ---------------------------------------------------------------------------------------------------------------
# linear: heavy-cancellation ladder.  Every class c owns one tuning feature t_c (weight 1, 0 for the other classes; a
# duplicate class shares its twin's column and bias, so the pair ties exactly); the body features are spread over
# 2^+-20 with both signs.  A row sets x_t = (target score) - (body score of that class), so each score is the
# cancellation of large terms of both signs, and the top pair sits at a chosen margin.
# ---------------------------------------------------------------------------------------------------------------
def spread64(rng, shape, lo=-20, hi=20):
    return rng.uniform(1.0, 2.0, size=shape) * rng.choice([-1.0, 1.0], size=shape) * np.exp2(rng.integers(lo, hi + 1, size=shape))


def ladder_model(F, C, rng, dups=(), binary=False, wexp=(-20, 20), anchor=None):
    """coef (C x F, or 1 x F for binary), intercept, tuning column of each class.  dups: (a, b) pairs, b copies a;
    wexp: exponent range of the body weights.  anchor: a weight given to feature 0 in every class (see ladder_rows)."""
    if binary:
        assert F >= 1
        coef = np.zeros((1, F))
        coef[0, :F - 1] = spread64(rng, F - 1, *wexp)
        coef[0, F - 1] = 1.0
        return coef, spread64(rng, 1), np.array([-1, F - 1])
    twin = {b: a for a, b in dups}
    own = [c for c in range(C) if c not in twin]
    assert F >= len(own) + 1, (F, C)
    coef = np.zeros((C, F))
    body = F - len(own)
    coef[:, :body] = spread64(rng, (C, body), *wexp)
    if anchor is not None:
        coef[:, 0] = anchor
    intercept = spread64(rng, C)
    tune = np.zeros(C, np.int64)
    for k, c in enumerate(own):
        tune[c] = body + k
        coef[c, body + k] = 1.0
    for b, a in twin.items():
        coef[b], intercept[b], tune[b] = coef[a], intercept[a], tune[a]
    return coef, intercept, tune


def ladder_rows(rng, coef, intercept, tune, tops, taus, kind="f64", anchor_x=None):
    """One row per (top pair (a, b), tau): exact score of a ~ S, of b ~ S - tau (so a wins), the others ~ 2^30 below.
    kind: the body features as float64 spread over 2^+-20, or int32 / int64 integers (int64 beyond 2^53); the truth is
    always taken on float64(x).  Returns the rows in the source dtype.

    S = 0, or with anchor_x the anchor term x_0 w_0 that feature 0 adds to every class alike (ladder_model's anchor).
    An integer tuning feature sets a margin only to within 0.5; the anchor makes every score, and so the bound beta,
    large enough (int32: 2^30 x 2^30) that 0.5 is far below beta / 4, without moving any margin."""
    binary = coef.shape[0] == 1
    F = coef.shape[1]
    body = F - (1 if binary else len(set(tune.tolist())))
    wq = [row[:body] for row in _fixed_rows(coef)]
    bq = [fixed(v) for v in np.atleast_1d(intercept)]
    rows = []
    for (a, b), tau in zip(tops, taus):
        if kind == "f64":
            xb = spread64(rng, body)
        elif kind == "i32":
            xb = rng.integers(-2**30, 2**30, size=body).astype(np.float64)
        else:
            xb = rng.integers(-2**58, 2**58, size=body).astype(np.float64)
        x = np.zeros(F)
        x[:body] = xb
        if anchor_x is not None:
            x[0] = xb[0] = anchor_x
            xb = xb.copy()
            xb[0] = 0.0  # common to every class: left out of B, so the tuning values stay small
        xq = [(f, fixed(v)) for f, v in enumerate(xb) if v != 0]
        if binary:  # s = B + x_t; target s = tau if a == 1 else -tau
            B = _int_scores(xq, wq, bq)[0]
            target = fixed(tau) << SHIFT
            x[F - 1] = ((target if a == 1 else -target) - B) / ONE2
        else:
            Bs = _int_scores(xq, wq, bq)
            for c in range(coef.shape[0]):
                if c != a and tune[c] == tune[a]:
                    continue  # a's twin follows a
                target = 0 if c == a else (-(fixed(tau) << SHIFT) if c == b else -(1 << 30) * ONE2)
                x[tune[c]] = (target - Bs[c]) / ONE2  # int / int: correctly rounded
        rows.append(x)
    X = np.array(rows)
    if kind == "i32":
        return np.rint(X).clip(-2**31, 2**31 - 1).astype(np.int32)
    if kind == "i64":
        # +1 on values >= 2^55 (spacing >= 8): an int64 that float64 rounds back to the value the truth is taken on
        return np.array([[int(v) + (1 if abs(v) >= 2.0**55 else 0) for v in r] for r in X], dtype=np.int64)
    return X


# ---------------------------------------------------------------------------------------------------------------
# hole 1: float64 products below DBL_MIN (x 2^-537 against weights 0.6 / 1.4 2^-537)
# ---------------------------------------------------------------------------------------------------------------
UF_X = 2.0**-537


def underflow_case(binary=False):
    """Exact: class 1 (1.4 q) beats class 0 (0.6 q + 0.6 q = 1.2 q), q = 2^-1074.  Lanes round each product to q,
    so float64 gives 2 q vs q.  Binary: s = -0.6 q - 0.6 q + 1.4 q = 0.2 q > 0, computed -q."""
    x = np.array([UF_X, UF_X, UF_X])
    if binary:
        return np.array([[-0.6 * UF_X, -0.6 * UF_X, 1.4 * UF_X]]), np.zeros(1), x
    return np.array([[0.6 * UF_X, 0.6 * UF_X, 0.0], [0.0, 0.0, 1.4 * UF_X]]), np.zeros(2), x


# ---------------------------------------------------------------------------------------------------------------
# hole 3: Pipeline(StandardScaler, LR) with mean_ >> scale_, the mean chosen so that every step of a plain sequential
# fold b' = b - sum_f mean_f w'_f rounds the same way
# ---------------------------------------------------------------------------------------------------------------
def sequential_fold(mean, wsc, b):
    """The old host fold of one class, in float64 scalar operations: acc -= mean_f * w'_f in feature order."""
    acc = float(b)
    for m, w in zip(mean.tolist(), wsc.tolist()):
        acc = acc - m * w
    return acc


def greedy_mean(rng, F, w, scale, centre=1e6):
    """mean_f near `centre` such that every step of the sequential fold rounds its running sum up."""
    wsc = w * (1.0 / scale)
    mean = np.empty(F)
    acc = 0.0
    for f in range(F):
        best = None
        for _ in range(64):
            m = centre * (1 + rng.uniform(-1e-3, 1e-3))
            p = m * wsc[f]
            new = acc - p
            err = Fraction(new) - (Fraction(acc) - Fraction(p))  # the step's rounding of the sum
            if best is None or err > best[0]:
                best = (err, m, new)
        mean[f], acc = best[1], best[2]
    return mean


def fold_model(F=784, seed=5):
    """(scaler mean_, scale_, coef (2 x F), intercept): class 0 carries every fold term, class 1 none."""
    rng = np.random.default_rng(seed)
    scale = 1e-2 * (1 + rng.uniform(0, 0.5, F))
    w0 = rng.uniform(0.5, 1.0, F)
    mean = greedy_mean(rng, F, w0, scale)
    coef = np.vstack([w0, np.zeros(F)])
    intercept = np.array([0.0, 0.0])
    return mean, scale, coef, intercept


def fold_rows(rng, mean, scale, coef, intercept, taus):
    """Rows x = mean + scale z whose exact margin (class 0 - class 1) on scikit-learn's z is ~ tau."""
    from sklearn.preprocessing import StandardScaler

    sc = StandardScaler().fit(np.vstack([mean - scale, mean + scale]))
    sc.mean_, sc.scale_, sc.var_ = mean.copy(), scale.copy(), scale**2
    F = mean.size
    rows = []
    for tau in taus:
        z = rng.uniform(-2, 2, F)
        x = mean + scale * z
        zs = sc.transform(x[None, :])[0]
        s = Fraction(float(intercept[0] - intercept[1])) + sum(Fraction(float(a)) * Fraction(float(b)) for a, b in zip(zs[1:], coef[0, 1:] - coef[1, 1:]))
        z0 = (Fraction(tau) - s) / Fraction(float(coef[0, 0] - coef[1, 0]))
        x[0] = float(Fraction(float(mean[0])) + Fraction(float(scale[0])) * z0)
        rows.append(x)
    return sc, np.array(rows)


def fold_truth(sc, X, coef, intercept):
    """Exact labels / margins on scikit-learn's own transform(X)."""
    return exact_linear(sc.transform(X), coef, intercept)


def fold_beta(sc, X, coef, intercept):
    """beta of the folded model: w' = w / scale_, bmag_c = |b_c| + sum_f |mean_f w'_cf|, fold_rel = 8 u."""
    inv = 1.0 / sc.scale_
    wsc = coef * inv
    bmag = np.abs(intercept) + np.abs(sc.mean_ * wsc).sum(axis=1)
    return linear_beta(X, wsc, intercept, bmag=bmag, fold_rel=8 * U)
