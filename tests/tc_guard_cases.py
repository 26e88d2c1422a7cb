"""A CPU model of the linear tile kernel's tensor-core guard (tier 1, DESIGN.md 3.2) and the row constructions of
tests/test_gpu_linear_tc_guard.py, importable without a GPU.

Tier 1 certifies a row iff m_tc > kappa a, where m_tc is the top-2 margin of the wgmma scores (W scaled by 2^sigma, as
fp16 hi and lo pieces) and a the bound column plus 2^sigma bias[C].  The operands are restated here from DESIGN.md 3.2
and the comments of build_tc_operands / upload_model, not imported from the engine.  A row's verdict comes from its
exact scaled margin m and its exact A_hat = sum_f x_f wb_f + tb[C]:
  must-certify  m >= kappa A_hat (1 + step)(1 + 4u) + 2 e_rel A_hat
  must-leave    m <= kappa A_hat (1 - step)(1 - 4u) - 2 e_rel A_hat
  either        otherwise.
The tensor-core score of a class errs by at most e_rel A_hat, the computed a by at most step (its wgmma column) and u
(the bias add) of A_hat, and kappa a and the margin's subtraction round once each: 4u covers those three roundings.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from tests.f64_stage_cases import exact_linear

U = 2.0**-24
FLT_MIN = 2.0**-126
SUB = 2.0**-150  # largest error of an fp32 rounding into the subnormals
STEP_BUDGET = 64.0  # u per k16 step of the f16 wgmma accumulation
U53 = 2.0**-53


# ---------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------
def f16_round(v, up=False):
    """The fp16 value nearest to each v (ties to even), or with up the smallest fp16 value >= v; |v| < 65520."""
    v = np.asarray(v, np.float64)
    h = v.astype(np.float16)
    if up:
        below = h.astype(np.float64) < v
        h = np.where(below, np.nextafter(h, np.float16(np.inf)), h)
    return h.astype(np.float64)


def margin_thr(F):
    """linear_margin_thr: the fp32 route certifies a row iff margin > thr A32."""
    return float(np.float32(2.0 * (F + 4.0) * U * (1.0 + F * 2.0**-21) * 1.0001))


def guard_terms(F):
    """(step, e_rel, kappa as float64 before its float32 rounding) of DESIGN.md 3.2 at F features."""
    f_pad = (F + 31) // 32 * 32
    step = STEP_BUDGET * U * (f_pad // 16)
    e_rel = (2.0**-21 + step * (1 + 2.0**-10) + 4 * U) * (1 + 2.0**-10)
    thr = margin_thr(F)
    return step, e_rel, (2 * e_rel + 2.5 * thr * (1 + (F + 2) * U)) / (1 - step) * (1 + 2.0**-10)


@dataclass
class TcOperands:
    C: int
    F: int
    f_pad: int
    sigma: int
    W: np.ndarray  # (C, F) float64, the expanded layout [0, w] of a binary model
    b: np.ndarray  # (C,)
    wt_bound: np.ndarray  # (F,) the fp32 route's wt[:, C] (float32 values)
    bias_bound: float  # the fp32 route's bias[C] (a float32 value)
    hi: np.ndarray  # (C, F) fp16 values of the scaled weights
    lo: np.ndarray
    wb: np.ndarray  # (F,) the bound column
    tb: np.ndarray  # (C + 1,) scaled biases, tb[C] the bound column's
    thr: float
    step: float
    e_rel: float
    kappa: float  # the float32 value the kernel compares with
    eligible: bool  # build_tc_operands' load-time checks


def operands(coef, intercept):
    """The tensor-core operands of a model from the caller's float64 coef (C x F, or 1 x F binary) and intercept."""
    coef = np.atleast_2d(np.asarray(coef, np.float64))
    intercept = np.atleast_1d(np.asarray(intercept, np.float64))
    if coef.shape[0] == 1:
        coef = np.vstack([np.zeros_like(coef), coef])
        intercept = np.concatenate([[0.0], intercept])
    C, F = coef.shape
    f_pad = (F + 31) // 32 * 32
    w32 = coef.astype(np.float32)
    wt_bound = np.maximum(np.abs(w32).max(axis=0), np.float32(FLT_MIN)).astype(np.float64)
    b32 = intercept.astype(np.float32)
    bmax = float(max(np.abs(b32).max(), np.abs(intercept).astype(np.float32).max()))
    wsum = 0.0
    for v in wt_bound:
        wsum += float(v)
    abs_err = (F + 2.0 + wsum) * SUB
    thr = margin_thr(F)
    bias_bound = float(np.float32(bmax + (FLT_MIN + 2.0 * abs_err) / thr * (1.0 + 1.0 / 1024)))
    wabs = float(np.abs(coef).max())
    ex = int(np.frexp(wabs)[1]) if wabs > 0 else 0
    sigma = 15 - ex
    v = np.ldexp(coef, sigma)
    hi = f16_round(v)
    lo = f16_round(v - hi)
    wmax = np.maximum(np.ldexp(wt_bound, sigma), np.abs(v).max(axis=0))
    wb = f16_round(np.maximum(wmax, 0.125), up=True)
    tb = np.zeros(C + 1)
    tb[:C] = np.ldexp(intercept, sigma).astype(np.float32)
    tb[C] = float(np.float32(np.ldexp(bias_bound, sigma)))
    a32 = bias_bound + 65504.0 * wsum
    eligible = (f_pad <= 64 and np.isfinite(coef).all() and np.isfinite(intercept).all()
                and np.ldexp(a32, max(sigma, 0)) < 2.0**100 and np.ldexp(bias_bound, sigma) > 2.0**-100
                and bool(np.all(wb <= 65504.0)))
    step, e_rel, kappa64 = guard_terms(F)
    return TcOperands(C, F, f_pad, sigma, coef, intercept, wt_bound, bias_bound, hi, lo, wb, tb, thr, step, e_rel,
                      float(np.float32(kappa64)), bool(eligible))


def a_hat(ops, X):
    """Exact A_hat = sum_f x_f wb_f + tb[C] of each row, as the float64 nearest to it (Python integers: x and wb are
    fp16 values, multiples of 2^-24)."""
    Xq = np.ldexp(np.asarray(X, np.float64), 24)
    assert np.all(Xq == np.rint(Xq)), "rows must hold fp16 values"
    wq = np.array([int(w) for w in np.ldexp(ops.wb, 24)], dtype=object)
    s = Xq.astype(np.int64).astype(object).dot(wq)
    return np.array([int(v) / 2**48 for v in s]) + ops.tb[ops.C]


# ---------------------------------------------------------------------------------------------------------------
# exact labels and margins
# ---------------------------------------------------------------------------------------------------------------
def truth(X, coef, intercept):
    """Exact labels (first maximum) and top-2 margins of float64 rows.  Rows whose float64 top-2 gap lies beyond four
    times float64's own error bound keep the float64 result (its margin is within that bound of the exact one); the
    others, exact ties included, are recomputed in integer fixed point (f64_stage_cases.exact_linear)."""
    X = np.asarray(X, np.float64)
    coef = np.atleast_2d(np.asarray(coef, np.float64))
    intercept = np.atleast_1d(np.asarray(intercept, np.float64))
    s = X @ coef.T + intercept
    a = np.abs(X) @ np.abs(coef).T + np.abs(intercept)
    if coef.shape[0] == 1:
        s = np.hstack([np.zeros_like(s), s])
        a = np.hstack([np.zeros_like(a), a])
    err = (X.shape[1] + 2) * U53 * a.max(axis=1) + 2.0**-1070
    order = np.argsort(-s, axis=1, kind="stable")
    top = np.take_along_axis(s, order[:, :2], axis=1)
    labels = order[:, 0].astype(np.int32)
    margins = top[:, 0] - top[:, 1]
    redo = np.flatnonzero(~(margins > 4 * err))
    if redo.size:
        lab, m = exact_linear(X[redo], coef, intercept)
        labels[redo], margins[redo] = lab, m
    return labels, margins


def verdicts(ops, X, margins):
    """+1 must-certify, -1 must-leave, 0 either, per row (margins: exact, unscaled)."""
    A = a_hat(ops, X)
    m = np.ldexp(np.asarray(margins, np.float64), ops.sigma)
    k = ops.kappa * A
    cert = m >= k * (1 + ops.step) * (1 + 4 * U) + 2 * ops.e_rel * A
    leave = m <= k * (1 - ops.step) * (1 - 4 * U) - 2 * ops.e_rel * A
    return np.where(cert, 1, np.where(leave, -1, 0))


def ratio(ops, X, margins):
    """Exact scaled margin over kappa A_hat, per row."""
    return np.ldexp(np.asarray(margins, np.float64), ops.sigma) / (ops.kappa * a_hat(ops, X))


# ---------------------------------------------------------------------------------------------------------------
# exact-on-the-tensor-cores family
# ---------------------------------------------------------------------------------------------------------------
# Scaled weights v = B_f + D_cf: B_f (common to every class) an fp16 value in [2^13, 2^14] on a grid of 8, feature 0's
# 2^14 (so sigma is the model's own).  A "lo" feature's D is a multiple of 1/4 below 4 in magnitude (hi piece B_f, lo
# piece D); a "hi" feature's D a multiple of 8 (hi piece B_f + D, lo piece 0).  Biases are multiples of 8.  A row uses
# lo features only (every score and partial sum a multiple of 1/4) or hi features only (multiples of 8), and stays below
# 2^22 (lo) or 2^26 (hi) in A_hat, so every column sum, the bound column and both epilogue adds are exact in fp32 under
# any accumulation order.  A twin class (a copy of another's weights and bias) gives exact ties.  Rows are drawn at
# random and kept where their exact ratio m / (kappa A_hat) sits on a rung.
SIGMA = 20
LO_LIMIT, HI_LIMIT = 2.0**21, 2.0**25
RUNGS = (0.0, 0.5, 0.99, 1.01, 2.0)
RUNG_TOL = {0.0: 0.0, 0.5: 0.05, 0.99: 0.005, 1.01: 0.005, 2.0: 0.1}
RUNG_TOL_F1 = {**RUNG_TOL, 0.99: 0.01, 1.01: 0.01}  # F = 1: 255 rows per model, the 1 % rungs fill slowly


def rung_window(F, r):
    """[lo, hi] of the exact ratio m / (kappa A_hat) a row of rung r has (the 0.99 / 1.01 rungs stay 0.005 clear of 1)."""
    tol = (RUNG_TOL_F1 if F == 1 else RUNG_TOL)[r]
    lo, hi = r - tol, r + tol
    if r == 0.99:
        hi = 0.995
    if r == 1.01:
        lo = 1.005
    return lo, hi


def exact_model(F, C, rng):
    """(coef, intercept, flavour per feature: 0 lo, 1 hi); class C - 1 is the twin of class 0 (C >= 3).  Two-row
    layouts only: a binary model's class 0 scores 0, so its margin |s| is small only where s cancels, which random
    integer rows rarely do; the other families cover that layout."""
    B = 8.0 * rng.integers(1025, 2048, size=F)
    hi_feat = np.zeros(F, bool)
    hi_feat[1:] = rng.random(F - 1) < 0.5
    D = np.where(hi_feat, 8.0 * rng.integers(-12, 13, size=(C, F)), rng.integers(-12, 13, size=(C, F)) / 4.0)
    v = B + D
    v[:, 0] = 2.0**14 + np.abs(D[:, 0])  # max |v| in [2^14, 2^15): sigma = SIGMA
    b = 8.0 * rng.integers(-64, 65, size=C)
    if C >= 4:  # a class that never leads with a bias as large as sum_f x_f wb_f: tb[C] then carries A_hat
        b[C - 2] = -8.0 * rng.integers(2**11, 2**15)
    if C >= 3:
        v[C - 1], b[C - 1] = v[0], b[0]
    return np.ldexp(v, -SIGMA), np.ldexp(b, -SIGMA), hi_feat.astype(int)


def _candidates(F, flav, rng, n, kind):
    """n random rows on the features of one flavour: about 3 of them nonzero, integers 1..255."""
    X = np.zeros((n, F))
    use = np.flatnonzero(flav == kind)
    if use.size:
        on = rng.random((n, use.size)) < min(1.0, 3.0 / use.size)
        X[:, use] = np.where(on, rng.integers(1, 256, size=(n, use.size)), 0)
    return X[X.any(axis=1)]


def exact_family(F, C, seed=0, per_rung=12):
    """Parts [(coef, intercept, X float32)] of the exact family at (F, C): together every rung holds >= per_rung rows
    (at F = 1 several models, each with its own rows).  Row order is shuffled within each part."""
    rng = np.random.default_rng(seed)
    parts, counts = [], {r: 0 for r in RUNGS}
    need = RUNGS
    if F == 1:
        per_rung = min(per_rung, 4)
    for _ in range(200):
        coef, intercept, flav = exact_model(F, C, rng)
        ops = operands(coef, intercept)
        assert ops.sigma == SIGMA and ops.eligible
        if F == 1:
            X = np.arange(1, 256, dtype=np.float64)[:, None]
        else:
            X = np.vstack([_candidates(F, flav, rng, 2000, 0), _candidates(F, flav, rng, 1000, 1)])
        # float64 is exact here (every term on the grid, far below 2^53 units); the CPU tests check that
        A = X @ ops.wb + ops.tb[C]
        X, A = X[A + np.abs(ops.tb).max() < np.where((X[:, flav == 1] != 0).any(axis=1), HI_LIMIT, LO_LIMIT)], None
        A = X @ ops.wb + ops.tb[C]
        top = -np.sort(-(X @ np.ldexp(ops.W, SIGMA).T + ops.tb[:C]), axis=1)[:, :2]
        rho = (top[:, 0] - top[:, 1]) / (ops.kappa * A)
        keep = []
        for r in RUNGS:
            lo, hi = rung_window(F, r)
            near = np.flatnonzero((rho >= lo) & (rho <= hi))
            take = near[: max(0, 4 * per_rung - counts[r])]
            counts[r] += take.size
            keep.append(take)
        keep = np.concatenate(keep)
        if keep.size:
            Xk = X[rng.permutation(keep)].astype(np.float32)
            parts.append((coef, intercept, Xk))
        if all(counts[r] >= per_rung for r in need):
            return parts
    raise AssertionError(f"exact family F={F} C={C}: rungs {counts}")


def rung_of(ops, X, margins):
    """The rung each row was kept for (exact ratio within RUNG_TOL of it), or nan."""
    rho = ratio(ops, X, margins)
    out = np.full(len(X), np.nan)
    for r in RUNGS:
        lo, hi = rung_window(ops.F, r)
        out[(rho >= lo) & (rho <= hi)] = r
    return out


def exact_column_bound_ok(ops, X, grid):
    """Every hi / lo / bound column partial sum and both epilogue adds of every row: multiples of `grid` below 2^24
    grid units, checked through their absolute bounds (any summation order stays inside them)."""
    X = np.asarray(X, np.float64)
    for M in (ops.hi, ops.lo, ops.wb[None, :]):
        P = X[:, None, :] * M[None, :, :]
        if not np.all(np.mod(P, grid) == 0):
            return False
        if not np.all(np.abs(P).sum(axis=2) < 2.0**24 * grid):
            return False
    top = (X @ np.abs(ops.hi).T + X @ np.abs(ops.lo).T + np.abs(ops.tb[: ops.C]))
    return bool(np.all(top < 2.0**24 * grid) and np.all(np.mod(ops.tb, grid) == 0))


# ---------------------------------------------------------------------------------------------------------------
# rounding family: the tensor cores round
# ---------------------------------------------------------------------------------------------------------------
def rounding_model(F, C, rng, binary=False):
    """Full-mantissa float64 weights spread over 2^+-12 across classes; class pairs (2k, 2k + 1) near-duplicates at a
    relative distance log-uniform over 2^-22 .. 2^-6, so the leading pair's margin runs over about 0.1 .. 10 kappa A;
    the last class (C >= 4) entirely below 2^-11 of max|W| (small hi pieces; a weight that scaled falls below 2^-14 is
    an fp16 subnormal or 0); feature 16 j (j >= 0) the dominant weight of its k16 group."""
    n = 1 if binary else C
    W = rng.uniform(0.5, 1.0, (n, F)) * rng.choice([-1.0, 1.0], (n, F))
    W[:, ::16] *= 64.0
    scale = np.exp2(rng.integers(-12, 13, size=n).astype(float))
    for c in range(1, n, 2):
        scale[c] = scale[c - 1]
        rel = np.exp2(rng.uniform(-22, -6))
        W[c] = W[c - 1] * (1 + rel * rng.uniform(-1, 1, F))
    W *= scale[:, None]
    if n >= 4:
        W[-1] = np.abs(W).max() * 2.0**-11 * rng.uniform(-1, 1, F) * np.exp2(rng.integers(-30, 0, size=F))
        W[-1, rng.random(F) < 0.25] = 0.0
    b = rng.uniform(-1, 1, n) * np.abs(W).max() * rng.choice([2.0**-20, 1.0, 64.0], n)
    for c in range(1, n, 2):
        b[c] = b[c - 1] * (1 + np.exp2(rng.uniform(-22, -6)) * rng.uniform(-1, 1))
    return W, b


def rounding_rows(F, rng, n, route):
    """half: fp16 values up to 65504, fp16 subnormals; byte: 0..255 with sparse 255s."""
    if route == "byte":
        X = rng.integers(0, 32, size=(n, F)).astype(np.float64)
        X[rng.random((n, F)) < 0.05] = 255.0
        X[rng.random((n, F)) < 0.3] = 0.0
        return X.astype(np.float32)
    e = rng.integers(-24, 16, size=(n, F))
    X = f16_round(np.minimum(rng.uniform(1, 2, (n, F)) * np.exp2(e), 65504.0))
    X[rng.random((n, F)) < 0.02] = 65504.0
    X[rng.random((n, F)) < 0.3] = 0.0
    return X.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# fp32-route-flags family: weights near 2^-120, so the fp32 route's bound is its K term (upload_model) and it flags
# every row whose margin is below ~FLT_MIN; tier 1 must leave all of them
# ---------------------------------------------------------------------------------------------------------------
def tiny_model(F, C, rng):
    """Weights 2^-120 (1 + d), |d| below 2^-6: the margins sit far below FLT_MIN."""
    W = 2.0**-120 * (1 + np.exp2(rng.uniform(-16, -6, (C, F))) * rng.uniform(-1, 1, (C, F)))
    return W, np.zeros(C)


def tiny_rows(F, rng, n, route):
    """byte: small integers on a few features; half: fp16 subnormals (the fp32 route's products are subnormal)."""
    X = np.zeros((n, F))
    for i in range(n):
        f = rng.choice(F, min(F, rng.integers(1, 4)), replace=False)
        X[i, f] = rng.integers(1, 64, size=f.size) if route == "byte" else rng.integers(1, 1024, size=f.size) * 2.0**-24
    return X.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# lossy float64 family: values v + 2^-30 that the fp32 cast (and so the byte and fp16 copies) rounds to v
# ---------------------------------------------------------------------------------------------------------------
def lossy_case(F, C, rng, n, binary=False):
    """(coef, intercept, X float64).  Classes a < b differ only on feature t (w_b,t = w_a,t + d) and in bias
    (b_b = b_a - 3 d), so on the cast row (x_t = 3) they tie and a wins, while x_t = 3 + 2^-30 gives b."""
    m = 1 if binary else C
    W = rng.integers(-4, 5, size=(m, F)).astype(np.float64)
    b = rng.integers(-8, 9, size=m).astype(np.float64)
    t = F - 1
    if not binary:
        W[1], b[1] = W[0], b[0]
        W[1, t] += 1.0
        b[1] -= 3.0
        W[0] += 8.0  # classes 0 and 1 lead every row
        W[1] += 8.0
    else:  # s = w.x + b: 0 on the cast row, 2^-30 d on the float64 one
        W[0, t] = 1.0
        W[0, :t] = 0.0
        b[0] = -3.0
    X = rng.integers(0, 8, size=(n, F)).astype(np.float64)
    X[:, t] = 3.0 + rng.choice([0.0, 2.0**-30, -2.0**-30], n)
    return W, b, X


# ---------------------------------------------------------------------------------------------------------------
# subnormal pieces: scaled weights around q = 2^-24, the fp16 subnormal spacing, where hi + lo errs by up to q / 2
# ---------------------------------------------------------------------------------------------------------------
def subnormal_pieces_case(F, C, route, n=1001):
    """(coef, intercept, X).  Scaled by 2^sigma (sigma = 14, set by a weight 1 on feature 0), class 0 has 1.49 q on
    feature 1, class 1 has 0.51 q on features 1 and 2, every other class 0 there.  Exactly class 0 leads by 0.47 q x
    on a row x_1 = x_2 = x; the pieces give class 0 q (hi q, lo 0) and class 1 2 q, so the tensor cores rank class 1
    first by q x.  Only the 2^-3 floor of wb puts that row out of tier 1's reach (wb of q and 2 q would not)."""
    assert F >= 3 and C >= 2
    q = 2.0**-24
    W = np.zeros((C, F))
    W[0, 0] = 1.0
    W[0, 1] = 1.49 * q * 2.0**-14
    W[1, 1] = W[1, 2] = 0.51 * q * 2.0**-14
    rng = np.random.default_rng(F * 31 + C)
    x = rng.integers(1, 256, size=n).astype(np.float64) if route == "byte" else f16_round(rng.uniform(1, 65504, n))
    X = np.zeros((n, F))
    X[:, 1] = X[:, 2] = x
    return W, np.zeros(C), X.astype(np.float32)
