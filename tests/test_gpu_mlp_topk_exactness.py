"""EXACT top-k of the MLP predictor against exact arithmetic, on every route that ranks classes.

EXACT top-k promises the exact order of the first k classes and the exact boundary between rank k and rank k + 1
(ties to the lower class index, np.argsort(-z, kind="stable")), or the row is counted in ``n_ambiguous``.  Two rules
keep that promise: the fp32 rank guard of the tile kernels (mlp_topk_certain: every consecutive gap among ranks
1 .. kk + 1, kk = min(k, C - 1), above 2δ) and the float64 rank rule behind them (mlp_f64_row_outputs: the same gaps
above twice the float64 logit bound), DESIGN.md 3.8 and 3.10.  The reference is tests/f64_stage_cases.exact_mlp_topk
(float64 where it is sure, Fractions elsewhere).

  a. the tile guard on data whose fp32 arithmetic is exact: a gap planted at 0, 0.5x and 3x the kernel's own 2δ
     between ranks r and r + 1 is flagged exactly when r <= k (and never when it is 3x);
  b. near-ties at every rank boundary, 1e-4x .. 100x 2δ, on data spread over 2^+-10;
  c. the underflow constructions of the label tests, moved below rank 1;
  d. the float64 rank rule on every route that uses it: gaps on the ladder of the stage's own bound beta, split into
     certain / inside / straddle batches (tests/test_gpu_f64_stage_edges.py's contract, applied to ranks).
"""
import numpy as np
import pandas as pd
import pytest
import torch

from tests import f64_stage_cases as K

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.test_gpu_exactness_edges import (  # noqa: E402
    MLP_CONSTRUCTIONS,
    MLP_EPS_FACTORS,
    PLANT_AT,
    exact_mlp_labels,
    mlp_construction,
    spread,
)
from tests.test_gpu_f64_stage_edges import check_batch  # noqa: E402
from tests.test_gpu_mlp_proba import _logit_bound  # noqa: E402

TILE_SHAPES = [({2: 32, 3: 50, 10: 128}[C], H, C) for H in (16, 32) for C in (2, 3, 10)]
KERNELS = {"tensor_core": ("1", 5), "cuda_core": ("0", 3)}
KMAX = 5  # kMlpTopkMax: larger k is served by the float64 kernel (path 2)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def shape_id(s):
    return "x".join(map(str, s))


# ---------------------------------------------------------------------------------------------------------------
# a. the tile guard at every rank boundary, on exact data.  Logit c = x0 + x_hi,c + x_lo,c through identity weights:
# every feature is a tf32 integer and every sum stays below 2^24, so fp32 (and the tensor cores' tf32 split of W1 = 1)
# compute each logit exactly, and the guard sees the planted gaps as they are.
# ---------------------------------------------------------------------------------------------------------------
BIG = 16.0  # every other consecutive gap, in units of 2δ


def boundary_case(F, H, C, r, factor, path, n=300, seed=0):
    """(weights, rows, 2δ per row): the gap between ranks r and r + 1 is factor x 2δ, every other gap BIG x 2δ, the
    classes in a random order per row."""
    rng = np.random.default_rng(seed)
    w1 = np.zeros((H, F), np.float32)
    w2 = np.zeros((C, H), np.float32)
    w1[0, 0] = 1.0
    w2[:, 0] = 1.0  # hidden unit 0 = x0 feeds every logit alike: it sets δ, not the gaps
    for c in range(C):
        w1[1 + c, 1 + 2 * c] = w1[1 + c, 2 + 2 * c] = 1.0
        w2[c, 1 + c] = 1.0
    w = (w1, np.zeros(H, np.float32), w2, np.zeros(C, np.float32))
    X = np.zeros((n, F), np.float32)
    X[:, 0] = rng.integers(1024, 2048, n) * 2.0**12  # tf32 integers in [2^22, 2^23)
    order = np.argsort(rng.random((n, C)), axis=1)  # order[i, j]: the class at rank j + 1 of row i
    units = np.full(C - 1, BIG)
    units[r - 1] = factor
    for _ in range(4):  # δ depends a little on the tuning features: settle it
        d2 = 2 * _logit_bound(X, w, path)
        g = np.rint(units[None, :] * d2[:, None])
        T = np.concatenate([np.cumsum(g[:, ::-1], axis=1)[:, ::-1], np.zeros((n, 1))], axis=1)  # rank j's offset
        assert T.max() < 2.0**18
        hi = np.floor(T / 128) * 128
        rows = np.arange(n)[:, None]
        X[rows, 1 + 2 * order] = hi
        X[rows, 2 + 2 * order] = T - hi
    assert not (X.view(np.uint32) & np.uint32(0x1FFF)).any() and X.max() < 2**23
    d2 = 2 * _logit_bound(X, w, path)
    ratio = g / d2[:, None]
    assert np.allclose(ratio[:, r - 1], factor, rtol=0.03, atol=0.0) and (np.delete(ratio, r - 1, axis=1) > BIG - 1).all()
    return w, X, d2


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("shape", TILE_SHAPES, ids=shape_id)
def test_tile_guard_rank_boundaries(engine, monkeypatch, shape, kernel):
    """A planted gap at 0.5x 2δ between ranks r and r + 1 is flagged on every row once k >= r and on none while k < r
    (the guard looks at ranks 1 .. k + 1, no further); at 3x it is never flagged; an exact tie (0x) is flagged, ranked
    lower index first and counted ambiguous.  FAST gives the same ranks: the data is exact."""
    F, H, C = shape
    tc, path = KERNELS[kernel]
    monkeypatch.setenv("UML_B200_MLP_TC", tc)
    fails = []
    for r in range(1, min(C - 1, KMAX) + 1):
        for factor in (0.0, 0.5, 3.0):
            w, X, _ = boundary_case(F, H, C, r, factor, path, seed=10 * r + int(2 * factor))
            m = engine.load_mlp(*w)
            b = engine.stage(X)
            n = len(X)
            for k in range(1, min(C, KMAX) + 1):
                want, gap = K.exact_mlp_topk(X, *w, k)
                tag = f"r={r} {factor}x k={k}"
                idx, _, st = engine.predict_mlp_topk(m, b, k, exact=True)
                assert st["path"] == path, (tag, st)
                if k == 1:  # k = 1 is the label guard
                    _, sl = engine.predict_mlp(m, b, exact=True)
                    if sl["n_flagged"] != st["n_flagged"]:
                        fails.append(f"{tag}: labels flag {sl['n_flagged']} rows, top-1 {st['n_flagged']}")
                flagged = factor < 1 and k >= r
                if st["n_flagged"] != (n if flagged else 0):
                    fails.append(f"{tag}: n_flagged {st['n_flagged']}, want {n if flagged else 0} of {n}")
                if st["n_ambiguous"] != (n if factor == 0 and k >= r else 0):
                    fails.append(f"{tag}: n_ambiguous {st['n_ambiguous']}")
                bad = np.flatnonzero(np.any(idx != want, axis=1))
                if bad.size:
                    fails.append(f"{tag} EXACT: {bad.size} rows differ, e.g. {idx[bad[0]].tolist()} want {want[bad[0]].tolist()}")
                fast, _, _ = engine.predict_mlp_topk(m, b, k, exact=False)
                bad = np.flatnonzero(np.any(fast != want, axis=1))
                if bad.size:
                    fails.append(f"{tag} FAST: {bad.size} rows differ, e.g. {fast[bad[0]].tolist()} want {want[bad[0]].tolist()}")
            b.free()
    assert not fails, "\n".join(fails[:20])


# ---------------------------------------------------------------------------------------------------------------
# b. near-ties at every rank boundary: w2_c = w2_0 (1 + eps r_c), features and weights spread over 2^+-10
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("shape", TILE_SHAPES, ids=shape_id)
def test_rank_near_tie_sweep(engine, monkeypatch, shape, kernel):
    F, H, C = shape
    tc, path = KERNELS[kernel]
    rng = np.random.default_rng(F * 7 + H * 3 + C)
    N = 8_000
    X = spread(rng, (N, F), -10, 10, tf32=True)
    w1, b1 = spread(rng, (H, F), -10, 10), spread(rng, H, -10, 10)
    w20, b20 = spread(rng, H, -10, 10).astype(np.float64), float(spread(rng, 1, -10, 10)[0])
    rc, rb = rng.standard_normal((C - 1, H)), rng.standard_normal(C - 1)
    x64 = X.astype(np.float64)
    h = np.maximum(x64 @ w1.astype(np.float64).T + b1, 0)
    d = h @ np.vstack([np.zeros(H), w20 * rc]).T + np.concatenate([[0.0], b20 * rb])  # logit offsets at eps = 1
    kmax = min(C, KMAX)
    ds = np.sort(d, axis=1)[:, ::-1]
    dgap = (ds[:, : min(kmax, C - 1)] - ds[:, 1 : min(kmax, C - 1) + 1]).min(axis=1)

    def net(eps):
        w2 = np.vstack([w20, w20 * (1 + eps * rc)]).astype(np.float32)
        b2 = np.concatenate([[b20], b20 * (1 + eps * rb)]).astype(np.float32)
        return w1, b1, w2, b2

    # eps = 1 gives gaps dgap; scale eps so that the gaps among ranks 1 .. kk + 1 span 1e-4x .. 100x 2δ
    base = np.median(2 * _logit_bound(X, net(1.0), path) / np.maximum(dgap, 1e-300))
    monkeypatch.setenv("UML_B200_MLP_TC", tc)
    b = engine.stage(X)
    n_fast_wrong = n_flagged = n_within = n_near = 0
    for f in MLP_EPS_FACTORS:
        w = net(f * base)
        delta = _logit_bound(X, w, path)
        m = engine.load_mlp(*w)
        flagged = []
        for k in range(1, kmax + 1):
            want, gap = K.exact_mlp_topk(X, *w, k)
            idx, _, st = engine.predict_mlp_topk(m, b, k, exact=True)
            assert st["path"] == path, st
            # at the smallest eps, eps r_c can fall below fp32's resolution of w2: some rows' exact gaps then sit inside
            # the float64 stage's bound beta (C = 2), and only those may be wrong, if counted in n_ambiguous
            near = gap <= 2 * K.mlp_beta(X, *w)
            bad = np.flatnonzero(np.any(idx != want, axis=1))
            assert near[bad].all(), (f"eps {f}x k={k}: EXACT wrong on rows {bad[~near[bad]].tolist()[:8]} whose gaps lie "
                                     f"beyond the float64 bound (flagged {st['n_flagged']})")
            assert bad.size <= st["n_ambiguous"] <= int(near.sum()), (f, k, bad.size, st["n_ambiguous"], int(near.sum()))
            n_near += int(near.sum())
            fast, _, _ = engine.predict_mlp_topk(m, b, k, exact=False)
            n_fast_wrong += int(np.any(fast != want, axis=1).sum())
            within = int((gap <= 2.02 * delta).sum())
            # a flagged row has a computed gap <= 2δ: a guard flagging rows whose exact gaps lie beyond is vacuous
            assert st["n_flagged"] <= within, (f, k, st["n_flagged"], within)
            flagged.append(st["n_flagged"])
            n_flagged += st["n_flagged"]
            n_within += within
        assert flagged == sorted(flagged), (f, flagged)  # more ranks to certify never certify more rows
    print(f"\nmlp {kernel} {F}->{H}->{C} top-1..{kmax}: FAST wrong {n_fast_wrong}, flagged {n_flagged} <= {n_within} "
          f"rows within 2.02 δ, {n_near} within 2 beta, of {N * len(MLP_EPS_FACTORS) * kmax}")
    assert n_fast_wrong >= 20  # the data has teeth: plain fp32 ranks many of these rows wrongly
    b.free()


# ---------------------------------------------------------------------------------------------------------------
# c. the underflow constructions, with the planted pair moved to ranks r, r + 1: classes 2 .. r sit above it at 2^j
# times its larger logit (the same magnitude: A2 barely moves, so the bound does not grow to hide a hole)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("shape", [(64, 32, 10), (128, 16, 3)], ids=shape_id)
@pytest.mark.parametrize("name", MLP_CONSTRUCTIONS)
def test_underflow_constructions_below_rank_one(engine, monkeypatch, name, shape, kernel):
    F, H, C = shape
    tc, path = KERNELS[kernel]
    rng = np.random.default_rng(F + H + C)
    w1, b1, w2, b2, x = mlp_construction(name, F, H, C, rng)
    X = np.zeros((10_007, F), np.float32)
    X[:, 4:] = rng.integers(0, 9, size=(10_007, F - 4))
    X[list(PLANT_AT)] = x
    z = K._exact_mlp_logits(x, w1, b1, w2, b2)
    top = max(z[0], z[1])
    assert min(z[0], z[1]) > 0 and all(v == 0 for v in z[2:])  # the other classes score their bias on the planted row
    monkeypatch.setenv("UML_B200_MLP_TC", tc)
    b = engine.stage(X)
    fails = []
    for r in range(2, min(C - 1, KMAX) + 1):
        b2r = b2.copy()
        for j in range(1, r):
            b2r[1 + j] = np.float32(float(top) * 2.0 ** (r - j))  # classes 2 .. r above the pair, in that order
        w = (w1, b1, w2, b2r)
        m = engine.load_mlp(*w)
        for k in range(r, min(C, KMAX) + 1):
            want, _ = K.exact_mlp_topk(X, *w, k)
            planted = want[list(PLANT_AT)]
            assert (planted[:, : r - 1] == np.arange(2, r + 1)).all() and set(planted[:, r - 1]) <= {0, 1}, planted
            if k > r:
                assert (np.sort(planted[:, r - 1 : r + 1], axis=1) == [0, 1]).all()
            assert (planted[:, 0] == exact_mlp_labels(X[list(PLANT_AT)], *w)).all()
            idx, _, st = engine.predict_mlp_topk(m, b, k, exact=True)
            assert st["path"] == path, st
            bad = np.flatnonzero(np.any(idx != want, axis=1))
            if bad.size:
                fails.append(f"r={r} k={k}: rows {bad.tolist()[:6]} got {idx[bad[:3]].tolist()} want {want[bad[:3]].tolist()}")
    b.free()
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------
# d. the float64 rank rule on every route.  tests/f64_stage_cases.mlp_rank_case: float64 is exact on these rows, so
# without ties rows below beta must be counted and rows above it certified (the bound factor itself); with a duplicated
# class the rungs are those of the label tests (certain >= 4 beta, inside <= beta / 4, straddle between).
# ---------------------------------------------------------------------------------------------------------------
def rank_rungs(gap, beta, tie):
    if tie:
        return K.rungs(gap, beta)
    return np.flatnonzero(gap > beta), np.flatnonzero(gap < beta), np.array([], np.int64)


def check_ranks(fails, tag, rung, got, st, want, pair=None):
    """check_batch on whole rows (a row is right when all k indices are); pair = (a, t): the exact-tie classes, of
    which the lower index must come first (and be there whenever the other is)."""
    C = int(max(got.max(), want.max())) + 1
    key = lambda a: (a.astype(np.int64) * C ** np.arange(a.shape[1])).sum(axis=1)  # noqa: E731
    check_batch(fails, tag, rung, key(got), st, key(want))
    if pair is not None and pair[1] >= 0:
        lo, hi = min(pair), max(pair)
        for row in got.tolist():
            if hi in row and (lo not in row or row.index(lo) > row.index(hi)):
                fails.append(f"{tag} {rung}: exact tie ranked {row}, {lo} must come before {hi}")
                break


def rank_cases(F, H, C, rs, ks, big=False):
    """(tag, net, X, k, rung, rows, pair) of every planted boundary r in rs, with and without a duplicated class."""
    out = []
    for r in rs:
        for tie in (False, True):
            if r + (2 if tie else 1) > C:
                continue
            net, X, _, _, (a, b, t) = K.mlp_rank_case(F, H, C, r, tie=tie, big=big, seed=F + H + C + r)
            beta = K.mlp_beta(X, *net)
            for k in ks:
                if k > C:
                    continue
                want, gap = K.exact_mlp_topk(X, *net, k)
                for rung, rows in zip(("certain", "inside", "straddle"), rank_rungs(gap, beta, tie)):
                    if rows.size:
                        tag = f"{F}-{H}-{C} r={r}{' tie' if tie else ''} k={k}"
                        out.append((tag, net, X, k, rung, rows, want, (a, t) if tie else None))
    return out


def topk_rows(engine, net, X, k, exact=True):
    m = engine.load_mlp(*net)
    b = engine.stage(X)
    idx, _, st = engine.predict_mlp_topk(m, b, k, exact=exact)
    b.free()
    return idx, st


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("shape", [(64, 32, 10), (50, 16, 3), (32, 16, 2)], ids=shape_id)
def test_rank_rule_behind_the_tile_kernels(engine, monkeypatch, shape, kernel):
    """mlp_topk_f64_kernel on the rows a tile kernel flagged (every non-certain row must be flagged: its gaps lie
    far inside the fp32 bound).  k == C covers kk = C - 1 at C = 2 and 3."""
    F, H, C = shape
    tc, path = KERNELS[kernel]
    monkeypatch.setenv("UML_B200_MLP_TC", tc)
    fails = []
    rs = range(1, min(C - 1, KMAX) + 1)
    ks = sorted({1, 2, 3, min(C, KMAX)})
    for tag, net, X, k, rung, rows, want, pair in rank_cases(F, H, C, rs, ks):
        idx, st = topk_rows(engine, net, X[rows], k)
        if st["path"] != path:
            fails.append(f"{tag}: path {st['path']} != {path}")
        if rung != "certain" and st["n_flagged"] < rows.size:
            fails.append(f"{tag} {rung}: n_flagged {st['n_flagged']} < {rows.size}")
        check_ranks(fails, tag, rung, idx, st, want[rows], pair)
    assert not fails, "\n".join(fails[:20])


def test_rank_rule_on_the_float64_kernel(engine):
    """Path 2, every row through mlp_topk_f64_kernel: k > 5 at C = 10 (k = 10: kk = 9, every gap), and a shape no tile
    kernel takes at ragged row counts (4 rows per warp pass)."""
    fails = []
    for tag, net, X, k, rung, rows, want, pair in rank_cases(64, 32, 10, (1, 6, 9), (6, 10)):
        idx, st = topk_rows(engine, net, X[rows], k)
        if st["path"] != 2:
            fails.append(f"{tag}: path {st['path']} != 2")
        check_ranks(fails, tag, rung, idx, st, want[rows], pair)
    for tag, net, X, k, rung, rows, want, pair in rank_cases(40, 24, 5, (1, 2, 4), (1, 2, 4, 5)):
        for n in (1, 2, 3, 5, 9, 10, 11):
            sub = np.resize(rows, n)
            idx, st = topk_rows(engine, net, X[sub], k)
            if st["path"] != 2:
                fails.append(f"{tag}: path {st['path']} != 2")
            check_ranks(fails, f"{tag} n={n}", rung, idx, st, want[sub], pair)
    assert not fails, "\n".join(fails[:20])


def test_rank_rule_through_the_chunk_pipeline(engine):
    """predict_mlp_topk_host with more than 64 rows in chunks of 128: float64 frames in C and F order, an int64 frame
    (integer rows, beta ~ 35), and a mixed frame whose first 2048 rows are tf32 values (the tensor cores are chosen)
    and whose planted rows, in a later chunk, are not: EXACT and FAST re-score them in float64 alike."""
    fails = []
    F, H, C = 64, 32, 10
    pad = lambda rows: np.resize(rows, max(300, rows.size))  # noqa: E731  (> 64 rows: not the online route)
    for big in (False, True):
        for tag, net, X, k, rung, rows, want, pair in rank_cases(F, H, C, (1, 3), (1, 3), big=big):
            m = engine.load_mlp(*net)
            sub = pad(rows)
            frames = {"int64": X[sub].astype(np.int64)} if big else {
                "float64 C": X[sub].astype(np.float64), "float64 F": np.asfortranarray(X[sub].astype(np.float64))}
            for name, frame in frames.items():
                idx, _, st = engine.predict_mlp_topk_host(m, frame, k, exact=True, chunk_rows=128)
                if st["path"] != 5:
                    fails.append(f"{tag} {name}: path {st['path']} != 5")
                check_ranks(fails, f"{tag} {name}", rung, idx, st, want[sub], pair)
    # the mixed frame: x2 with its lowest mantissa bit set is not a tf32 value (its exact gaps are measured again)
    for tag, net, X, k, rung, rows, want, pair in rank_cases(F, H, C, (1, 3), (1, 3)):
        if pair is not None:  # (a filler row would tie the duplicated class with its twin at 0)
            continue
        Xp = X[rows].copy()
        Xp[:, 2] = (Xp[:, 2].view(np.uint32) | np.uint32(1)).view(np.float32)
        filler = np.zeros((2048, F), np.float32)  # h0 = 0: every gap >= c0 = 16 beta, exact in any arithmetic
        frame = np.concatenate([filler, Xp]).astype(np.float64)
        want_all, gap = K.exact_mlp_topk(frame, *net, k)
        beta = K.mlp_beta(frame, *net)
        planted = np.arange(2048, len(frame))
        sel = rank_rungs(gap[planted], beta[planted], pair is not None)[("certain", "inside", "straddle").index(rung)]
        if sel.size != planted.size:  # the set bit moved a row to another rung: keep this batch to one rung
            continue
        m = engine.load_mlp(*net)
        for exact in (True, False):
            idx, _, st = engine.predict_mlp_topk_host(m, frame, k, exact=exact, chunk_rows=1024)
            mode = "EXACT" if exact else "FAST"
            if st["path"] != 5 or st["n_flagged"] < planted.size:
                fails.append(f"{tag} mixed {mode}: path {st['path']}, n_flagged {st['n_flagged']} < {planted.size}")
            if np.any(idx[:2048] != want_all[:2048]):
                fails.append(f"{tag} mixed {mode}: tf32 rows ranked wrongly")
            check_ranks(fails, f"{tag} mixed {mode}", rung, idx[planted], st, want_all[planted], pair)
    assert not fails, "\n".join(fails[:20])


def test_rank_rule_on_the_online_route(engine):
    """<= 64 rows: one mlp_small_kernel launch, replayed as a CUDA graph for the same key; float64 ranks in FAST and
    EXACT, ambiguity reported through the row's status."""
    fails = []
    for tag, net, X, k, rung, rows, want, pair in rank_cases(64, 32, 10, (1, 3, 5), (1, 3, 5, 10)):
        m = engine.load_mlp(*net)
        for n in (1, 7, 64):
            sub = np.resize(rows, n)
            for exact in (True, False):
                for call in ("capture", "replay"):
                    idx, _, st = engine.predict_mlp_topk_host(m, X[sub].astype(np.float64), k, exact=exact)
                    if st["path"] != 4:
                        fails.append(f"{tag} n={n}: path {st['path']} != 4")
                    check_ranks(fails, f"{tag} n={n} {'EXACT' if exact else 'FAST'} {call}", rung, idx, st, want[sub], pair)
    for tag, net, X, k, rung, rows, want, pair in rank_cases(32, 16, 3, (1, 2), (3,)):  # k == C at C = 3
        m = engine.load_mlp(*net)
        idx, _, st = engine.predict_mlp_topk_host(m, X[rows].astype(np.float64), k)
        check_ranks(fails, f"{tag} online", rung, idx, st, want[rows], pair)
    assert not fails, "\n".join(fails[:20])


def test_rank_rule_through_mlp_predict_topk(engine):
    """The public predictor on a DataFrame: indices as int64, ambiguity through last_ambiguous_rows()."""
    import torch.nn as nn

    from unionml_b200 import predictors

    F, H, C = 64, 32, 10
    fails = []
    for tag, net, X, k, rung, rows, want, pair in rank_cases(F, H, C, (3,), (3,)):
        module = nn.Sequential(nn.Linear(F, H), nn.ReLU(), nn.Linear(H, C))
        with torch.no_grad():
            for layer, (w, bias) in ((module[0], net[:2]), (module[2], net[2:])):
                layer.weight.copy_(torch.from_numpy(w))
                layer.bias.copy_(torch.from_numpy(bias))
        sub = np.resize(rows, max(100, rows.size))
        _, idx = predictors.mlp_predict_topk(module, pd.DataFrame(X[sub].astype(np.float64)), k=k)
        assert idx.dtype == np.int64
        st = {"n_ambiguous": predictors.last_ambiguous_rows()}
        check_ranks(fails, f"{tag} mlp_predict_topk", rung, idx, st, want[sub], pair)
    assert not fails, "\n".join(fails)
