"""The float64 re-score stage of EXACT mode against exact arithmetic, on every route that gives it the final label.

Contract: in EXACT mode every row either gets the argmax of its exact scores (integer arithmetic in units of 2^-2148,
numpy's first-maximum rule), or is counted in ``n_ambiguous``.  Since ``n_ambiguous`` is a count, planted rows go in
separate batches by their exact margin against the stage's own bound beta (tests/f64_stage_cases.py restates the
kernels' formulas):
  certain  (margin >= 4 beta): every label exact and n_ambiguous == 0;
  inside   (exact ties, margin <= beta / 4): n_ambiguous == rows;
  straddle (between): rows with a wrong label <= n_ambiguous <= rows.
The scores are cancellations of terms spread over 2^+-20 with both signs, so float64 really errs: the inside rows
often get a label other than the exact one.  Near-ties at float64 resolution always fail the fp32 guard, so on the
tile routes n_flagged >= planted rows, and every case asserts the route (`path`) it took.

Also here: the bound factor on data whose float64 arithmetic is exact (rows at 0.6..0.9 beta must be counted, rows at
1.3..3 beta certified), products below DBL_MIN, finite features whose float64 scores overflow to inf / NaN (the
reference is LogisticRegression.predict itself), and the StandardScaler fold with mean_ >> scale_.
"""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from tests import f64_stage_cases as K
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)


def run_report(func, env, args=""):
    """Run tests.test_gpu_f64_stage_edges.<func>(args) in a fresh interpreter (the re-score modes are read once per
    process); it returns a list of failure strings."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from tests.test_gpu_f64_stage_edges import %s as f\n"
        "fails = f(%s)\n"
        "print('\\n'.join(fails)); print('failures', len(fails))\n"
    ) % (str(ROOT), func, args)
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    print(r.stdout)
    assert r.stdout.strip().endswith("failures 0"), r.stdout[-6000:]


def check_batch(fails, tag, rung, got, st, want, lower=None):
    """The contract for one batch.  lower: rows whose computed scores are bitwise ties (duplicate classes) and must get
    the lower index, like np.argmax."""
    n = got.size
    wrong = int((got != want).sum())
    amb = int(st["n_ambiguous"])
    if rung == "certain" and (wrong or amb):
        fails.append(f"{tag} certain: {wrong} wrong labels, n_ambiguous {amb} of {n}")
    if rung == "inside" and amb != n:
        fails.append(f"{tag} inside: n_ambiguous {amb} != {n} rows")
    if rung == "straddle" and not (wrong <= amb <= n):
        fails.append(f"{tag} straddle: {wrong} wrong > n_ambiguous {amb} (rows {n})")
    if lower is not None and np.any(got[lower[0]] != lower[1]):
        bad = np.flatnonzero(got[lower[0]] != lower[1])
        fails.append(f"{tag}: exact ties got {got[lower[0]][bad][:6].tolist()} want {lower[1][bad][:6].tolist()}")
    return wrong


def ladder_case(F, C, binary, seed, kind="f64", n_per=24, dups=None, wexp=(-20, 20), anchor=None):
    """Model and planted rows on the margin ladder: (coef, intercept, X, want, margin, beta, tie rows, tie labels).
    anchor: feature 0 gets this weight in every class and this value in every row (f64_stage_cases.ladder_rows)."""
    rng = np.random.default_rng(seed)
    if dups is None:
        dups = [] if binary or C < 4 else [(0, C - 1)]
    coef, intercept, tune = K.ladder_model(F, C, rng, dups=dups, binary=binary, wexp=wexp, anchor=anchor)
    twins = {b for _, b in dups} | {a for a, _ in dups}
    free = [c for c in range(C) if c not in twins]
    tops, ks = [], []
    ladder = [0.0, 1e-3, 0.02, 0.1, 0.2, 0.5, 1.0, 2.0, 5.0, 10.0, 100.0]
    for k in ladder:
        for i in range(n_per if k else n_per // 2):
            if binary:
                tops.append((i % 2, 1 - i % 2))
            else:
                a, b = rng.choice(free, 2, replace=False)
                if C > 16 and i % 3 == 0:  # across the 16-class groups: later group on top, and the reverse
                    a, b = (free[-1], free[1]) if i % 2 else (free[1], free[-1])
                tops.append((int(a), int(b)))
            ks.append(k)
    n_ties = 0
    for a, b in dups:  # exact ties: the duplicate pair on top
        tops += [(a, b)] * (n_per // 2)
        ks += [0.0] * (n_per // 2)
        n_ties += n_per // 2
    state = rng.bit_generator.state
    X0 = K.ladder_rows(rng, coef, intercept, tune, tops, [0.0] * len(tops), kind, anchor)
    beta = K.linear_beta(X0.astype(np.float64), coef, intercept)
    rng.bit_generator.state = state
    X = K.ladder_rows(rng, coef, intercept, tune, tops, [k * b for k, b in zip(ks, beta)], kind, anchor)
    Xf = X.astype(np.float64)
    want, margin = K.exact_linear(Xf, coef, intercept)
    beta = K.linear_beta(Xf, coef, intercept)
    ties = np.arange(len(tops) - n_ties, len(tops))
    return coef, intercept, X, want, margin, beta, ties, np.array([tops[i][0] for i in ties], np.int32)


def run_rungs(fails, tag, predict, X, want, margin, beta, ties, tie_want, path, flagged=True):
    """Predict each rung as its own batch; returns (inside rows, inside rows with a label other than the exact one)."""
    n_in = n_in_wrong = 0
    for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
        if rows.size == 0:
            fails.append(f"{tag}: no planted rows in the {rung} batch")
            continue
        got, st = predict(X[rows])
        if st["path"] != path:
            fails.append(f"{tag} {rung}: path {st['path']} != {path}")
        if flagged and rung != "certain" and st["n_flagged"] < rows.size:
            fails.append(f"{tag} {rung}: n_flagged {st['n_flagged']} < {rows.size} planted near-ties")
        pos = np.searchsorted(rows, ties)
        hit = (pos < rows.size) & (rows[np.minimum(pos, rows.size - 1)] == ties)
        lower = (pos[hit], tie_want[hit]) if hit.any() else None
        wrong = check_batch(fails, tag, rung, got, st, want[rows], lower)
        if rung == "inside":
            n_in += rows.size
            n_in_wrong += wrong
    return n_in, n_in_wrong


LINEAR_TILE = [(F, C, b) for F in (1, 32, 33, 64, 65) for C, b in ((2, True), (2, False), (3, False), (10, False), (16, False))
               if not (F < C + 2 and not b)]


TILE_FIELDS = ("coef", "intercept", "X", "want", "margin", "beta", "ties", "tie_want")


def tile_cases():
    """(tag, ladder case) of every tile-kernel shape; F = 784 takes the separate re-score kernel with W in shared
    memory (in both modes), under PDL."""
    cases = [(f"tile F={F} C={C}{' binary' if b else ''}", ladder_case(F, C, b, seed=F * 31 + C)) for F, C, b in LINEAR_TILE]
    return cases + [("tile F=784 C=10", ladder_case(784, 10, False, seed=7, n_per=8))]


def linear_tile_report(path):
    """Tile kernel + the fp64 stage of this process's re-score mode, staged float64 batches (path 1), on the cases
    tile_cases() saved to `path` (built once, shared by both re-score modes)."""
    from unionml_b200.engine import Engine

    eng = Engine(0)
    fails = []
    tot_in = tot_wrong = 0
    with np.load(path) as z:
        for i, tag in enumerate(z["tags"]):
            coef, intercept, X, want, margin, beta, ties, tie_want = (z[f"{k}{i}"] for k in TILE_FIELDS)
            m = eng.load_linear(coef, intercept)
            n_in, n_wrong = run_rungs(fails, str(tag), lambda x: eng.predict(m, eng.stage(x), exact=True), X, want,
                                      margin, beta, ties, tie_want, path=1)
            tot_in += n_in
            tot_wrong += n_wrong
    print(f"inside rows {tot_in}, float64 label differs from the exact one on {tot_wrong}")
    if tot_wrong < tot_in // 10:
        fails.append(f"no teeth: only {tot_wrong} of {tot_in} inside rows got a non-exact label")
    return fails


@pytest.fixture(scope="module")
def tile_cases_file(tmp_path_factory):
    cases = tile_cases()
    arrays = {f"{k}{i}": v for i, (_, case) in enumerate(cases) for k, v in zip(TILE_FIELDS, case)}
    path = tmp_path_factory.mktemp("f64_stage") / "tile_cases.npz"
    np.savez(path, tags=np.array([t for t, _ in cases]), **arrays)
    return path


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_linear_tile_routes(mode, tile_cases_file):
    run_report("linear_tile_report", {"UML_B200_RESCORE_MODE": mode}, repr(str(tile_cases_file)))


def test_linear_generic_path(engine):
    """C > 16: every row through rescore_f64_kernel.  Ties and near-ties across the 16-class groups (3 vs 19, 15 vs
    16, later group on top); F = 640 at C = 40 does not fit W in shared memory (smem_weights = 0)."""
    # launch_rescore_f64 stages W and b in shared memory only if (F * w64_stride + 2 C) doubles fit in 200 KiB
    stride = lambda C: 2 * ((C + 1) // 2 + (1 - (C + 1) // 2 % 2))  # noqa: E731  (linear_w64_stride)
    assert (640 * stride(40) + 2 * 40) * 8 > 200 * 1024 >= (48 * stride(40) + 2 * 40) * 8
    fails = []
    for F, C, dups, n_per in ((24, 17, [(15, 16)], 12), (48, 40, [(3, 19), (15, 16)], 12), (640, 40, [(3, 19), (15, 16)], 4)):
        coef, intercept, X, want, margin, beta, ties, tie_want = ladder_case(F, C, False, seed=F + C, dups=dups, n_per=n_per)
        m = engine.load_linear(coef, intercept)
        run_rungs(fails, f"generic F={F} C={C}", lambda x: engine.predict(m, engine.stage(x), exact=True), X, want,
                  margin, beta, ties, tie_want, path=2, flagged=False)
    assert not fails, "\n".join(fails)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def test_linear_online_path(engine):
    """Path 4 (<= 64 rows, linear_small_kernel): 1, 7 and 64 rows, through Engine.predict_host and linear_argmax."""
    from sklearn.linear_model import LogisticRegression

    from unionml_b200 import predictors

    fails = []
    for F, C, binary in ((33, 10, False), (8, 2, True), (40, 20, False)):
        coef, intercept, X, want, margin, beta, ties, tie_want = ladder_case(F, C, binary, seed=3 * F + C)
        m = engine.load_linear(coef, intercept)
        est = LogisticRegression()
        est.coef_, est.intercept_, est.n_features_in_ = coef, intercept, F
        est.classes_ = np.arange(max(2, coef.shape[0]), dtype=np.float64)
        for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
            for n in (1, 7, 64):
                sub = rows[:n]
                if sub.size < n:
                    continue
                got, st = engine.predict_host(m, X[sub], exact=True)
                if st["path"] != 4:
                    fails.append(f"online F={F}: path {st['path']}")
                check_batch(fails, f"online F={F} C={C} n={n}", rung, got, st, want[sub])
                lab = np.asarray(predictors.linear_argmax(est, pd.DataFrame(X[sub]))).astype(np.int32)
                st2 = dict(st, n_ambiguous=predictors.last_ambiguous_rows())
                check_batch(fails, f"linear_argmax F={F} C={C} n={n}", rung, lab, st2, want[sub])
    assert not fails, "\n".join(fails)


def test_linear_sources(engine):
    """The stage reads each source as the caller passed it: float64 in C and F order and int32 / int64 through SrcView
    (predict_host), the keep_f64 copy of a resident batch, and fp32 rows."""
    fails = []
    F, C = 48, 10
    # int32: a tuning feature can only move a margin by whole units, so an anchor (2^30 x 2^30 in every class) makes
    # beta ~ 2^11 and the ladder reaches inside it; int64 values ~ 2^58 give beta ~ 2^6 on their own
    for kind, wexp, anchor in (("f64", (-20, 20), None), ("i32", (-26, -12), 2.0**30), ("i64", (-22, -10), None)):
        coef, intercept, X, want, margin, beta, ties, tie_want = ladder_case(F, C, False, seed=11, kind=kind, wexp=wexp,
                                                                             n_per=12, anchor=anchor)
        for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
            inside_near = rung == "inside" and np.setdiff1d(rows, ties).size == 0
            if rows.size == 0 or inside_near:
                fails.append(f"{kind}: no planted {'near-ties' if inside_near else 'rows'} in the {rung} batch")
        m = engine.load_linear(coef, intercept)
        routes = {"predict_host(C)": lambda x: engine.predict_host(m, np.ascontiguousarray(x), exact=True),
                  "predict_host(F)": lambda x: engine.predict_host(m, np.asfortranarray(x), exact=True)}
        if kind == "f64":
            routes["stage(keep_f64)"] = lambda x: engine.predict(m, engine.stage(x, keep_f64=True), exact=True)
        for name, fn in routes.items():
            pad = lambda x: np.concatenate([x] * max(1, -(-65 // x.shape[0])))[: max(65, x.shape[0])]  # noqa: E731
            for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
                if rows.size == 0:
                    continue
                xs = pad(X[rows])  # > 64 rows: the chunk pipeline, not the online kernel
                idx = np.concatenate([rows] * max(1, -(-65 // rows.size)))[: xs.shape[0]]
                got, st = fn(xs)
                if st["path"] != 1:
                    fails.append(f"{kind} {name}: path {st['path']}")
                check_batch(fails, f"{kind} {name}", rung, got, st, want[idx])
    # fp32 rows: the stage scores float64(x32); near-ties from a 32-bit tuning feature cannot reach float64 resolution,
    # so the rows are plain heavy-cancellation rows, measured in Fractions and split by their margins
    rng = np.random.default_rng(5)
    coef = K.spread64(rng, (C, F))
    intercept = K.spread64(rng, C)
    coef[C - 1], intercept[C - 1] = coef[0], intercept[0]  # class C-1 ties class 0 exactly on every row
    X32 = K.spread64(rng, (400, F)).astype(np.float32)
    want, margin = K.exact_linear(X32.astype(np.float64), coef, intercept)
    beta = K.linear_beta(X32.astype(np.float64), coef, intercept)
    m = engine.load_linear(coef, intercept)
    for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
        if rows.size:
            got, st = engine.predict(m, engine.stage(X32[rows]), exact=True)
            check_batch(fails, "fp32 rows", rung, got, st, want[rows])
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------
# the bound factor, on data whose float64 arithmetic is exact: an anchor feature adds 2^40 to classes 0 and 1 alike,
# so beta ~ 2^-9 while the row's margin is set exactly by a 2^-12-grid tuning feature
# ---------------------------------------------------------------------------------------------------------------
INSIDE_K = (0.6, 0.75, 0.9)
CERTAIN_K = (1.3, 1.6, 3.0)


def exact_factor_case(F, C):
    coef = np.zeros((C, F))
    coef[:2, 0] = 2.0**20
    coef[0, 1] = 2.0**-12
    intercept = np.full(C, -(2.0**41))
    intercept[:2] = 0.0
    x0 = np.zeros(F)
    x0[0] = 2.0**20
    beta = float(K.linear_beta(x0[None, :], coef, intercept)[0])  # the tuning feature moves beta by < 2^-40
    rows, ks = [], []
    for k in INSIDE_K + CERTAIN_K:
        for sign in (1, -1):
            x = x0.copy()
            x[1] = sign * np.ceil(k * beta * 2.0**12)
            rows.append(x)
            ks.append(k)
    X = np.array(rows)
    want, margin = K.exact_linear(X, coef, intercept)
    return coef, intercept, X, want, margin, K.linear_beta(X, coef, intercept), np.array(ks)


def exact_factor_report():
    from unionml_b200.engine import Engine

    eng = Engine(0)
    fails = []
    for F, C, path in ((32, 3, 1), (64, 10, 1), (784, 10, 1), (40, 20, 2)):
        coef, intercept, X, want, margin, beta, ks = exact_factor_case(F, C)
        r = margin / beta  # the 2^-12 grid rounds each margin up by < 0.06 beta
        assert np.all((r >= ks) & (r <= ks + 0.06)) and np.all(r[ks < 1] < 0.97), (r, ks)
        m = eng.load_linear(coef, intercept)
        for rung, sel in (("inside", ks < 1), ("certain", ks > 1)):
            rows = np.flatnonzero(sel)
            got, st = eng.predict(m, eng.stage(X[rows]), exact=True)
            if st["path"] != path:
                fails.append(f"F={F}: path {st['path']}")
            wrong = int((got != want[rows]).sum())
            if rung == "inside" and st["n_ambiguous"] != rows.size:
                fails.append(f"F={F} C={C}: margins 0.6..0.9 beta, n_ambiguous {st['n_ambiguous']} != {rows.size}")
            if rung == "certain" and (st["n_ambiguous"] or wrong):
                fails.append(f"F={F} C={C}: margins 1.3..3 beta, n_ambiguous {st['n_ambiguous']}, wrong {wrong}")
            got, st = eng.predict_host(m, X[rows], exact=True)  # online path
            if rung == "inside" and st["n_ambiguous"] != rows.size:
                fails.append(f"online F={F} C={C}: n_ambiguous {st['n_ambiguous']} != {rows.size}")
            if rung == "certain" and st["n_ambiguous"]:
                fails.append(f"online F={F} C={C}: certified rows counted ({st['n_ambiguous']})")
    return fails


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_linear_bound_factor_exact_data(mode):
    run_report("exact_factor_report", {"UML_B200_RESCORE_MODE": mode})


# ---------------------------------------------------------------------------------------------------------------
# MLP: hidden unit 0 = x0 - x1 + x2 with x0 = x1 = 2^20 (it cancels, so herr w2sum dominates the bound), logit 0 =
# h0, logit 1 = b2_1, the others -1; the margin h0 - b2_1 is exact.  Class 2 copies class 0 in the tie model.
# ---------------------------------------------------------------------------------------------------------------
def mlp_exact_case(F, H, C, tie=False):
    w1 = np.zeros((H, F), np.float32)
    w1[0, :3] = [1.0, -1.0, 1.0]
    b1 = np.zeros(H, np.float32)
    w2 = np.zeros((C, H), np.float32)
    w2[0, 0] = 1.0
    b2 = np.full(C, -1.0, np.float32)
    b2[0], b2[1] = 0.0, 2.0**-25
    if tie:
        w2[C - 1], b2[C - 1] = w2[0], b2[0]
    x0 = np.zeros(F, np.float32)
    x0[:3] = [2.0**20, 2.0**20, 2.0**-25]
    beta = float(K.mlp_beta(x0[None, :], w1, b1, w2, b2)[0])
    rows, ks = [], []
    for k in (INSIDE_K + CERTAIN_K if not tie else (0.0, 0.5, 3.0, 10.0)):
        for sign in (1, -1):
            x = x0.copy()
            x[2] = np.float32(2.0**-25 + sign * k * beta)
            x[2] = (np.array([x[2]], np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)[0]  # tf32
            rows.append(x)
            ks.append(k)
    X = np.array(rows, np.float32)
    want, margin = K.exact_mlp(X, w1, b1, w2, b2)
    return (w1, b1, w2, b2), X, want, margin, K.mlp_beta(X, w1, b1, w2, b2)


def mlp_report():
    from unionml_b200.engine import Engine

    eng = Engine(0)
    fails = []
    for F, H, C, tc, path in ((64, 32, 10, "1", 5), (64, 32, 10, "0", 3), (32, 16, 3, "1", 5), (32, 16, 3, "0", 3),
                              (40, 24, 5, "1", 2)):
        os.environ["UML_B200_MLP_TC"] = tc
        for tie in (False, True):
            net, X, want, margin, beta = mlp_exact_case(F, H, C, tie)
            m = eng.load_mlp(*net)
            tag = f"mlp {F}-{H}-{C} tc={tc}{' tie' if tie else ''}"
            for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
                if not tie:  # the exact data: inside means 0.6..0.9 beta here, certain 1.3..3 beta
                    rows = np.flatnonzero(margin < beta) if rung == "inside" else (
                        np.flatnonzero(margin > beta) if rung == "certain" else np.array([], np.int64))
                if rows.size == 0:
                    continue
                counts = [rows.size] if path != 2 else [1, 2, 3, 5, 9, 10, 11]  # generic: 4 rows per pass, ragged ends
                for n in counts:
                    sub = np.resize(rows, n)
                    got, st = eng.predict_mlp(m, eng.stage(X[sub]), exact=True)
                    if st["path"] != path:
                        fails.append(f"{tag}: path {st['path']} != {path}")
                    if path != 2 and rung != "certain" and st["n_flagged"] < n:
                        fails.append(f"{tag} {rung}: n_flagged {st['n_flagged']} < {n}")
                    ties = np.flatnonzero(margin[sub] == 0) if tie else np.array([], np.int64)
                    lower = (ties, np.zeros(ties.size, np.int32)) if ties.size else None
                    check_batch(fails, f"{tag} n={n}", rung, got, st, want[sub], lower)
    return fails


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_mlp_routes(mode):
    """mlp_rescore_f64_kernel behind the CUDA-core kernel (path 3), the tensor-core kernel's re-score (path 5) as the
    queue and as a second kernel, and the generic shapes (path 2) at ragged row counts."""
    run_report("mlp_report", {"UML_B200_MLP_RESCORE_MODE": mode})


# ---------------------------------------------------------------------------------------------------------------
# hole 1: float64 products below DBL_MIN; hole 2: finite features whose float64 scores overflow
# ---------------------------------------------------------------------------------------------------------------
def pad_classes(coef, intercept, C):
    """Extra classes with zero weights and bias: they score 0 and change no bound."""
    c2 = np.zeros((C, coef.shape[1]))
    c2[: coef.shape[0]] = coef
    b2 = np.zeros(C)
    b2[: intercept.size] = intercept
    return c2, b2


def edge_routes(eng, coef, intercept, X, path):
    """Labels, stats and the path each route must take: a resident batch and > 64 host rows take `path` (1: tile
    kernel, 2: generic), <= 64 host rows the online kernel (4)."""
    m = eng.load_linear(coef, intercept)
    return {
        "stage": (eng.predict(m, eng.stage(X), exact=True), path),
        "predict_host": (eng.predict_host(m, np.concatenate([X] * 70), exact=True), path),
        "online": (eng.predict_host(m, X, exact=True), 4),
    }


def underflow_report():
    from unionml_b200.engine import Engine

    eng = Engine(0)
    fails = []
    for binary in (False, True):
        coef, intercept, x = K.underflow_case(binary)
        X = np.repeat(x[None, :], 5, axis=0)
        want = K.exact_linear(X, coef, intercept)[0]
        models = [("tile", coef, intercept, 1)] + ([] if binary else [("generic", *pad_classes(coef, intercept, 17), 2)])
        for name, c, b, path in models:
            for route, ((got, st), want_path) in edge_routes(eng, c, b, X, path).items():
                w = np.resize(want, got.size)
                if st["path"] != want_path:
                    fails.append(f"{name} {route}: path {st['path']}")
                if (got != w).any() and st["n_ambiguous"] < int((got != w).sum()):
                    fails.append(f"underflow{' binary' if binary else ''} {name} {route}: got {got[:3].tolist()} "
                                 f"want {w[:3].tolist()}, n_ambiguous {st['n_ambiguous']}")
    return fails


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_float64_underflow(mode):
    run_report("underflow_report", {"UML_B200_RESCORE_MODE": mode})


OVERFLOW = {  # (coef rows over x = [1e300, 1e300], what float64 makes of the scores)
    "inf_one_class": [[1e10, 0.0], [1.0, 0.0], [-1.0, 0.0]],
    "inf_two_classes": [[1.0, 0.0], [1e10, 0.0], [1e10, 1.0]],
    "nan_one_class": [[1.0, 0.0], [1e10, -1e10], [-1.0, 0.0]],
    "nan_two_classes": [[1.0, 0.0], [1e10, -1e10], [-1e10, 1e10]],
    "binary_inf": [[1e10, 0.0]],
    "binary_minus_inf": [[-1e10, 0.0]],
    "binary_nan": [[1e10, -1e10]],
}


def overflow_report():
    from sklearn.linear_model import LogisticRegression

    from unionml_b200.engine import Engine

    eng = Engine(0)
    fails = []
    X = np.full((3, 2), 1e300)
    for name, rows in OVERFLOW.items():
        coef = np.array(rows)
        intercept = np.zeros(coef.shape[0])
        est = LogisticRegression()
        est.coef_, est.intercept_, est.n_features_in_ = coef, intercept, 2
        est.classes_ = np.arange(max(2, coef.shape[0]))
        with np.errstate(all="ignore"):
            want = est.predict(X).astype(np.int32)
        models = [("tile", coef, intercept, 1)] + (
            [] if coef.shape[0] == 1 else [("generic", *pad_classes(coef, intercept, 17), 2)])
        for mname, c, b, path in models:
            for route, ((got, st), want_path) in edge_routes(eng, c, b, X, path).items():
                w = np.resize(want, got.size)
                if st["path"] != want_path:
                    fails.append(f"{name} {mname} {route}: path {st['path']} != {want_path}")
                if (got != w).any() or st["n_ambiguous"] != got.size:
                    fails.append(f"{name} {mname} {route}: got {got[:3].tolist()} want {w[:3].tolist()}, n_ambiguous "
                                 f"{st['n_ambiguous']} of {got.size}")
    return fails


@pytest.mark.parametrize("mode", ["queue", "kernel"])
def test_float64_overflow(mode):
    run_report("overflow_report", {"UML_B200_RESCORE_MODE": mode})


# ---------------------------------------------------------------------------------------------------------------
# hole 3: Pipeline(StandardScaler, LR) folded into w' = w / scale_, b' = b - sum_f mean_f w'_f
# ---------------------------------------------------------------------------------------------------------------
def test_scaler_fold(engine):
    from sklearn.linear_model import LogisticRegression
    from sklearn.pipeline import Pipeline

    from unionml_b200 import predictors

    mean, scale, coef, intercept = K.fold_model()
    rng = np.random.default_rng(9)
    sc, X1 = K.fold_rows(rng, mean, scale, coef, intercept, [1.0])
    beta = float(K.fold_beta(sc, X1, coef, intercept)[0])
    ks = [s * k for k in (0.02, 0.05, 0.1, 0.2, 0.5, 1.0, 2.0, 5.0, 10.0) for s in (1, -1) for _ in range(4)]
    sc, X = K.fold_rows(rng, mean, scale, coef, intercept, [k * beta for k in ks])
    want, margin = K.fold_truth(sc, X, coef, intercept)
    beta = K.fold_beta(sc, X, coef, intercept)
    lr = LogisticRegression()
    lr.coef_, lr.intercept_, lr.n_features_in_, lr.classes_ = coef, intercept, coef.shape[1], np.array([0.0, 1.0])
    pipe = Pipeline([("scaler", sc), ("clf", lr)])
    m = engine.load_linear(coef, intercept)
    m.set_affine(shift=sc.mean_, scale=1.0 / sc.scale_)
    fails = []
    for rung, rows in zip(("certain", "inside", "straddle"), K.rungs(margin, beta)):
        if rows.size == 0:
            continue
        got, st = engine.predict_host(m, X[rows], exact=True)
        check_batch(fails, "predict_host after set_affine", rung, got, st, want[rows])
        lab = np.asarray(predictors.linear_argmax(pipe, pd.DataFrame(X[rows]))).astype(np.int32)
        stats = predictors.last_call_stats()
        if predictors.last_ambiguous_rows() != stats.get("n_ambiguous"):
            fails.append(f"{rung}: last_ambiguous_rows {predictors.last_ambiguous_rows()} != {stats.get('n_ambiguous')}")
        check_batch(fails, "linear_argmax(Pipeline, DataFrame)", rung, lab, stats, want[rows])
    assert not fails, "\n".join(fails)
