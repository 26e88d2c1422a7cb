"""Tier 2 of the linear tile kernel's tensor-core schedules (kByteMma, kHalfMma) settles the rows tier 1 leaves in
batches of up to 32, one row per lane: a batch starts once 32 rows are queued, and the rows left when every scoring
warp has published are split evenly over the warps that drain the queue.

A 512-row batch (two tiles) holds k planted near-ties, k in {1, 31, 32, 33, 65, 200, 512}: one batch short of full,
full, one over, two full and one over, and every row queued.  Classes 0 and 1 share their weights except feature 1,
where class 1 has 2^-12 more, and both win by far on rows that light feature 0.  A planted row's margin is then
2^-12 x_1: an exact tie at x_1 = 0 and a margin under the fp32 route's threshold at x_1 = 20 (float64 settles both),
and margins between that threshold and tier 1's at x_1 in {100, 120, 140} (the fp32 replay certifies them).  Tier 1
leaves every planted row.  Labels and n_flagged must equal the fp32 route's on both schedules, and the replay must
certify some rows and send others to float64 (UML_B200_TC_REPLAY=0 counts what tier 1 left).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests import tc_guard_cases as tg  # noqa: E402

C, F, N = 10, 64, 512
X1 = (0, 20, 140, 120, 100)  # per planted row, in turn: float64, float64, then three the replay certifies
ROUTES = {"byte": ({}, 1), "half": ({"UML_B200_COMPACT_ROWS": "2"}, 2)}
ENV = ("UML_B200_COMPACT_ROWS", "UML_B200_LINEAR_TC", "UML_B200_TC_REPLAY")


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def near_tie_case(k, seed):
    rng = np.random.default_rng(seed)
    coef = np.round(rng.standard_normal((C, F)) * 1024) / 4096  # fine enough that other rows are no near-ties
    coef[:, :2] = 0.0
    coef[1] = coef[0]
    coef[0, 0] = coef[1, 0] = 8.0
    coef[1, 1] = 2.0**-12
    intercept = np.round(rng.standard_normal(C) * 4) / 4
    intercept[0] = intercept[1] = -64.0
    X = rng.integers(0, 17, size=(N, F)).astype(np.float32)
    X[:, :2] = 0.0
    rows = np.sort(rng.choice(N, size=k, replace=False))
    X[rows, 0] = 255.0
    X[rows, 1] = np.array(X1, np.float32)[np.arange(k) % len(X1)]
    return coef, intercept, X, rows


def run(engine, monkeypatch, model, b, route=None, replay=True):
    """One EXACT predict: the fp32 route (route None) or a tensor-core schedule, with or without tier 2's replay."""
    for key in ENV:
        monkeypatch.delenv(key, raising=False)
    if route is None:
        monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
        read = 4
    else:
        env, read = ROUTES[route]
        monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
        if not replay:
            monkeypatch.setenv("UML_B200_TC_REPLAY", "0")
        for key, v in env.items():
            monkeypatch.setenv(key, v)
    try:
        got, st = engine.predict(model, b, exact=True)
    finally:
        for key in ENV:
            monkeypatch.delenv(key, raising=False)
    assert st["x_read_bytes"] == read, st
    return got, st


def test_planted_rows_straddle_both_thresholds():
    """The planted rows sit where the docstring says: below tier 1's threshold, and on both sides of the fp32 route's."""
    coef, intercept, X, rows = near_tie_case(len(X1), 1)
    ops = tg.operands(coef, intercept)
    assert ops.eligible
    labels, margins = tg.truth(X[rows], coef, intercept)
    assert np.all(tg.verdicts(ops, X[rows], margins) == -1)
    a32 = ops.bias_bound + np.abs(X[rows]).astype(np.float64) @ ops.wt_bound
    over = margins / (ops.thr * a32)
    np.testing.assert_array_equal(over > 1.2, [False, False, True, True, True])
    assert np.all((over < 0.5) | (over > 1.2)), over
    np.testing.assert_array_equal(labels, [0, 1, 1, 1, 1])


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("k", [1, 31, 32, 33, 65, 200, 512])
def test_batches_match_fp32_route(engine, monkeypatch, k, route):
    coef, intercept, X, rows = near_tie_case(k, 100 + k)
    model = engine.load_linear(coef, intercept)
    b = engine.stage(X)
    want, st_f = run(engine, monkeypatch, model, b)
    got, st = run(engine, monkeypatch, model, b, route)
    np.testing.assert_array_equal(got, want)
    assert st["n_flagged"] == st_f["n_flagged"], (st, st_f)
    _, st_t1 = run(engine, monkeypatch, model, b, route, replay=False)
    assert st_t1["n_flagged"] >= k, st_t1  # tier 1 left every planted row
    fp64 = sum(1 for i in range(k) if X1[i % len(X1)] in (0, 20))
    assert st["n_flagged"] >= fp64
    if k >= 3:  # rows of both kinds: the replay certified some and sent the others to float64
        assert 0 < st["n_flagged"] < st_t1["n_flagged"], (st, st_t1)
