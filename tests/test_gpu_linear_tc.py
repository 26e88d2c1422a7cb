"""The tensor-core schedule of the linear tile kernel (kHalfMma) against the fp32 route and the CUDA-core fp16 route.

A staged batch whose fp16 copy holds no negative value is scored on the tensor cores in EXACT mode with the in-kernel
queue.  Rows the tensor-core guard does not certify are replayed on the fp32 route's arithmetic by the re-score warp,
so labels must be byte-equal to the fp32 route (UML_B200_COMPACT_ROWS=0) and to the CUDA-core fp16 schedule
(UML_B200_LINEAR_TC=0), and n_flagged (the rows sent to float64) equal, for every class count 2..16 and widths
1..64, at row counts around one and two m64 blocks, one ring item (256 rows) and a few items.  Operand edges: fp16
features 65504 and subnormal fp16 features, weights spread over 2^+-60 (lo pieces subnormal or 0), a class whose
weights all fall below fp16 after scaling.  Dispatch: a batch with a -1 keeps the CUDA-core schedule, a -0 batch does
not need to.  UML_B200_LINEAR_TC=1 makes a call fail unless it takes the tensor-core schedule, so every comparison
below knows that schedule ran.  The existing fp16-schedule workers run again with UML_B200_LINEAR_TC=0, so the
CUDA-core schedule keeps its queue, uint8-peer, ring-floor and graph-replay coverage.
"""
import os
import subprocess
import sys

from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there
    pytest.skip("needs a CUDA device", allow_module_level=True)

ROOT = Path(__file__).resolve().parent.parent
ROWS = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1025, 20_001)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def tie_prone(seed, C, F):
    """Weights on a 1/4 grid (integer rows then give many exact and near ties, so EXACT mode flags rows)."""
    rng = np.random.default_rng(seed)
    n = 1 if C == 2 else C  # C = 2: sklearn's binary layout (one coef_ row)
    return np.round(rng.standard_normal((n, F)) * 4) / 4, np.round(rng.standard_normal(n) * 4) / 4


def three_routes(engine, monkeypatch, model, b):
    monkeypatch.delenv("UML_B200_COMPACT_ROWS", raising=False)
    monkeypatch.delenv("UML_B200_LINEAR_TC", raising=False)
    monkeypatch.setenv("UML_B200_LINEAR_TC", "1")  # fails unless the tensor-core schedule runs
    got_t, st_t = engine.predict(model, b, exact=True)
    monkeypatch.setenv("UML_B200_LINEAR_TC", "0")
    got_h, st_h = engine.predict(model, b, exact=True)
    monkeypatch.delenv("UML_B200_LINEAR_TC")
    monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
    got_f, st_f = engine.predict(model, b, exact=True)
    monkeypatch.delenv("UML_B200_COMPACT_ROWS")
    return (got_t, st_t), (got_h, st_h), (got_f, st_f)


def assert_same(routes, what):
    (got_t, st_t), (got_h, st_h), (got_f, st_f) = routes
    assert got_t.tobytes() == got_h.tobytes() == got_f.tobytes(), (what, int((got_t != got_f).sum()))
    assert st_t["n_flagged"] == st_h["n_flagged"] == st_f["n_flagged"], (what, st_t, st_f)
    assert st_t["kernel_launches"] == st_f["kernel_launches"], (what, st_t, st_f)
    assert st_t["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4


@pytest.mark.parametrize("C", list(range(2, 17)))
@pytest.mark.parametrize("F", [1, 16, 32, 33, 64])
def test_tc_route_equals_fp32_and_half_routes(engine, monkeypatch, F, C):
    model = engine.load_linear(*tie_prone(4000 + 37 * F + C, C, F))
    X = np.random.default_rng(F * 211 + C).integers(0, 17, size=(ROWS[-1], F)).astype(np.float32)
    for rows in ROWS:
        assert_same(three_routes(engine, monkeypatch, model, engine.stage(X[:rows])), rows)


def test_operand_edges(engine, monkeypatch):
    rng = np.random.default_rng(7)
    C, F, n = 10, 64, 4097
    W = rng.standard_normal((C, F)) * np.exp2(rng.integers(-60, 61, size=(C, F)))
    W[3] = rng.standard_normal(F) * 2.0**-80  # a class whose every weight falls below fp16 after scaling
    b = rng.standard_normal(C)
    X = rng.integers(0, 17, size=(n, F)).astype(np.float32)
    X[::7, 5] = 65504.0
    X[1::3, 9] = np.float32(2.0**-24) * rng.integers(1, 1024, size=X[1::3, 9].shape)  # fp16 subnormals
    model = engine.load_linear(W, b)
    assert_same(three_routes(engine, monkeypatch, model, engine.stage(X)), "edges")
    from oracle import linear as olin

    got, _ = engine.predict(model, engine.stage(X), exact=True)
    want = olin.predict_indices(olin.decision_function(X.astype(np.float64), W, b))
    assert np.array_equal(got, want)


def test_planted_near_ties(engine, monkeypatch):
    """Integer weights and rows: many rows tie exactly or nearly, so tier 1 leaves rows to the replay and the replay
    leaves some to float64 - both must match the other routes."""
    rng = np.random.default_rng(11)
    C, F, n = 10, 64, 70_001
    W = rng.integers(-3, 4, size=(C, F)).astype(np.float64)
    W[:, :8] += rng.integers(-2, 3, size=(C, 8)) * 2.0**-20  # margins of a few 2^-20: near the fp32 guard
    b = np.zeros(C)
    X = rng.integers(0, 3, size=(n, F)).astype(np.float32)
    model = engine.load_linear(W, b)
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, "near ties")
    assert routes[0][1]["n_flagged"] > 0


def test_all_ties_backed_up_queue(engine, monkeypatch):
    """Every row ties: the queue backs up, the scoring warps wait for room, and every row is counted."""
    C, F, n = 4, 64, 300_000
    W = np.ones((C, F))
    X = np.random.default_rng(3).integers(0, 17, size=(n, F)).astype(np.float32)
    model = engine.load_linear(W, np.zeros(C))
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, "ties")
    assert routes[0][1]["n_flagged"] == n
    assert not routes[0][0].any()


def test_ring_floor(engine, monkeypatch):
    model = engine.load_linear(*tie_prone(5, 10, 64))
    X = np.random.default_rng(5).integers(0, 17, size=(50_001, 64)).astype(np.float32)
    monkeypatch.setenv("UML_B200_STAGES", "1")  # raised to the schedule's floor (one stage per warpgroup)
    assert_same(three_routes(engine, monkeypatch, model, engine.stage(X)), "floor")


def test_sign_dispatch(engine, monkeypatch):
    model = engine.load_linear(*tie_prone(9, 10, 64))
    X = np.random.default_rng(9).integers(0, 17, size=(5_000, 64)).astype(np.float32)
    X[4_321, 17] = -0.0
    assert_same(three_routes(engine, monkeypatch, model, engine.stage(X)), "-0")  # -0 takes the tensor cores
    X[4_321, 17] = -1.0
    b = engine.stage(X)
    monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
    with pytest.raises(Exception):
        engine.predict(model, b, exact=True)
    monkeypatch.delenv("UML_B200_LINEAR_TC")
    got, st = engine.predict(model, b, exact=True)  # the CUDA-core fp16 schedule
    monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
    want, st_f = engine.predict(model, b, exact=True)
    assert got.tobytes() == want.tobytes() and st["n_flagged"] == st_f["n_flagged"] and st["x_elem_bytes"] == 2


THR64 = 2 * 68 * 2.0**-24 * (1 + 64 * 2.0**-21) * 1.0001  # linear_margin_thr(64)


@pytest.mark.parametrize("ratio,flagged", [(3.0, False), (0.5, True)])
def test_planted_margins(engine, monkeypatch, ratio, flagged):
    """Rows of 32 ones (feature 0 among them) and classes [1...1], [1 + d, 1...1], 0: every score is exact in fp32 and
    the margin is d = ratio thr A.  At 3 thr the fp32 route certifies every row, but tier 1 cannot (its factor kappa is
    > 2.5 thr + 2 x 4 x 64u, about 6 thr): every row goes through the replay, which must certify it, so no row is
    counted.  At 0.5 thr the fp32 route flags every row: all are counted, with float64 labels."""
    C, F, n = 3, 64, 20_000
    rng = np.random.default_rng(17)
    X = np.zeros((n, F), dtype=np.float32)
    X[:, 0] = 1
    for i in range(n):
        X[i, 1 + rng.choice(F - 1, 31, replace=False)] = 1
    d = round(ratio * THR64 * 32 * 2**20) * 2.0**-20
    W = np.ones((C, F))
    W[1, 0] += d
    W[2] = 0
    model = engine.load_linear(W, np.zeros(C))
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, ratio)
    assert routes[0][1]["n_flagged"] == (n if flagged else 0)
    assert np.all(routes[0][0] == 1)


@pytest.mark.parametrize("module,marker", [("test_gpu_linear_half_tiles", "half tiles ok"),
                                           ("test_gpu_linear_half_consumers", "half consumers ok")])
@pytest.mark.parametrize("stages,graph", [("", "1"), ("1", "")])
def test_cuda_core_fp16_schedule_queue_peers_graph(tmp_path, module, marker, stages, graph):
    import importlib

    script = tmp_path / "worker.py"
    script.write_text(importlib.import_module(f"tests.{module}")._WORKER)
    env = dict(os.environ, UML_ROOT=str(ROOT), UML_B200_RESCORE_MODE="queue", UML_TEST_GRAPH=graph,
               UML_B200_LINEAR_TC="0")
    env.pop("UML_B200_COMPACT_ROWS", None)
    if stages:
        env["UML_B200_STAGES"] = stages
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and marker in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_full_cfg2_batch(engine):
    """bench.py's cfg 2: 10M digits rows and the golden model, labels equal to float64 on a sample of rows, and
    n_flagged equal to the fp32 route's."""
    sys.path.insert(0, str(ROOT))
    import bench

    z = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    coef, intercept = z["coef"], z["intercept"]
    n = 10_000_000
    X = np.empty((n, 64), dtype=np.float32)
    bench.digits_rows(0, n, X)
    model = engine.load_linear(coef, intercept, z["classes"])
    b = engine.stage(X)
    os.environ["UML_B200_LINEAR_TC"] = "1"
    try:
        got, st = engine.predict(model, b, exact=True)
    finally:
        del os.environ["UML_B200_LINEAR_TC"]
    os.environ["UML_B200_COMPACT_ROWS"] = "0"
    try:
        want_f, st_f = engine.predict(model, b, exact=True)
    finally:
        del os.environ["UML_B200_COMPACT_ROWS"]
    assert got.tobytes() == want_f.tobytes() and st["n_flagged"] == st_f["n_flagged"]
    rows = np.random.default_rng(0).choice(n, 200_000, replace=False)
    s = X[rows].astype(np.float64) @ coef.T.astype(np.float64) + intercept
    assert np.array_equal(got[rows], np.argmax(s, axis=1))
