"""The byte schedule of the linear tile kernel (kByteMma) against the fp16 tensor-core schedule and the fp32 route.

A staged batch whose every value is an integer in [0, 255] gets a byte copy next to its fp16 copy, and in EXACT mode
with the in-kernel queue the tensor-core schedule reads the bytes, widened in registers to the f16 values kHalfMma
reads from the fp16 copy.  Labels must be byte-equal to kHalfMma (UML_B200_COMPACT_ROWS=2) and to the fp32 route
(UML_B200_COMPACT_ROWS=0), and n_flagged equal, for every class count 2..16 and widths 1..64, at row counts around one
ring item (256 rows), one claim group (3 x 256) and 1024, with ragged last tiles.  uml_stats.x_read_bytes says which
copy a call read (1, 2 or 4) and UML_B200_LINEAR_TC=1 makes a call fail unless it takes a tensor-core schedule, so every
comparison below knows which schedule ran.  Values: 0, 255 and -0.0 take the byte copy; 256 or 0.5 keep kHalfMma; -1
keeps the CUDA-core fp16 schedule.  The full cfg 2 batch is checked against float64 on every row.
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

from tests.test_gpu_linear_tc import tie_prone  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
ITEM = 256
ROWS = (1, 64, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 3 * 1024 + 77, 20_001)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def predict_env(engine, monkeypatch, model, b, **env):
    for k in ("UML_B200_COMPACT_ROWS", "UML_B200_LINEAR_TC"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return engine.predict(model, b, exact=True)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def three_routes(engine, monkeypatch, model, b):
    """(byte schedule, kHalfMma, fp32 route), each asserted to be the route it names."""
    byte = predict_env(engine, monkeypatch, model, b, UML_B200_LINEAR_TC="1")
    half = predict_env(engine, monkeypatch, model, b, UML_B200_COMPACT_ROWS="2", UML_B200_LINEAR_TC="1")
    fp32 = predict_env(engine, monkeypatch, model, b, UML_B200_COMPACT_ROWS="0")
    assert (byte[1]["x_read_bytes"], half[1]["x_read_bytes"], fp32[1]["x_read_bytes"]) == (1, 2, 4)
    return byte, half, fp32


def assert_same(routes, what):
    (got_b, st_b), (got_h, st_h), (got_f, st_f) = routes
    assert got_b.tobytes() == got_h.tobytes() == got_f.tobytes(), (what, int((got_b != got_f).sum()))
    assert st_b["n_flagged"] == st_h["n_flagged"] == st_f["n_flagged"], (what, st_b, st_h, st_f)
    assert st_b["kernel_launches"] == st_f["kernel_launches"], (what, st_b, st_f)
    # the byte schedule multiplies the fp16 values kHalfMma reads
    assert st_b["x_elem_bytes"] == st_h["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4


@pytest.mark.parametrize("C", list(range(2, 17)))
@pytest.mark.parametrize("F", [1, 16, 32, 33, 64])
def test_byte_route_equals_half_and_fp32_routes(engine, monkeypatch, F, C):
    model = engine.load_linear(*tie_prone(6000 + 37 * F + C, C, F))
    X = np.random.default_rng(F * 307 + C).integers(0, 17, size=(ROWS[-1], F)).astype(np.float32)
    for rows in ROWS:
        assert_same(three_routes(engine, monkeypatch, model, engine.stage(X[:rows])), rows)


def test_value_edges(engine, monkeypatch):
    """0, 255 and -0.0 in every feature position: the byte copy holds each at the place the f16 A fragment wants it."""
    from oracle import linear as olin

    rng = np.random.default_rng(23)
    C, F, n = 10, 64, 4_097
    W, b = rng.standard_normal((C, F)), rng.standard_normal(C)
    X = rng.integers(0, 256, size=(n, F)).astype(np.float32)
    X[0::5] = 0.0
    X[1::5] = 255.0
    X[2::5, rng.integers(0, F)] = -0.0
    X[3::5] = np.where(rng.random((len(X[3::5]), F)) < 0.5, 255.0, -0.0)
    model = engine.load_linear(W, b)
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, "edges")
    want = olin.predict_indices(olin.decision_function(X.astype(np.float64), W, b))
    assert np.array_equal(routes[0][0], want)


def test_one_hot_features_land_in_place(engine, monkeypatch):
    """Row f holds 255 in feature f alone and class c's weight is 1 on feature c only: row f's label is f, so a byte
    stored at the wrong position, or widened into the wrong half of an A register, gives a wrong label."""
    F = C = 16
    for f0 in (0, 16, 32, 48):
        W = np.zeros((C, 64))
        W[np.arange(C), f0 + np.arange(C)] = 1.0
        X = np.zeros((ITEM, 64), dtype=np.float32)
        X[np.arange(ITEM), f0 + np.arange(ITEM) % F] = 255.0
        model = engine.load_linear(W, np.zeros(C))
        routes = three_routes(engine, monkeypatch, model, engine.stage(X))
        assert_same(routes, f0)
        assert np.array_equal(routes[0][0], np.arange(ITEM) % F)


@pytest.mark.parametrize("value", [256.0, 0.5])
def test_fp16_values_keep_khalfmma(engine, monkeypatch, value):
    model = engine.load_linear(*tie_prone(9, 10, 64))
    X = np.random.default_rng(9).integers(0, 17, size=(5_000, 64)).astype(np.float32)
    X[4_321, 17] = value
    b = engine.stage(X)
    got, st = predict_env(engine, monkeypatch, model, b, UML_B200_LINEAR_TC="1")  # kHalfMma: no byte copy
    want, st_f = predict_env(engine, monkeypatch, model, b, UML_B200_COMPACT_ROWS="0")
    assert got.tobytes() == want.tobytes() and st["n_flagged"] == st_f["n_flagged"]
    assert st["x_elem_bytes"] == st["x_read_bytes"] == 2


def test_negative_value_keeps_cuda_core_schedule(engine, monkeypatch):
    model = engine.load_linear(*tie_prone(10, 10, 64))
    X = np.random.default_rng(10).integers(0, 17, size=(5_000, 64)).astype(np.float32)
    X[1_234, 40] = -1.0
    b = engine.stage(X)
    with pytest.raises(Exception):
        predict_env(engine, monkeypatch, model, b, UML_B200_LINEAR_TC="1")
    got, st = predict_env(engine, monkeypatch, model, b)
    want, st_f = predict_env(engine, monkeypatch, model, b, UML_B200_COMPACT_ROWS="0")
    assert got.tobytes() == want.tobytes() and st["n_flagged"] == st_f["n_flagged"]
    assert st["x_elem_bytes"] == st["x_read_bytes"] == 2


def test_fast_mode_keeps_cuda_core_schedule(engine, monkeypatch):
    """FAST mode has no tensor-core schedule: a batch with a byte copy reads its fp16 copy."""
    model = engine.load_linear(*tie_prone(12, 10, 64))
    X = np.random.default_rng(12).integers(0, 17, size=(3_000, 64)).astype(np.float32)
    b = engine.stage(X)
    got, st = engine.predict(model, b, exact=False)
    assert st["x_elem_bytes"] == st["x_read_bytes"] == 2
    _, st_e = engine.predict(model, b, exact=True)
    assert st_e["x_read_bytes"] == 1


def test_planted_near_ties(engine, monkeypatch):
    rng = np.random.default_rng(13)
    C, F, n = 10, 64, 70_001
    W = rng.integers(-3, 4, size=(C, F)).astype(np.float64)
    W[:, :8] += rng.integers(-2, 3, size=(C, 8)) * 2.0**-20  # margins of a few 2^-20: near the fp32 guard
    X = rng.integers(0, 3, size=(n, F)).astype(np.float32)
    model = engine.load_linear(W, np.zeros(C))
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, "near ties")
    assert routes[0][1]["n_flagged"] > 0


def test_all_ties_backed_up_queue(engine, monkeypatch):
    C, F, n = 4, 64, 300_000
    X = np.random.default_rng(3).integers(0, 17, size=(n, F)).astype(np.float32)
    model = engine.load_linear(np.ones((C, F)), np.zeros(C))
    routes = three_routes(engine, monkeypatch, model, engine.stage(X))
    assert_same(routes, "ties")
    assert routes[0][1]["n_flagged"] == n
    assert not routes[0][0].any()


def test_ring_floor(engine, monkeypatch):
    model = engine.load_linear(*tie_prone(5, 10, 64))
    X = np.random.default_rng(5).integers(0, 17, size=(50_001, 64)).astype(np.float32)
    monkeypatch.setenv("UML_B200_STAGES", "1")  # raised to the schedule's floor (one stage per warpgroup)
    assert_same(three_routes(engine, monkeypatch, model, engine.stage(X)), "floor")


_WORKER = r'''
import os, sys
import numpy as np, torch
sys.path.insert(0, os.environ["UML_ROOT"])
from unionml_b200.engine import Engine
from tests.test_gpu_linear_tc import tie_prone
dev = torch.device("cuda", 0)
e = Engine(0); s = torch.cuda.Stream(device=dev); torch.cuda.set_stream(s); e.set_stream(s.cuda_stream)
OFF = 3  # peer vectors start at an odd byte: the first and last words of every 128-row group take the byte path
for F, C in ((64, 10), (33, 16), (16, 3)):
    m = e.load_linear(*tie_prone(F * 7 + C, C, F))
    X = np.random.default_rng(F + C).integers(0, 256, size=(50_001, F)).astype(np.float32)
    for rows in (257, 1025, 50_001):
        b = e.stage(X[:rows])
        out = {r: torch.full((rows + OFF + 5,), 255, dtype=torch.uint8, device=dev) for r in ("b", "h", "f")}
        st = {}
        for r, env in (("b", "1"), ("h", "2"), ("f", "0")):
            os.environ["UML_B200_COMPACT_ROWS"] = env
            st[r] = e.predict_peers(m, b, [out[r].data_ptr()], OFF, exact=True, want_stats=True, label_bytes=1)
        os.environ.pop("UML_B200_COMPACT_ROWS")
        assert st["b"]["n_flagged"] == st["h"]["n_flagged"] == st["f"]["n_flagged"], (F, C, rows, st)
        assert [st[r]["x_read_bytes"] for r in ("b", "h", "f")] == [1, 2, 4], (F, C, rows, st)
        assert torch.equal(out["b"], out["h"]) and torch.equal(out["b"], out["f"]), (F, C, rows)
        assert int(out["b"][:OFF].min()) == 255 and int(out["b"][OFF + rows:].min()) == 255  # nothing outside the rows
        if os.environ.get("UML_TEST_GRAPH") and rows == 50_001:
            # the byte schedule replayed as a CUDA graph: every replay claims its tiles from counters the previous one
            # handed back at zero, and writes the labels of the eager launch
            os.environ["UML_B200_COMPACT_ROWS"] = "1"
            e.predict_peers(m, b, [out["b"].data_ptr()], OFF, exact=True, label_bytes=1)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                e.predict_peers(m, b, [out["b"].data_ptr()], OFF, exact=True, label_bytes=1)
            os.environ.pop("UML_B200_COMPACT_ROWS")
            for _ in range(3):
                out["b"].fill_(255)
                g.replay()
                torch.cuda.synchronize()
                assert torch.equal(out["b"], out["f"]), (F, C, rows)
print("byte rows ok")
'''


@pytest.mark.parametrize("stages,graph", [("", "1"), ("1", "")])
def test_uint8_peers_odd_offset_and_graph_replay(tmp_path, stages, graph):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, UML_ROOT=str(ROOT), UML_B200_RESCORE_MODE="queue", UML_TEST_GRAPH=graph)
    env.pop("UML_B200_COMPACT_ROWS", None)
    env.pop("UML_B200_LINEAR_TC", None)
    if stages:
        env["UML_B200_STAGES"] = stages
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "byte rows ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


def test_full_cfg2_batch(engine):
    """bench.py's cfg 2: 10M digits rows and the golden model through the byte schedule, labels byte-equal to the fp32
    route, n_flagged equal, and every row's label the float64 argmax (first maximum) except at rows whose float64
    top-2 margin is within rounding of a tie."""
    sys.path.insert(0, str(ROOT))
    import bench

    z = np.load(ROOT / "tests" / "golden" / "digits_lr.npz")
    coef, intercept = z["coef"], z["intercept"]
    n = 10_000_000
    X = np.empty((n, 64), dtype=np.float32)
    bench.digits_rows(0, n, X)
    model = engine.load_linear(coef, intercept, z["classes"])
    b = engine.stage(X)
    got, st = engine.predict(model, b, exact=True)
    assert st["x_read_bytes"] == 1
    os.environ["UML_B200_COMPACT_ROWS"] = "0"
    try:
        want_f, st_f = engine.predict(model, b, exact=True)
    finally:
        del os.environ["UML_B200_COMPACT_ROWS"]
    assert got.tobytes() == want_f.tobytes() and st["n_flagged"] == st_f["n_flagged"]
    W = torch.tensor(np.asarray(coef, dtype=np.float64), device="cuda")
    bias = torch.tensor(np.asarray(intercept, dtype=np.float64), device="cuda")
    wmax = W.abs().max(dim=0).values
    labels = torch.from_numpy(got.astype(np.int64)).cuda()
    for r0 in range(0, n, 1 << 20):
        x = torch.from_numpy(X[r0 : r0 + (1 << 20)]).to("cuda", torch.float64)
        s = x @ W.T + bias
        want = s.argmax(dim=1)
        diff = want != labels[r0 : r0 + x.shape[0]]
        if bool(diff.any()):
            top = torch.topk(s[diff], 2, dim=1).values
            a = x[diff].abs() @ wmax + bias.abs().max()
            assert bool(((top[:, 0] - top[:, 1]) <= 1e-12 * a).all()), r0
