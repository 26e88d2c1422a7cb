"""The compact fp16 copy of resident rows (F <= 64, every value an fp16 value) and the linear tile kernel's schedule that
reads it.

The fp16 route converts each feature back to the fp32 value the fp32 route reads and runs the same FMAs in the same
order, so its labels, flags and re-scored rows must equal the fp32 route's bit for bit - not within a tolerance.
UML_B200_COMPACT_ROWS=0 (read per call) sends a batch that has the copy down the fp32 route, so both routes run on one
staged batch.  A batch with any value that is not an fp16 value gets no copy and keeps the fp32 route.
"""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import linear as olin

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there (the -m gpu run happens on an H100)
    pytest.skip("needs a CUDA device", allow_module_level=True)

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def int_rows(seed, rows, F, hi=17):
    return np.random.default_rng(seed).integers(0, hi, size=(rows, F), dtype=np.int64).astype(np.float32)


def tie_prone_model(engine, seed, C, F):
    """Weights on a 1/4 grid and integer rows: many exact and near ties, so EXACT mode flags and re-scores rows."""
    rng = np.random.default_rng(seed)
    n = 1 if C == 2 else C  # C = 2: sklearn's binary layout (one coef_ row)
    coef = np.round(rng.standard_normal((n, F)) * 4) / 4
    intercept = np.round(rng.standard_normal(n) * 4) / 4
    return engine.load_linear(coef, intercept)


def both_routes(engine, model, batch, exact, monkeypatch):
    monkeypatch.delenv("UML_B200_COMPACT_ROWS", raising=False)
    got_h, st_h = engine.predict(model, batch, exact=exact)
    monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
    got_f, st_f = engine.predict(model, batch, exact=exact)
    monkeypatch.delenv("UML_B200_COMPACT_ROWS")
    return (got_h, st_h), (got_f, st_f)


def oracle_idx(X, coef, intercept):
    return olin.predict_indices(olin.decision_function(np.asarray(X, dtype=np.float64), coef, intercept)).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# bit-identity of the two routes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("C", [2, 3, 10, 16])
@pytest.mark.parametrize("F", [1, 7, 8, 31, 32, 33, 63, 64])
def test_fp16_route_equals_fp32_route(engine, monkeypatch, F, C, exact):
    model = tie_prone_model(engine, 100 + F * 17 + C, C, F)
    X = int_rows(F * 31 + C, 300_001, F)
    for rows in (1, 127, 128, 129, 300_001):
        b = engine.stage(X[:rows])
        (got_h, st_h), (got_f, st_f) = both_routes(engine, model, b, exact, monkeypatch)
        assert st_h["path"] == st_f["path"] == 1
        assert st_h["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4, (st_h, st_f)
        np.testing.assert_array_equal(got_h, got_f)
        assert st_h["n_flagged"] == st_f["n_flagged"]
        assert st_h["n_ambiguous"] == st_f["n_ambiguous"]


_WORKER = r'''
import os, sys
import numpy as np
sys.path.insert(0, os.environ["UML_ROOT"])
from unionml_b200.engine import Engine
e = Engine(0)
flagged = 0
for F in (7, 33, 64):
    for C in (2, 10):
        rng = np.random.default_rng(F * 100 + C)
        coef = np.round(rng.standard_normal((1 if C == 2 else C, F)) * 4) / 4
        m = e.load_linear(coef, np.round(rng.standard_normal(coef.shape[0]) * 4) / 4)
        X = rng.integers(0, 17, size=(300_001, F)).astype(np.float32)
        for rows in (129, 300_001):
            b = e.stage(X[:rows])
            for exact in (True, False):
                os.environ.pop("UML_B200_COMPACT_ROWS", None)
                gh, sh = e.predict(m, b, exact=exact)
                os.environ["UML_B200_COMPACT_ROWS"] = "0"
                gf, sf = e.predict(m, b, exact=exact)
                assert sh["x_elem_bytes"] == 2 and sf["x_elem_bytes"] == 4, (sh, sf)
                assert np.array_equal(gh, gf), (F, C, rows, exact)
                assert sh["n_flagged"] == sf["n_flagged"] and sh["kernel_launches"] == sf["kernel_launches"]
                flagged += sh["n_flagged"]
print("routes ok", flagged)
'''


@pytest.mark.parametrize("rescore_mode,stages", [("queue", ""), ("kernel", ""), ("queue", "8"), ("kernel", "8")])
def test_fp16_route_rescore_modes_and_shallowest_ring(tmp_path, rescore_mode, stages):
    """Both re-score modes (in-kernel queue / flag list + kernel), and the shallowest legal ring (8 stages)."""
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, UML_ROOT=str(ROOT), UML_B200_RESCORE_MODE=rescore_mode)
    env.pop("UML_B200_COMPACT_ROWS", None)
    if stages:
        env["UML_B200_STAGES"] = stages
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "routes ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert int(r.stdout.split()[-1]) > 0  # the tie-prone models did send rows to the fp64 re-score


# ---------------------------------------------------------------------------------------------------------------
# which batches get the copy
# ---------------------------------------------------------------------------------------------------------------
ONE_MILLION = 1_000_000


@pytest.fixture(scope="module")
def million_rows():
    return int_rows(7, ONE_MILLION, 64)


@pytest.mark.parametrize("value", [65505.0, 2049.0, 1.0 + 2.0**-11, 2.0**-25, 1.0 / 3.0])
def test_one_value_outside_fp16_keeps_the_fp32_route(engine, digits_model, million_rows, value):
    X = million_rows.copy()
    X[654_321, 37] = np.float32(value)
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    got, st = engine.predict(m, engine.stage(X), exact=True)
    assert st["x_elem_bytes"] == 4, st
    np.testing.assert_array_equal(got, oracle_idx(X, digits_model["coef"], digits_model["intercept"]))


@pytest.mark.parametrize("value", [65504.0, -65504.0, 2048.0, 1.0 + 2.0**-10, 2.0**-24, -0.0])
def test_fp16_values_keep_the_fp16_route(engine, digits_model, million_rows, monkeypatch, value):
    X = million_rows.copy()
    X[654_321, 37] = np.float32(value)
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    b = engine.stage(X)
    (got_h, st_h), (got_f, st_f) = both_routes(engine, m, b, True, monkeypatch)
    assert st_h["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4
    np.testing.assert_array_equal(got_h, got_f)
    assert st_h["n_flagged"] == st_f["n_flagged"]
    np.testing.assert_array_equal(got_h, oracle_idx(X, digits_model["coef"], digits_model["intercept"]))


def test_wide_rows_take_the_fp32_route(engine):
    rng = np.random.default_rng(65)
    X = int_rows(65, 20_000, 65)
    coef, intercept = rng.standard_normal((10, 65)), rng.standard_normal(10)
    got, st = engine.predict(engine.load_linear(coef, intercept), engine.stage(X), exact=True)
    assert st["path"] == 1 and st["x_elem_bytes"] == 4
    np.testing.assert_array_equal(got, oracle_idx(X, coef, intercept))


def test_wrapped_device_rows_get_no_copy(engine, digits_model):
    X = torch.from_numpy(int_rows(11, 100_000, 64)).cuda()
    b = engine.wrap_device(X.data_ptr(), X.shape[0], 64, 64, keepalive=X)
    got, st = engine.predict(engine.load_linear(digits_model["coef"], digits_model["intercept"]), b, exact=True)
    assert st["path"] == 1 and st["x_elem_bytes"] == 4
    np.testing.assert_array_equal(got, oracle_idx(X.cpu().numpy(), digits_model["coef"], digits_model["intercept"]))


def test_float64_frame_through_the_chunked_staging_gets_the_copy(engine, digits_model, monkeypatch):
    import pandas as pd

    X = int_rows(12, 200_003, 64).astype(np.float64)
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    want = oracle_idx(X, digits_model["coef"], digits_model["intercept"])
    for src in (pd.DataFrame(X), np.asfortranarray(X), X):  # feature-major block, and row-major through the convert kernel
        (got_h, st_h), (got_f, st_f) = both_routes(engine, m, engine.stage(src), True, monkeypatch)
        assert st_h["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4
        np.testing.assert_array_equal(got_h, want)
        np.testing.assert_array_equal(got_f, want)
    Xl = X.copy()
    Xl[100_000, 5] = 0.1  # a float64 value that is not an fp16 value: no copy
    _, st = engine.predict(m, engine.stage(pd.DataFrame(Xl)), exact=True)
    assert st["x_elem_bytes"] == 4


# ---------------------------------------------------------------------------------------------------------------
# fused peer stores
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("label_bytes", [1, 4])
def test_peer_stores_equal_the_fp32_route(engine, digits_model, monkeypatch, label_bytes):
    """Two shards of ragged sizes at a row offset that is not a multiple of 4, into two local vectors."""
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"])
    X = int_rows(21, 380_002, 64)
    shards = [(3, X[:250_001]), (3 + 250_001, X[250_001:])]
    batches = [(off, engine.stage(rows)) for off, rows in shards]
    dtype = torch.uint8 if label_bytes == 1 else torch.int32
    out = {}
    for route in ("fp16", "fp32"):
        if route == "fp32":
            monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
        vecs = [torch.full((X.shape[0] + 7,), 0x5A, dtype=dtype, device="cuda") for _ in range(2)]
        flagged = 0
        for off, b in batches:
            st = engine.predict_peers(m, b, [v.data_ptr() for v in vecs], off, exact=True, want_stats=True,
                                      label_bytes=label_bytes)
            assert st["x_elem_bytes"] == (2 if route == "fp16" else 4)
            flagged += st["n_flagged"]
        out[route] = ([v.cpu().numpy() for v in vecs], flagged)
        monkeypatch.delenv("UML_B200_COMPACT_ROWS", raising=False)
    for a, b in zip(out["fp16"][0], out["fp32"][0]):
        assert a.tobytes() == b.tobytes()
    assert out["fp16"][1] == out["fp32"][1]
    want = oracle_idx(X, digits_model["coef"], digits_model["intercept"])
    np.testing.assert_array_equal(out["fp16"][0][1][3 : 3 + X.shape[0]].astype(np.int32), want)


# ---------------------------------------------------------------------------------------------------------------
# the full cfg 2 batch
# ---------------------------------------------------------------------------------------------------------------
def test_cfg2_batch_both_routes(engine, digits_model, monkeypatch):
    sys.path.insert(0, str(ROOT))
    from bench import digits_rows

    n = 10_000_000
    X = np.empty((n, 64), dtype=np.uint8)
    digits_rows(0, n, X)
    Xf = X.astype(np.float32)
    m = engine.load_linear(digits_model["coef"], digits_model["intercept"], digits_model["classes"])
    b = engine.stage(Xf)
    del Xf
    res = {}
    for route in ("fp16", "fp32"):
        if route == "fp32":
            monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
        lab = torch.empty(n, dtype=torch.uint8, device="cuda")
        st = engine.predict_peers(m, b, [lab.data_ptr()], 0, exact=True, want_stats=True, label_bytes=1)
        res[route] = (lab.cpu().numpy(), st)
        monkeypatch.delenv("UML_B200_COMPACT_ROWS", raising=False)
    (lh, sh), (lf, sf) = res["fp16"], res["fp32"]
    assert sh["x_elem_bytes"] == 2 and sf["x_elem_bytes"] == 4
    assert lh.tobytes() == lf.tobytes()
    assert sh["n_flagged"] == sf["n_flagged"] > 0
    sample = np.random.default_rng(0).choice(n, size=200_000, replace=False)
    want = oracle_idx(X[sample], digits_model["coef"], digits_model["intercept"])
    np.testing.assert_array_equal(lh[sample].astype(np.int32), want)
