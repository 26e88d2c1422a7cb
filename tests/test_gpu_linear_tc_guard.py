"""Tier 1 of the linear tile kernel's tensor-core schedules (kByteMma, kHalfMma) against exact arithmetic.

Tier 1 certifies a row iff m_tc > kappa a (DESIGN.md 3.2); tier 2 replays every other row on the fp32 route's
arithmetic, which hides tier 1's decisions.  UML_B200_TC_REPLAY=0 sends every row tier 1 leaves straight to float64,
so n_flagged is tier 1's count of uncertified rows, and every label must still be the exact argmax (or the row is
counted in n_ambiguous).  tests/tc_guard_cases.py restates the guard's operands and gives each row a verdict from its
exact margin: must-certify, must-leave or either.  Families:
  exact     everything exact on the tensor cores, margins planted at r kappa A_hat, r in {0, 0.5, 0.99, 1.01, 2}:
            n_flagged is the count of r < 1 (kappa pinned to +-1 %), n_ambiguous the exact ties
  rounding  full-mantissa weights, fp16 rows up to 65504 and subnormals (half route), bytes with sparse 255s (byte
            route): n_flagged within [#must-leave, n - #must-certify], the tensor cores' real error against e_rel
  tiny      weights near 2^-120: the fp32 route's bound is its K term and it flags rows tier 1 must leave too
  lossy     a float64 batch whose values the fp32 cast rounds: rows whose exact argmax differs from the cast's end
            with float64 labels
On every family tier 1 may only certify rows the fp32 route certifies: n_flagged >= the fp32 route's.  With the hook
off, labels and n_flagged equal the fp32 route's.  UML_B200_LINEAR_TC=1 makes a call fail unless a tensor-core
schedule runs, and x_read_bytes says which copy it read.
"""
import functools
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

from tests import tc_guard_cases as tg  # noqa: E402

ROOT = Path(__file__).resolve().parent.parent
ROUTES = {"byte": ({}, 1), "half": ({"UML_B200_COMPACT_ROWS": "2"}, 2)}
SHAPES = [(F, C) for F in (1, 16, 32, 33, 64) for C in (2, 3, 8, 9, 10, 15, 16)]
LAYOUTS = [(F, C, False) for F, C in SHAPES] + [(F, 2, True) for F in (1, 16, 32, 33, 64)]
ENV = ("UML_B200_COMPACT_ROWS", "UML_B200_LINEAR_TC", "UML_B200_TC_REPLAY")


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def run(engine, monkeypatch, model, b, route, replay=False):
    """One EXACT predict on a tensor-core schedule (the call fails otherwise), with or without tier 2's replay."""
    env, read = ROUTES[route]
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
    if not replay:
        monkeypatch.setenv("UML_B200_TC_REPLAY", "0")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        got, st = engine.predict(model, b, exact=True)
    finally:
        for k in ENV:
            monkeypatch.delenv(k, raising=False)
    assert st["x_read_bytes"] == read, st
    return got, st


def fp32_route(engine, monkeypatch, model, b):
    monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
    try:
        got, st = engine.predict(model, b, exact=True)
    finally:
        monkeypatch.delenv("UML_B200_COMPACT_ROWS")
    assert st["x_read_bytes"] == 4
    return got, st


def check_all(engine, monkeypatch, coef, intercept, X, route, what, labels=None, margins=None):
    """The rules of every family; returns (stats with the hook, stats of the fp32 route, verdicts)."""
    ops = tg.operands(coef, intercept)
    assert ops.eligible, what
    if labels is None:
        labels, margins = tg.truth(X, coef, intercept)
    model = engine.load_linear(coef, intercept)
    b = engine.stage(X)
    got, st = run(engine, monkeypatch, model, b, route)
    wrong = int((got != labels).sum())
    assert wrong <= st["n_ambiguous"], (what, wrong, st)
    v = tg.verdicts(ops, X, margins) if margins is not None else None
    if v is not None:
        assert (v == -1).sum() <= st["n_flagged"] <= len(X) - (v == 1).sum(), (what, st, np.bincount(v + 1, minlength=3))
    got_f, st_f = fp32_route(engine, monkeypatch, model, b)
    assert st["n_flagged"] >= st_f["n_flagged"], (what, st, st_f)
    got_r, st_r = run(engine, monkeypatch, model, b, route, replay=True)
    assert got_r.tobytes() == got_f.tobytes() and st_r["n_flagged"] == st_f["n_flagged"], (what, st_r, st_f)
    return st, st_f, v


@functools.lru_cache(maxsize=None)
def exact_parts(F, C):
    return tg.exact_family(F, C, seed=7000 + 97 * F + C)


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("F,C", SHAPES)
def test_exact_family_pins_kappa(engine, monkeypatch, F, C, route):
    """Every rung below 1 is left and every rung above 1 certified: n_flagged is the count of r < 1."""
    for i, (coef, intercept, X) in enumerate(exact_parts(F, C)):
        ops = tg.operands(coef, intercept)
        labels, margins = tg.truth(X, coef, intercept)
        rung = tg.rung_of(ops, X, margins)
        assert not np.isnan(rung).any()
        st, _, _ = check_all(engine, monkeypatch, coef, intercept, X, route, (F, C, i), labels, margins)
        assert st["n_flagged"] == int((rung < 1).sum()), (F, C, i, st, np.unique(rung, return_counts=True))
        assert st["n_ambiguous"] == int((rung == 0).sum()), (F, C, i, st)


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("F,C,binary", LAYOUTS)
def test_rounding_family_within_budget(engine, monkeypatch, F, C, binary, route):
    rng = np.random.default_rng(8000 + 97 * F + C + (50 if binary else 0) + (1 if route == "half" else 0))
    W, b = tg.rounding_model(F, C, rng, binary)
    X = tg.rounding_rows(F, rng, 3001, route)
    check_all(engine, monkeypatch, W, b, X, route, (F, C, binary))


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("F,C", [(1, 3), (16, 2), (33, 9), (64, 10), (64, 16)])
def test_rows_the_fp32_route_flags_are_left(engine, monkeypatch, F, C, route):
    rng = np.random.default_rng(9000 + 97 * F + C)
    W, b = tg.tiny_model(F, C, rng)
    X = tg.tiny_rows(F, rng, 2001, route)
    st, st_f, _ = check_all(engine, monkeypatch, W, b, X, route, (F, C))
    assert st_f["n_flagged"] > 0


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("F,C", [(16, 3), (33, 16), (64, 10)])
def test_subnormal_pieces_are_left(engine, monkeypatch, F, C, route):
    """The tensor cores rank these rows wrongly by q x; wb's 2^-3 floor keeps them in tier 2."""
    W, b, X = tg.subnormal_pieces_case(F, C, route)
    labels, _ = tg.truth(X, W, b)
    assert np.all(labels == 0)
    st, _, v = check_all(engine, monkeypatch, W, b, X, route, (F, C), labels, tg.truth(X, W, b)[1])
    assert st["n_flagged"] == len(X) and np.all(v == -1)


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("F,C,binary", [(1, 2, True), (16, 3, False), (64, 10, False), (33, 16, False)])
def test_lossy_float64_rows_end_with_float64_labels(engine, monkeypatch, F, C, binary, route):
    rng = np.random.default_rng(9500 + 97 * F + C)
    W, b, X = tg.lossy_case(F, C, rng, 3001, binary)
    labels, _ = tg.truth(X, W, b)
    cast, _ = tg.truth(X.astype(np.float32), W, b)
    assert (labels != cast).sum() > 0
    model = engine.load_linear(W, b)
    batch = engine.stage(X, keep_f64=True)
    for replay in (False, True):
        got, st = run(engine, monkeypatch, model, batch, route, replay=replay)
        assert np.array_equal(got, labels), (replay, int((got != labels).sum()), st)


_WORKER = r'''
import os, sys
import numpy as np, torch
sys.path.insert(0, os.environ["UML_ROOT"])
from unionml_b200.engine import Engine
from tests import tc_guard_cases as tg
dev = torch.device("cuda", 0)
e = Engine(0); s = torch.cuda.Stream(device=dev); torch.cuda.set_stream(s); e.set_stream(s.cuda_stream)
OFF = 3  # peer vectors start at an odd byte
os.environ["UML_B200_LINEAR_TC"] = "1"
for F, C in ((64, 10), (33, 16), (16, 3)):
    coef, intercept, X = tg.exact_family(F, C, seed=7000 + 97 * F + C)[0]
    rng = np.random.default_rng(F * C)
    W, b = tg.rounding_model(F, C, rng)
    Xr = tg.rounding_rows(F, rng, 20_001, "byte")
    for m_args, rows in (((coef, intercept), X), ((W, b), Xr)):
        m = e.load_linear(*m_args)
        want, _ = tg.truth(rows, *m_args)
        n = len(rows)
        batch = e.stage(rows)
        out = torch.full((n + OFF + 5,), 255, dtype=torch.uint8, device=dev)
        os.environ["UML_B200_TC_REPLAY"] = "0"
        st = e.predict_peers(m, batch, [out.data_ptr()], OFF, exact=True, want_stats=True, label_bytes=1)
        _, st_p = e.predict(m, batch, exact=True)
        assert st["x_read_bytes"] == 1 and st["n_flagged"] == st_p["n_flagged"], (F, C, st, st_p)
        wrong = int((out[OFF:OFF + n].cpu().numpy() != want).sum())
        assert wrong <= st["n_ambiguous"], (F, C, wrong, st)
        assert int(out[:OFF].min()) == 255 and int(out[OFF + n:].min()) == 255
        ref = out.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            e.predict_peers(m, batch, [out.data_ptr()], OFF, exact=True, label_bytes=1)
        os.environ.pop("UML_B200_TC_REPLAY")  # read when the launch is captured: the replays run with the hook
        for _ in range(3):
            out.fill_(255)
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref), (F, C)
print("tc guard graph ok")
'''


def test_hook_through_uint8_peers_and_graph_replay(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, UML_ROOT=str(ROOT), UML_B200_RESCORE_MODE="queue")
    for k in ENV:
        env.pop(k, None)
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "tc guard graph ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
