"""256-row ring items of the linear tile kernel's fp16 schedule (four scoring warps, 8 rows per lane, tiles claimed four
at a time).

On one staged batch the fp16 schedule and the fp32 route (UML_B200_COMPACT_ROWS=0) run the same FMAs in the same order,
so labels must be byte-equal and n_flagged equal - for every class count 2..16 (8 rows of up to 17 accumulators per
lane) and widths 1, 32, 33 and 64, at row counts around one item (256), two items (512) and one claim group
(4 x 256 = 1024), where the last item's second 128-row box lies wholly or partly past the batch; in FAST and EXACT
mode, with the in-kernel queue and with the
flag list, with the ring at its 4-item floor, with uint8 peer stores at an odd offset (nothing written outside the rows),
and replayed as a CUDA graph.
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
ITEM, GROUP = 256, 4 * 256  # rows of one ring item and of one claim group of the fp16 schedule
ROWS = (1, 127, 129, ITEM - 1, ITEM, ITEM + 1, 2 * ITEM - 1, 2 * ITEM, 2 * ITEM + 1, GROUP - 1, GROUP, GROUP + 1,
        3 * GROUP + 200, 60_001)


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def tie_prone(seed, C, F):
    """Weights on a 1/4 grid (integer rows then give many exact and near ties, so EXACT mode flags rows)."""
    rng = np.random.default_rng(seed)
    n = 1 if C == 2 else C  # C = 2: sklearn's binary layout (one coef_ row)
    return np.round(rng.standard_normal((n, F)) * 4) / 4, np.round(rng.standard_normal(n) * 4) / 4


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("C", list(range(2, 17)))
@pytest.mark.parametrize("F", [1, 32, 33, 64])
def test_256_row_items_equal_fp32_route(engine, monkeypatch, F, C, exact):
    model = engine.load_linear(*tie_prone(2000 + 37 * F + C, C, F))
    X = np.random.default_rng(F * 173 + C).integers(0, 17, size=(ROWS[-1], F)).astype(np.float32)
    flagged = 0
    for rows in ROWS:
        b = engine.stage(X[:rows])
        monkeypatch.delenv("UML_B200_COMPACT_ROWS", raising=False)
        got_h, st_h = engine.predict(model, b, exact=exact)
        monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
        got_f, st_f = engine.predict(model, b, exact=exact)
        monkeypatch.delenv("UML_B200_COMPACT_ROWS")
        assert st_h["path"] == st_f["path"] == 1
        assert st_h["x_elem_bytes"] == 2 and st_f["x_elem_bytes"] == 4, (st_h, st_f)
        assert got_h.tobytes() == got_f.tobytes(), (rows, int((got_h != got_f).sum()))
        assert st_h["n_flagged"] == st_f["n_flagged"], rows
        flagged += st_h["n_flagged"]
    # EXACT did send rows to the fp64 re-score (the binary layout's single score column rarely ties exactly)
    assert not exact or F == 1 or C == 2 or flagged > 0


_WORKER = r'''
import os, sys
import numpy as np, torch
sys.path.insert(0, os.environ["UML_ROOT"])
from unionml_b200.engine import Engine
dev = torch.device("cuda", 0)
e = Engine(0); s = torch.cuda.Stream(device=dev); torch.cuda.set_stream(s); e.set_stream(s.cuda_stream)
OFF = 3  # peer vectors start at an odd byte: the first and last words of every 128-row group take the byte path
flagged = 0
for C in range(2, 17):
    F = (33, 64)[C % 2]
    rng = np.random.default_rng(F * 100 + C)
    n = 1 if C == 2 else C
    m = e.load_linear(np.round(rng.standard_normal((n, F)) * 4) / 4, np.round(rng.standard_normal(n) * 4) / 4)
    X = rng.integers(0, 17, size=(50_001, F)).astype(np.float32)
    for rows in (129, 1025, 50_001):
        b = e.stage(X[:rows])
        out = {r: torch.full((rows + OFF + 5,), 255, dtype=torch.uint8, device=dev) for r in ("h", "f")}
        for exact in (True, False):
            os.environ.pop("UML_B200_COMPACT_ROWS", None)
            sh = e.predict_peers(m, b, [out["h"].data_ptr()], OFF, exact=exact, want_stats=True, label_bytes=1)
            os.environ["UML_B200_COMPACT_ROWS"] = "0"
            sf = e.predict_peers(m, b, [out["f"].data_ptr()], OFF, exact=exact, want_stats=True, label_bytes=1)
            os.environ.pop("UML_B200_COMPACT_ROWS")
            assert sh["x_elem_bytes"] == 2 and sf["x_elem_bytes"] == 4, (sh, sf)
            assert torch.equal(out["h"], out["f"]), (F, C, rows, exact)
            assert int(out["h"][:OFF].min()) == 255 and int(out["h"][OFF + rows:].min()) == 255  # nothing outside the rows
            assert int(out["h"][OFF:OFF + rows].max()) < C
            assert sh["n_flagged"] == sf["n_flagged"] and sh["kernel_launches"] == sf["kernel_launches"]
            flagged += sh["n_flagged"]
        if os.environ.get("UML_TEST_GRAPH") and rows == 50_001:
            # the EXACT fp16 launch replayed as a CUDA graph: every replay claims its tiles from counters the previous
            # one handed back at zero, and writes the labels of the eager launch
            e.predict_peers(m, b, [out["h"].data_ptr()], OFF, exact=True, label_bytes=1)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                e.predict_peers(m, b, [out["h"].data_ptr()], OFF, exact=True, label_bytes=1)
            os.environ["UML_B200_COMPACT_ROWS"] = "0"
            e.predict_peers(m, b, [out["f"].data_ptr()], OFF, exact=True, label_bytes=1)
            os.environ.pop("UML_B200_COMPACT_ROWS")
            want = out["f"].clone()
            for _ in range(3):
                out["h"].fill_(255)
                g.replay()
                torch.cuda.synchronize()
                assert torch.equal(out["h"], want), (F, C, rows)
print("half tiles ok", flagged)
'''


@pytest.mark.parametrize("rescore_mode,stages,graph", [("queue", "", "1"), ("kernel", "", ""), ("queue", "4", ""),
                                                        ("kernel", "4", ""), ("queue", "1", "")])
def test_uint8_peers_rescore_modes_ring_floor_and_graph_replay(tmp_path, rescore_mode, stages, graph):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, UML_ROOT=str(ROOT), UML_B200_RESCORE_MODE=rescore_mode, UML_TEST_GRAPH=graph)
    env.pop("UML_B200_COMPACT_ROWS", None)
    if stages:  # 4: the fp16 schedule's floor; 1 is raised to it
        env["UML_B200_STAGES"] = stages
    r = subprocess.run([sys.executable, str(script)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "half tiles ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    assert int(r.stdout.split()[-1]) > 0  # the tie-prone models did send rows to the fp64 re-score
