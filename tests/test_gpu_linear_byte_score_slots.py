"""The byte schedule's score slots (kByteMma): each MMA warpgroup posts every ring item it takes to one of its two
slots and its pair of epilogue warps walks the same sequence, so a CTA's last item can end on any slot and phase.

Ring item n of a CTA is warpgroup n % 2's item n / 2, in slot (n / 2) % 2 with phase (n / 4) % 2, and a CTA claims two
items at a time.  Batches of 1-7 tiles put the last scored item on each of those positions, and the unscored items
after it (past the batch, then the sentinel) on the rest; batches just past one, two and three claim groups per CTA of
the whole grid do the same for CTAs with more than one group.  Labels and n_flagged must equal the fp32 route's, at C = 2
and C = 16 (the largest slots), with the default ring and at its floor of one stage per warpgroup.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.test_gpu_linear_tc import tie_prone  # noqa: E402

ITEM = 256


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def tile_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return list(range(1, 8)) + [2 * sms + k for k in (1, 2, 3)] + [4 * sms + k for k in (1, 3)] + [6 * sms + k for k in (2, 5)]


@pytest.mark.parametrize("stages", ["", "1"])
@pytest.mark.parametrize("C", [2, 16])
def test_last_item_on_every_slot_and_phase(engine, monkeypatch, C, stages):
    F = 64
    model = engine.load_linear(*tie_prone(900 + C, C, F))
    counts = tile_counts()
    X = np.random.default_rng(C).integers(0, 17, size=(counts[-1] * ITEM, F)).astype(np.float32)
    if stages:
        monkeypatch.setenv("UML_B200_STAGES", stages)  # raised to the schedule's floor
    for tiles in counts:
        for rows in (tiles * ITEM, tiles * ITEM - 77):
            b = engine.stage(X[:rows])
            monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
            got, st = engine.predict(model, b, exact=True)
            monkeypatch.delenv("UML_B200_LINEAR_TC")
            monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
            want, st_f = engine.predict(model, b, exact=True)
            monkeypatch.delenv("UML_B200_COMPACT_ROWS")
            assert (st["x_read_bytes"], st_f["x_read_bytes"]) == (1, 4), (tiles, rows)
            assert got.tobytes() == want.tobytes(), (tiles, rows, int((got != want).sum()))
            assert st["n_flagged"] == st_f["n_flagged"], (tiles, rows, st, st_f)
