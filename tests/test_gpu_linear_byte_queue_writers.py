"""Every label of the byte schedule (kByteMma) has one writer: a row tier 1 certifies is stored by its scoring warp, a
row it queues only by the re-score warp, and the byte words of uint8 peers leave the queued rows' bytes alone.

A model whose classes 0 and 1 share their weights and bias gives any row that lights feature 0 an exact tie between
them: tier 1 queues it, and float64 settles it on class 0.  Such rows are planted at every position mod 4 within a
label word, in the last (ragged) tile, and in batches where every row is one (the queue backs up and the scoring warps
wait for room).  Labels go to uint8 peers at row offsets 0-3 and to an int32 local vector with an int32 peer, and must
equal the fp32 route's, with the same n_flagged.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there
    pytest.skip("needs a CUDA device", allow_module_level=True)

C, F = 10, 64
SENTINEL = 0xAB


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


def tie_model(seed):
    rng = np.random.default_rng(seed)
    coef = np.round(rng.standard_normal((C, F)) * 4) / 16
    coef[:, 0] = 0.0
    coef[0, 0] = 8.0
    coef[1] = coef[0]
    intercept = np.round(rng.standard_normal(C) * 4) / 4
    intercept[1] = intercept[0]
    return coef, intercept


def planted_rows(n, seed, every=False):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 17, size=(n, F)).astype(np.float32)
    X[:, 0] = 0.0
    if every:
        X[:, 0] = 255.0
        return X
    idx = set()
    for k in range(4):  # every position within a label word, alone and next to each other
        idx.update(4 * m + k for m in (3, 40, 41, 200) if 4 * m + k < n)
    idx.update(range(512, 516))
    idx.update((n - 1, n - 2, n - 4, n - 7))  # the last tile
    X[sorted(i for i in idx if 0 <= i < n), 0] = 255.0
    return X


def fp32_route(engine, monkeypatch, model, b):
    monkeypatch.setenv("UML_B200_COMPACT_ROWS", "0")
    try:
        return engine.predict(model, b, exact=True)
    finally:
        monkeypatch.delenv("UML_B200_COMPACT_ROWS")


@pytest.mark.parametrize("n,every", [(5003, False), (20_001, False), (257, False), (6001, True)])
def test_uint8_peers_at_every_offset(engine, monkeypatch, n, every):
    coef, intercept = tie_model(n)
    model = engine.load_linear(coef, intercept)
    b = engine.stage(planted_rows(n, n + 1, every))
    want, st_f = fp32_route(engine, monkeypatch, model, b)
    assert st_f["n_flagged"] > 0
    monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
    for off in range(4):
        peers = [torch.full((off + n + 5,), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        st = engine.predict_peers(model, b, [p.data_ptr() for p in peers], off, exact=True, want_stats=True,
                                  label_bytes=1)
        torch.cuda.synchronize()
        assert st["x_read_bytes"] == 1 and st["n_flagged"] == st_f["n_flagged"], (off, st, st_f)
        for p in peers:
            got = p.cpu().numpy()
            np.testing.assert_array_equal(got[off:off + n], want.astype(np.uint8), err_msg=f"offset {off}")
            assert np.all(got[:off] == SENTINEL) and np.all(got[off + n:] == SENTINEL)


@pytest.mark.parametrize("n,every", [(5003, False), (6001, True)])
def test_int32_local_vector_and_peer(engine, monkeypatch, n, every):
    coef, intercept = tie_model(n + 2)
    model = engine.load_linear(coef, intercept)
    b = engine.stage(planted_rows(n, n + 3, every))
    want, st_f = fp32_route(engine, monkeypatch, model, b)
    monkeypatch.setenv("UML_B200_LINEAR_TC", "1")
    got, st = engine.predict(model, b, exact=True)
    assert st["x_read_bytes"] == 1 and st["n_flagged"] == st_f["n_flagged"]
    np.testing.assert_array_equal(got, want)
    off = 3
    peers = [torch.full((off + n + 5,), -7, dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    st = engine.predict_peers(model, b, [p.data_ptr() for p in peers], off, exact=True, want_stats=True, label_bytes=4)
    torch.cuda.synchronize()
    assert st["x_read_bytes"] == 1 and st["n_flagged"] == st_f["n_flagged"]
    for p in peers:
        g = p.cpu().numpy()
        np.testing.assert_array_equal(g[off:off + n], want)
        assert np.all(g[:off] == -7) and np.all(g[off + n:] == -7)
