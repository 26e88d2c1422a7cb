"""The fused all-gather epilogue of the linear tile kernel on one GPU: Engine.predict_peers with two local device buffers
standing in for two ranks' label vectors, at a row offset that is not a multiple of 4 and a ragged row count, on both
sides of the tile schedule choice (whole-row stages at F <= 64, 32-feature chunks beyond)."""
import numpy as np
import pytest
import torch

from oracle import linear as olin

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected on CPU boxes, skipped there (the -m gpu run happens on an H100)
    pytest.skip("needs a CUDA device", allow_module_level=True)

SENTINEL = 0xAB


@pytest.fixture(scope="module")
def engine():
    from unionml_b200.engine import Engine

    return Engine(0)


@pytest.mark.parametrize("label_bytes", [1, 4])
@pytest.mark.parametrize("n_features", [40, 64, 100])
@pytest.mark.parametrize("rows,row_offset", [(100_003, 5), (61, 7)])
def test_peer_stores_two_targets(engine, n_features, rows, row_offset, label_bytes):
    rng = np.random.default_rng(n_features * 1000 + rows)
    coef = rng.standard_normal((10, n_features)) * 0.05
    intercept = rng.standard_normal(10)
    X = rng.integers(0, 17, size=(rows, n_features)).astype(np.float32)
    want = olin.predict_indices(olin.decision_function(X.astype(np.float64), coef, intercept))

    m = engine.load_linear(coef, intercept)
    b = engine.stage(X)
    dtype = torch.uint8 if label_bytes == 1 else torch.int32
    total = row_offset + rows + 9
    peers = [torch.full((total,), SENTINEL, dtype=dtype, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    st = engine.predict_peers(m, b, [p.data_ptr() for p in peers], row_offset, exact=True, want_stats=True,
                              label_bytes=label_bytes)
    torch.cuda.synchronize()
    assert st["path"] == 1  # the tile kernel's own epilogue stored the labels
    for p in peers:
        got = p.cpu().numpy().astype(np.int64)
        np.testing.assert_array_equal(got[row_offset:row_offset + rows], want)
        assert np.all(got[:row_offset] == SENTINEL) and np.all(got[row_offset + rows:] == SENTINEL)
