"""GPU tests of where a resident-batch call writes its outputs: every ``Engine`` call on a resident batch, once into
host memory and once into device memory (``out_device_ptr`` / ``idx_device_ptr``), on the same seeded batch.  The two
must give the same bytes and, apart from the times and ``d2h_bytes``, the same stats; the device form without stats is
the asynchronous one.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from tests.conftest import GOLDEN, digits_batch  # noqa: E402

TIMES = ("kernel_ms", "recheck_ms", "total_ms", "d2h_bytes")


@pytest.fixture(scope="module")
def setup(digits_model):
    from unionml_b200.engine import Engine

    eng = Engine(0)
    lin = eng.load_linear(digits_model["coef"], digits_model["intercept"], digits_model["classes"])
    z = np.load(GOLDEN / "mlp_64_32_10.npz")
    mlp = eng.load_mlp(z["w1"], z["b1"], z["w2"], z["b2"])
    rows = digits_batch(7, 5000, np.float64)
    rows[::97] += 0.3  # values off the integer grid: fp32 rows that are not tf32 values, re-scored rows
    return eng, lin, mlp, eng.stage(rows)


def _device(shape, dtype):
    return torch.empty(shape, dtype=dtype, device="cuda")


# name -> (engine method, positional model argument, keyword arguments, device outputs as (shape, torch dtype) per row)
CALLS = {
    "predict_exact": ("predict", "lin", {"exact": True}, [((), torch.int32)]),
    "predict_fast": ("predict", "lin", {"exact": False}, [((), torch.int32)]),
    "predict_mlp": ("predict_mlp", "mlp", {"exact": True}, [((), torch.int32)]),
    "predict_mlp_proba": ("predict_mlp_proba", "mlp", {}, [((10,), torch.float32)]),
    "predict_mlp_topk": ("predict_mlp_topk", "mlp", {"k": 3}, [((3,), torch.int32), ((3,), torch.float32)]),
    "predict_mlp_topk_f64": ("predict_mlp_topk", "mlp", {"k": 7, "exact": False}, [((7,), torch.int32), ((7,), torch.float32)]),
    "predict_proba": ("predict_proba", "lin", {}, [((10,), torch.float32)]),
    "decision_function": ("decision_function", "lin", {}, [((10,), torch.float64)]),
    "predict_proba_f64": ("predict_proba_f64", "lin", {}, [((10,), torch.float64)]),
    "predict_log_proba_f64": ("predict_proba_f64", "lin", {"log": True}, [((10,), torch.float64)]),
}


def _run(eng, fn, model, batch, kwargs, device_outs, stats):
    """(outputs as numpy arrays, stats or None) of one call, with host or (device_outs) device outputs."""
    if fn != "predict_proba":
        kwargs = dict(kwargs, want_stats=stats)
    if device_outs is None:
        res = getattr(eng, fn)(model, batch, **kwargs)
        if fn == "predict_proba":
            return [res], None
        *outs, st = res
        return outs, st
    bufs = [_device((batch.n_rows, *shape), dtype) for shape, dtype in device_outs]
    if fn == "predict_mlp_topk":
        kwargs.update(idx_device_ptr=bufs[0].data_ptr(), proba_device_ptr=bufs[1].data_ptr())
    else:
        kwargs.update(out_device_ptr=bufs[0].data_ptr())
    res = getattr(eng, fn)(model, batch, **kwargs)
    st = None if fn == "predict_proba" else res[-1]
    eng.synchronize()
    return [b.cpu().numpy() for b in bufs], st


@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("name", sorted(CALLS))
def test_host_and_device_outputs_agree(setup, name, stats):
    eng, lin, mlp, batch = setup
    fn, which, kwargs, device_outs = CALLS[name]
    if fn == "predict_proba" and stats:
        pytest.skip("uml_linear_predict_proba reports no stats")
    model = lin if which == "lin" else mlp
    host, st_host = _run(eng, fn, model, batch, kwargs, None, stats)
    dev, st_dev = _run(eng, fn, model, batch, kwargs, device_outs, stats)
    assert len(host) == len(dev)
    for h, d in zip(host, dev):
        assert h is not None and d.dtype == h.dtype
        assert d.reshape(h.shape).tobytes() == h.tobytes(), name
    if stats:
        assert st_host["n_rows"] == batch.n_rows
        assert st_host["d2h_bytes"] == sum(h.nbytes for h in host)
        assert st_dev["d2h_bytes"] == 0
        assert {k: v for k, v in st_host.items() if k not in TIMES} == {k: v for k, v in st_dev.items() if k not in TIMES}
    else:
        assert st_host is None and st_dev is None
