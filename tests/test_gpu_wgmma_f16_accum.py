"""Measured error of the Hopper f16 wgmma accumulation against the budget of the linear tile kernel's tensor-core guard.

`linear_argmax_tma_kernel<..., kHalfMma>` certifies a row on its tensor-core margin with a bound that budgets
kTcStepBudget = 64u (u = 2^-24) of the running absolute sum per accumulating m64nNk16 step (engine.cu, DESIGN.md 3.2).
Here the product's own `WgmmaF16<N>::mma` runs on chosen fp16 operands (tests/cuda/wgmma_f16_accum_probe.cu, a
test-only library built by `build()`), and every element of D is compared with the exact sum: f16 x f16 products are
exact in float64, and `math.fsum` rounds their sum once.  For each element the error is divided by u * sum_s S_s, where
S_s is the sum of |a_k b_k| over the first s + 1 steps - the per-step budget - and the worst ratio must stay 4x inside
the budget.  The subnormal family would show a flush of fp16 subnormal operands as a ratio near 2^24.
"""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

PROBE = ROOT / "build" / "tests" / "libwgmma_f16_accum_probe.so"
U = 2.0**-24
BUDGET_PER_STEP = 64  # engine.cu: kTcStepBudget
STEPS = 4  # k16 steps of a 64-feature row


@pytest.fixture(scope="module")
def probe():
    if not PROBE.exists():
        pytest.fail(f"{PROBE} is missing: build() compiles tests/cuda/wgmma_f16_accum_probe.cu into it")
    lib = ctypes.CDLL(str(PROBE))
    lib.uml_probe_wgmma_f16.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    lib.uml_probe_wgmma_f16.restype = ctypes.c_int
    torch.cuda.init()

    def run(a, b):
        a = np.ascontiguousarray(a, dtype=np.float32)
        b = np.ascontiguousarray(b, dtype=np.float32)
        n, k = b.shape
        assert a.shape == (64, k) and k % 16 == 0
        d = np.empty((64, n), dtype=np.float32)
        rc = lib.uml_probe_wgmma_f16(a.ctypes.data, b.ctypes.data, d.ctypes.data, n, k // 16)
        assert rc == 0, f"probe launch failed: cudaError {rc}"
        return d

    return run


def f16(x):
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def worst_ratio(probe, a, b):
    a, b = f16(a), f16(b)
    assert np.all(np.isfinite(a)) and np.all(np.isfinite(b))
    d = probe(a, b).astype(np.float64)
    worst = 0.0
    for i in range(a.shape[0]):
        for j in range(b.shape[0]):
            p = a[i] * b[j]  # exact
            exact = math.fsum(p)
            budget = sum(np.abs(p[: 16 * (s + 1)]).sum() for s in range(a.shape[1] // 16))
            err = abs(d[i, j] - exact)
            if budget == 0.0:
                assert err == 0.0
                continue
            worst = max(worst, err / (U * budget))
    return worst


def families(rng, n, k):
    def spread():
        return (rng.standard_normal((64, k)) * np.exp2(rng.integers(-8, 9, (64, k))),
                rng.standard_normal((n, k)) * np.exp2(rng.integers(-8, 9, (n, k))))

    def dominant():
        a = rng.standard_normal((64, k))
        a[:, ::16] *= 1024.0
        return a, rng.standard_normal((n, k))

    def cancellation():
        a = np.abs(rng.standard_normal((64, k))) * 16
        b = rng.standard_normal((n, k))
        b[:, 1::2] = -b[:, 0::2] * (1 + rng.integers(-4, 5, (n, k // 2)) * 2.0**-10)
        return a, b

    def large_accumulator():
        a = np.abs(rng.standard_normal((64, k))) * 16
        b = rng.standard_normal((n, k)) * 2.0**-12
        b[:, :16] = rng.standard_normal((n, 16)) * 2.0**12
        return a, b

    def subnormal():
        a = rng.integers(1, 1024, (64, k)) * 2.0**-24  # subnormal features
        a[:, ::3] = rng.integers(0, 17, (64, len(range(0, k, 3))))
        b = rng.standard_normal((n, k)) * 2.0**14
        b[:, 1::2] = rng.integers(-1023, 1024, (n, k // 2)) * 2.0**-24  # subnormal lo pieces
        return a, b

    return {"spread": spread, "dominant": dominant, "cancellation": cancellation,
            "large_accumulator": large_accumulator, "subnormal": subnormal}


@pytest.mark.parametrize("n", [16, 32])
@pytest.mark.parametrize("family", ["spread", "dominant", "cancellation", "large_accumulator", "subnormal"])
def test_f16_accumulation_inside_budget(probe, family, n):
    rng = np.random.default_rng(zlib.crc32(f"{family}{n}".encode()))
    worst = 0.0
    for steps in range(1, STEPS + 1):
        a, b = families(rng, n, 16 * steps)[family]()
        worst = max(worst, worst_ratio(probe, a, b))
    print(f"f16 wgmma {family} n={n}: worst error {worst:.3f} u per step of the running |.| sum")
    assert worst * 4 <= BUDGET_PER_STEP, (family, worst)
