"""Measured error of the Hopper tf32 wgmma accumulation against the budget the tensor-core MLP bound assumes.

`mlp_argmax_tc_kernel` certifies a row when its logit margin exceeds an error bound that budgets 32u (u = 2^-24) of the
running absolute sum per accumulating m64nNk8 step (DESIGN.md 3.3).  That figure comes from a model of the hardware
(a truncating aligner without guard bits: 20u).  Here the product's own `WgmmaTf32<N>::mma` runs on chosen operands
(tests/cuda/wgmma_accum_probe.cu, a test-only library built by `build()`), and every element of D is compared with
the exact sum: tf32 x tf32 products are exact in float64, and `math.fsum` rounds their sum once.

For each element the error is divided by u * sum_s S_s, where S_s is the sum of |a_k b_k| over the first s + 1 steps:
the per-step budget of the bound, so a ratio <= 32 is what the kernel assumes.  Below FLT_MIN the budget is absolute:
the bound allows FLT_MIN per product and per step result (a flush), and the probe records what the hardware does.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

PROBE = ROOT / "build" / "tests" / "libwgmma_accum_probe.so"
U = 2.0**-24
FLT_MIN = 2.0**-126
BUDGET_PER_STEP = 32  # mlp_tc_kernels.cu: e1_scale = (32 n_mma + 12) u ...


@pytest.fixture(scope="module")
def probe():
    if not PROBE.exists():
        pytest.fail(f"{PROBE} is missing: build() compiles tests/cuda/wgmma_accum_probe.cu into it")
    lib = ctypes.CDLL(str(PROBE))
    lib.uml_probe_wgmma_tf32.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    lib.uml_probe_wgmma_tf32.restype = ctypes.c_int
    torch.cuda.init()

    def run(a, b):
        a = np.ascontiguousarray(a, dtype=np.float32)
        b = np.ascontiguousarray(b, dtype=np.float32)
        n, k = b.shape
        assert a.shape == (64, k) and k % 8 == 0
        d = np.empty((64, n), dtype=np.float32)
        rc = lib.uml_probe_wgmma_tf32(a.ctypes.data, b.ctypes.data, d.ctypes.data, n, k // 8)
        assert rc == 0, f"probe launch failed: cudaError {rc}"
        return d

    return run


def tf32(x):
    """Round to the nearest tf32 value (10 mantissa bits), as mlp_tc_build_w1_tiles does."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def spread(rng, shape, lo, hi):
    """tf32 values with random signs and exponents uniform in [lo, hi]."""
    m = rng.uniform(1.0, 2.0, size=shape) * rng.choice([-1.0, 1.0], size=shape)
    return tf32(np.ldexp(m, rng.integers(lo, hi + 1, size=shape)))


def exact_and_scale(a, b):
    """Exact D (fsum of exact products) and u * sum_s S_s per element."""
    p = a.astype(np.float64)[:, None, :] * b.astype(np.float64)[None, :, :]  # exact: 11 x 11 mantissa bits
    d = np.array([[math.fsum(p[r, c]) for c in range(p.shape[1])] for r in range(p.shape[0])])
    running = np.cumsum(np.abs(p), axis=2)[:, :, 7::8]  # S_s after each k8 step
    return d, U * running.sum(axis=2)


def family(name, rng, k):
    if name == "spread_2^+-30":  # products spread over 2^+-30
        return spread(rng, (64, k), -15, 15), lambda n: spread(rng, (n, k), -15, 15)
    if name == "one_large_seven_small":  # per k8 group one product 2^22 above the other seven: aligner truncation
        a = spread(rng, (64, k), -3, 3)
        big = np.zeros(k, dtype=bool)
        big[np.arange(0, k, 8) + rng.integers(0, 8, size=k // 8)] = True

        def b(n):
            v = spread(rng, (n, k), -3, 3)
            v[:, ~big] = tf32(v[:, ~big] * np.float32(2.0**-22))
            return v

        return a, b
    if name == "cancellation":  # pairs +p, -p(1 + d) inside each group: results far below the addends
        a = spread(rng, (64, k), 0, 4)
        a[:, 1::2] = a[:, 0::2]

        def b(n):
            v = spread(rng, (n, k), 0, 4)
            v[:, 1::2] = tf32(-v[:, 0::2] * (1 + np.ldexp(rng.integers(1, 64, size=(n, k // 2)), -10)).astype(np.float32))
            return v

        return a, b
    if name == "large_accumulator":  # step 0 leaves ~2^20 in D, later steps add 2^-10..2^0
        a = spread(rng, (64, k), -5, 0)
        a[:, :8] = spread(rng, (64, 8), 9, 10)

        def b(n):
            v = spread(rng, (n, k), -5, 0)
            v[:, :8] = spread(rng, (n, 8), 9, 10)
            return v

        return a, b
    raise KeyError(name)


@pytest.mark.parametrize("n", [64, 32])
def test_fragment_layout(probe, n):
    """D[r][c] = r * n + c exactly: a permuted fragment store (or descriptor) fails here at once."""
    for steps in (1, 5, 16):
        a = np.zeros((64, 8 * steps), np.float32)
        b = np.zeros((n, 8 * steps), np.float32)
        s = steps - 1  # the operands sit in the last step; earlier steps add zeros
        a[:, 8 * s] = np.arange(64)
        a[:, 8 * s + 3] = 1.0
        b[:, 8 * s] = n
        b[:, 8 * s + 3] = np.arange(n)
        np.testing.assert_array_equal(probe(a, b), np.arange(64)[:, None] * n + np.arange(n)[None, :])


@pytest.mark.parametrize("n", [64, 32])
@pytest.mark.parametrize("name", ["spread_2^+-30", "one_large_seven_small", "cancellation", "large_accumulator"])
def test_accumulation_error_within_the_budget(probe, n, name):
    worst = 0.0
    for seed, steps in enumerate((2, 8, 16) * 4):
        rng = np.random.default_rng(1000 * seed + n)
        a, bf = family(name, rng, 8 * steps)
        b = bf(n)
        d = probe(a, b).astype(np.float64)
        want, scale = exact_and_scale(a, b)
        ratio = np.abs(d - want) / scale  # error per u of the summed running |.| sums
        worst = max(worst, float(ratio.max()))
    print(f"\nwgmma m64n{n}k8 tf32 {name}: max error / (u sum_s S_s) = {worst:.3f} (budget {BUDGET_PER_STEP})")
    assert worst <= BUDGET_PER_STEP


@pytest.mark.parametrize("n", [64, 32])
def test_below_flt_min(probe, n):
    """Subnormal tf32 operands, and normal operands whose products fall below FLT_MIN.  Two checks: the result stays
    inside the flush-tolerant absolute budget of the bound (FLT_MIN per product and per step result, FLT_MIN |w| for a
    subnormal operand), and it shows the behaviour DESIGN.md 3.3 records for the H100: nothing is flushed, the error
    stays inside the relative budget.  Hardware that flushes is still covered by the bound; it fails the second check
    so that the record is revisited."""
    rng = np.random.default_rng(7 + n)
    steps = 4
    k = 8 * steps
    out = {}
    # subnormal A (multiples of 2^-136 below 2^-126 are tf32 values), B = 2^20 +- : products ~2^-116, normal
    a = tf32(np.ldexp(rng.integers(1, 1024, size=(64, k)).astype(np.float64) * rng.choice([-1, 1], size=(64, k)), -136))
    assert (np.abs(a) < FLT_MIN).all() and (a != 0).all()
    b = spread(rng, (n, k), 19, 20)
    cases = {"subnormal operands": (a, b)}
    # normal operands, products 2^-140 .. 2^-130
    cases["subnormal products"] = (spread(rng, (64, k), -70, -66), spread(rng, (n, k), -70, -64))
    for label, (a, b) in cases.items():
        d = probe(a, b).astype(np.float64)
        want, scale = exact_and_scale(a, b)
        err = np.abs(d - want)
        flushed = bool(np.all(d == 0.0))
        kept = bool(np.all(err <= scale * BUDGET_PER_STEP))
        out[label] = "flushed to zero" if flushed else ("kept (within the relative budget)" if kept else "partly lost")
        print(f"\nwgmma m64n{n}k8 tf32 {label}: {out[label]}; max |err| = {err.max():.3e} = {err.max() / FLT_MIN:.3f} FLT_MIN")
        # what mlp_tc_kernels.cu budgets below FLT_MIN: 8 products + the step result per step, FLT_MIN each, and a
        # subnormal operand x at most FLT_MIN |w| (the w1max_f FLT_MIN terms)
        operand = FLT_MIN * np.abs(b.astype(np.float64)).sum(axis=1)[None, :]
        assert np.all(err <= scale * BUDGET_PER_STEP + 9 * steps * FLT_MIN + operand)
        assert kept, f"{label}: {out[label]}, but DESIGN.md 3.3 records that the tensor cores keep subnormals"
