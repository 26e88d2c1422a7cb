"""pytest configuration: the ``gpu`` marker and shared fixtures (golden digits model, seeded batches)."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def digits_model():
    """coef (10x64 f64), intercept (10), classes (10) of the golden digits LogisticRegression."""
    z = np.load(GOLDEN / "digits_lr.npz")
    return {"coef": z["coef"], "intercept": z["intercept"], "classes": z["classes"]}


@pytest.fixture(scope="session")
def known_answer():
    return json.loads((GOLDEN / "known_answer.json").read_text())


@pytest.fixture(scope="session")
def synthetic_digits():
    z = np.load(GOLDEN / "synthetic_digits_4096.npz")
    return {k: z[k] for k in z.files}


@pytest.fixture(scope="session")
def binary_mock():
    z = np.load(GOLDEN / "binary_mock.npz")
    return {k: z[k] for k in z.files}


def digits_batch(seed: int, rows: int, dtype=np.float32) -> np.ndarray:
    """cfg-2 style synthetic rows (SURVEY.md 8d): integers 0..16, exactly representable in fp32."""
    return np.random.default_rng(seed).integers(0, 17, size=(rows, 64), dtype=np.uint8).astype(dtype)
