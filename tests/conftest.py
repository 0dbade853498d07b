import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on the H100 box)")


def rel_err(got: np.ndarray, ref: np.ndarray) -> float:
    """The parity metric of BASELINE.md: max|got - ref| / max|ref| over one blob."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    denom = max(float(np.abs(ref).max()), 1e-30)
    return float(np.abs(got - ref).max()) / denom


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build(ref=True)
    return O


@pytest.fixture(scope="session")
def restatement(oracle):
    return oracle.restatement()


@pytest.fixture(scope="session")
def reference(oracle):
    if not oracle.reference_available():
        pytest.skip("oracle/_ref/libfeather_ref.so not built (needs /root/reference at build time)")
    return oracle.Reference()


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("models")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


@pytest.fixture(autouse=True)
def _default_precision():
    """Every test starts in the engine's default arithmetic mode (FP32_SPLIT); tests that pin a mode set it themselves."""
    try:
        from feathercnn_b200 import booster
        booster.set_precision(booster.PRECISION_FP32_SPLIT)
    except Exception:  # libraries not built (pure-oracle CPU tests)
        pass
    yield
