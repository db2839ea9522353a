"""pytest configuration: the `gpu` marker and session-level builds.

`-m "not gpu"` tests run in the build container (no GPU): oracle vs golden vectors, host logic,
and that the C-ABI library loads and exports every declared symbol.  `-m gpu` tests are the
parity tests proper (CUDA path vs oracle / golden) and run on an H100.
"""
import os
import sys

import pytest

os.environ.setdefault("SIGE_FUSED_STRICT", "1")      # a lowering bug must fail a test, not fall back silently
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device AND the built library: skip them (loudly) anywhere else, e.g. a plain `pytest tests`
    in the build container."""
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100): pytest -m gpu")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def cabi_lib():
    """Path of libsige_b200.so (built on demand when nvcc is available)."""
    from sige_b200 import build as b

    if not b.up_to_date() and os.path.isfile(b.NVCC):
        b.build()
    assert os.path.isfile(b.LIB_PATH), "libsige_b200.so missing and nvcc unavailable"
    return b.LIB_PATH


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O

    O.build()
    return O


@pytest.fixture(scope="session")
def ref_cpu():
    """The reference's own compiled CPU backend (oracle/_ref), or None if it did not travel."""
    from oracle.build_ref import load_ref

    try:
        return load_ref()
    except Exception:  # noqa: BLE001
        return None


def golden(name):
    import numpy as np

    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)
