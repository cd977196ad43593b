import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "reference: needs the reference tree (OVC_REFERENCE, or the oracle/_ref copy)")


def pytest_collection_modifyitems(config, items):
    from oracle import refboot

    have_ref = refboot.available()
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    for item in items:
        if "reference" in item.keywords and not have_ref:
            item.add_marker(pytest.mark.skip(reason="reference tree not present"))
        if "gpu" in item.keywords and not have_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))


@pytest.fixture(scope="session", autouse=True)
def _native_artifacts():
    """Build the CUDA library (nvcc cross-compiles without a GPU) and the C oracle if they are missing or
    older than their sources, so the suites do not depend on build() having been called first."""
    from oracle import cpu as oracle_cpu
    from overcooked_ai_b200 import build as native_build

    oracle_cpu.build()
    try:
        native_build.build()
    except Exception as e:  # no nvcc on this box: the prebuilt in-tree .so must already be there
        if not os.path.exists(native_build.OUT):
            raise RuntimeError("libovc_b200.so is missing and could not be built: %s" % e)
    yield
