import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _gpu_available() -> bool:
    """True when the CUDA library is built and hs_engine_create finds a device (no torch import needed)."""
    try:
        from happysim_b200 import engine
        e = engine.Engine(0)
        e.close()
        return True
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """Plain `pytest` on a host without a CUDA device skips the gpu-marked tests instead of erroring;
    `-m gpu` on such a host still reports them as skipped, never as passed."""
    gpu_items = [it for it in items if "gpu" in it.keywords]
    if not gpu_items or _gpu_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device (hs_engine_create: HS_ERR_NO_DEVICE) or libhs_b200.so not built")
    for it in gpu_items:
        it.add_marker(skip)
