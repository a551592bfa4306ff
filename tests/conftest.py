import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "visual-chinese-llama-alpaca_b200")
for p in (ROOT, PKG, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True)
def _device_hang_watchdog(request):
    """A hung CUDA kernel blocks inside a C call where pytest-timeout cannot interrupt: dump the stack and exit instead
    of burning GPU-box minutes."""
    import faulthandler
    if "gpu" not in request.keywords:
        yield
        return
    limit = int(os.environ.get("VCLA_TEST_WATCHDOG", "420"))
    faulthandler.dump_traceback_later(limit, exit=True)
    try:
        yield
    finally:
        faulthandler.cancel_dump_traceback_later()
