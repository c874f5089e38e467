import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


@pytest.fixture(scope="session")
def lib():
    """The in-tree C-ABI library (built on demand; loading never needs a device)."""
    from tensorrt_laboratory_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return capi.load()


@pytest.fixture(scope="session")
def gpu(lib):
    from tensorrt_laboratory_b200 import capi
    if capi.device_count() < 1:
        pytest.fail("test marked gpu but no CUDA device is visible (no CPU fallback exists)")
    info = capi.device_info(0)
    assert tuple(info["cc"]) == (9, 0), f"expected an sm_90 device, found {info}"
    return info
