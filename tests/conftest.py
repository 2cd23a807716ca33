import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests are skipped (not failed) on a box without a CUDA device, so a plain `pytest` works anywhere."""
    try:
        import build_native
        build_native.build(verbose=False)
        from wide_deep_b200 import _native
        have_gpu = _native.lib().wd_device_count() > 0
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (wd_device_count() == 0)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def native_lib():
    """libwd_b200.so, built in-tree if missing (nvcc cross-compiles without a GPU)."""
    import build_native
    build_native.build(verbose=False)
    from wide_deep_b200 import _native
    return _native.lib()
