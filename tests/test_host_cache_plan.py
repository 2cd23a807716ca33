"""Host-side part of the HBM cache of host-table records: Plan(host_cache_bytes=...), the estimator keyword and the C-ABI."""
import pytest

from tests.test_abi import header_symbols
from tests.test_gpu_parity import small_conf
from wide_deep_b200.plan import Plan


def test_host_cache_bytes_is_validated():
    fc, cross, model = small_conf()
    assert Plan(fc, cross, model).host_cache_bytes == 0
    assert Plan(fc, cross, model, host_tables="all", host_cache_bytes=1 << 30).host_cache_bytes == 1 << 30
    for bad in (-1, 1.5, "1G", None, True):
        with pytest.raises(ValueError, match="host_cache_bytes must be an int >= 0"):
            Plan(fc, cross, model, host_cache_bytes=bad)


def test_estimator_takes_host_cache_bytes(tmp_path):
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import build_custom_estimator
    est = build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, host_tables="all", host_cache_bytes=4096)
    assert est.plan.host_cache_bytes == 4096
    with pytest.raises(ValueError):
        build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, host_cache_bytes=-5)


def test_cache_entry_points_are_declared_bound_and_exported(native_lib):
    from wide_deep_b200 import _native
    for name in ("wd_host_cache_enable", "wd_host_cache_stats"):
        assert name in header_symbols() and name in _native.SYMBOLS and hasattr(native_lib, name)
    # a null model is refused without touching a device
    assert native_lib.wd_host_cache_enable(None, 0) == _native.EINVAL
    assert native_lib.wd_host_cache_stats(None, None, 0, 0) == _native.EINVAL
