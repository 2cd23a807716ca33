"""Host-side part of the owner's HBM cache of host shard records: Plan(shard_cache_bytes=...), the estimator keyword and the
C-ABI entry point."""
import ctypes

import pytest

from tests.test_abi import header_symbols
from tests.test_gpu_parity import small_conf
from wide_deep_b200.plan import Plan


def _sharded(**kw):
    fc, cross, model = small_conf()
    return Plan(fc, cross, model, "wide_deep", max_batch=64, max_nnz=64 * 64, max_keys=64 * 64, dense_exchange_max_rows=30,
                shard_world=2, shard_rank=1, shard_slack=2.0, **kw)


def test_shard_cache_bytes_is_validated():
    assert _sharded().shard_cache_bytes == 0
    assert _sharded(host_tables="all", shard_cache_bytes=1 << 30).shard_cache_bytes == 1 << 30
    for bad in (-1, 1.5, "1G", None, True):
        with pytest.raises(ValueError, match="shard_cache_bytes must be an int >= 0"):
            _sharded(shard_cache_bytes=bad)


def test_shard_cache_needs_a_sharded_plan():
    fc, cross, model = small_conf()
    assert Plan(fc, cross, model, shard_cache_bytes=0).shard_cache_bytes == 0
    with pytest.raises(ValueError, match="host_cache_bytes"):
        Plan(fc, cross, model, host_tables="all", shard_cache_bytes=1 << 20)


def test_plan_descriptor_does_not_change():
    """The budget reaches the library through wd_shard_cache_enable, not through WdPlanDesc."""
    plain, keep_a = _sharded(host_tables="all").to_c()
    cached, keep_b = _sharded(host_tables="all", shard_cache_bytes=1 << 24).to_c()
    for name, ctype in type(plain)._fields_:
        if issubclass(ctype, (ctypes._Pointer, ctypes.c_void_p)):
            continue
        a, b = getattr(plain, name), getattr(cached, name)
        assert (a == b) if isinstance(a, (int, float)) else bytes(a) == bytes(b), name      # (bytes: the optimizer structs)
    # the arrays the pointers point at (kept alive beside the descriptor) hold the same bytes
    assert len(keep_a) == len(keep_b)
    for a, b in zip(keep_a, keep_b):
        assert bytes(memoryview(a)) == bytes(memoryview(b))


def test_estimator_takes_shard_cache_bytes(tmp_path):
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import build_custom_estimator
    est = build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, shard_world=2, shard_rank=0,
                                 host_tables="all", shard_cache_bytes=4096)
    assert est.plan.shard_cache_bytes == 4096
    with pytest.raises(ValueError):
        build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, shard_cache_bytes=4096)


def test_shard_cache_entry_point_is_declared_bound_and_exported(native_lib):
    from wide_deep_b200 import _native
    assert "wd_shard_cache_enable" in header_symbols() and "wd_shard_cache_enable" in _native.SYMBOLS
    assert hasattr(native_lib, "wd_shard_cache_enable")
    # a null model is refused without touching a device
    assert native_lib.wd_shard_cache_enable(None, 0) == _native.EINVAL
