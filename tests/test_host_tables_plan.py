"""Host-side part of table placement: Plan(host_tables=...) -> WdPlanDesc::table_placement, and the C-ABI entry point."""
import ctypes

import pytest

from tests.test_abi import header_symbols
from tests.test_gpu_parity import small_conf
from wide_deep_b200.plan import API_VERSION, PLACE_AUTO, PLACE_HBM, PLACE_HOST, Plan


def _placement(plan):
    d, keep = plan.to_c()
    assert d.api_version == API_VERSION == 3
    p = ctypes.cast(d.table_placement, ctypes.POINTER(ctypes.c_uint8))
    return [p[i] for i in range(len(plan.tables))], keep


def test_placement_flags_are_packed_per_table():
    fc, cross, model = small_conf()
    names = [t["name"] for t in Plan(fc, cross, model).tables]
    assert len(names) >= 4 and "h3_embedding" in names
    got, _ = _placement(Plan(fc, cross, model))
    assert got == [PLACE_AUTO] * len(names)
    got, _ = _placement(Plan(fc, cross, model, host_tables="all"))
    assert got == [PLACE_HOST] * len(names)
    got, _ = _placement(Plan(fc, cross, model, host_tables=[]))
    assert got == [PLACE_HBM] * len(names)
    pick = ["h3_embedding", names[0]]
    plan = Plan(fc, cross, model, host_tables=pick)
    got, _ = _placement(plan)
    assert got == [PLACE_HOST if n in pick else PLACE_HBM for n in names]
    s = plan.summary()["placement"]
    assert list(s) == names and all(s[n] == ("host" if n in pick else "hbm") for n in names)
    assert set(Plan(fc, cross, model).summary()["placement"].values()) == {"auto"}


def test_placement_field_is_last_in_the_descriptor():
    from wide_deep_b200.plan import PlanDescC
    assert PlanDescC._fields_[-1][0] == "table_placement"


def test_host_tables_argument_is_validated():
    fc, cross, model = small_conf()
    with pytest.raises(ValueError, match="no embedding table named"):
        Plan(fc, cross, model, host_tables=["h3_embedding", "nope_embedding"])
    with pytest.raises(ValueError, match="host_tables must be"):
        Plan(fc, cross, model, host_tables="some")
    # a wide-only model has no embedding tables to place
    with pytest.raises(ValueError, match="no embedding table named"):
        Plan(fc, cross, model, "wide", host_tables=["h3_embedding"])
    assert Plan(fc, cross, model, "wide", host_tables="all").tables == []


def test_estimator_takes_host_tables(tmp_path):
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import build_custom_estimator
    est = build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, host_tables="all")
    assert set(est.plan.summary()["placement"].values()) == {"host"}


def test_memory_usage_is_declared_bound_and_exported(native_lib):
    from wide_deep_b200 import _native
    assert "wd_memory_usage" in header_symbols()
    assert "wd_memory_usage" in _native.SYMBOLS
    assert hasattr(native_lib, "wd_memory_usage")
    # a null model is refused without touching a device
    assert native_lib.wd_memory_usage(None, None, None) == _native.EINVAL
    assert native_lib.wd_version() == 3
