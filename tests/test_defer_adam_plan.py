"""Host-side part of deferred Adam tables: Plan(defer_adam=...) -> the WD_PLACE_DEFER_ADAM bit of WdPlanDesc::table_placement,
the summary, the estimator keyword and the C-ABI entry point of its counters."""
import ctypes

from tests.test_abi import header_symbols
from tests.test_gpu_parity import small_conf
from wide_deep_b200.plan import API_VERSION, PLACE_AUTO, PLACE_DEFER_ADAM, PLACE_HBM, PLACE_HOST, Plan, PlanDescC


def _placement(plan):
    d, keep = plan.to_c()
    assert d.api_version == API_VERSION == 3
    p = ctypes.cast(d.table_placement, ctypes.POINTER(ctypes.c_uint8))
    return [p[i] for i in range(len(plan.tables))], keep


def test_defer_bit_is_set_on_host_and_auto_entries_only():
    fc, cross, model = small_conf(dnn_opt="Adam")
    names = [t["name"] for t in Plan(fc, cross, model).tables]
    assert PLACE_DEFER_ADAM == 4
    got, _ = _placement(Plan(fc, cross, model, defer_adam=True))
    assert got == [PLACE_AUTO | PLACE_DEFER_ADAM] * len(names)
    got, _ = _placement(Plan(fc, cross, model, host_tables="all", defer_adam=True))
    assert got == [PLACE_HOST | PLACE_DEFER_ADAM] * len(names)
    got, _ = _placement(Plan(fc, cross, model, host_tables=[], defer_adam=True))
    assert got == [PLACE_HBM] * len(names)
    pick = ["h3_embedding", names[0]]
    plan = Plan(fc, cross, model, host_tables=pick, defer_adam=True)
    got, _ = _placement(plan)
    assert got == [(PLACE_HOST | PLACE_DEFER_ADAM) if n in pick else PLACE_HBM for n in names]
    s = plan.summary()["placement"]
    assert list(s) == names and all(s[n] == ("host+defer" if n in pick else "hbm") for n in names)
    assert set(Plan(fc, cross, model, defer_adam=True).summary()["placement"].values()) == {"auto+defer"}
    # off by default: the placement of every existing plan is unchanged
    got, _ = _placement(Plan(fc, cross, model, host_tables=pick))
    assert got == [PLACE_HOST if n in pick else PLACE_HBM for n in names]
    assert PlanDescC._fields_[-1][0] == "table_placement"


def test_estimator_takes_defer_adam(tmp_path):
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import build_custom_estimator
    est = build_custom_estimator(str(tmp_path), "wide_deep", config=Config(), max_batch=64, host_tables="all", defer_adam=True)
    assert set(est.plan.summary()["placement"].values()) == {"host+defer"}
    est = build_custom_estimator(str(tmp_path / "b"), "wide_deep", config=Config(), max_batch=64, host_tables="all")
    assert set(est.plan.summary()["placement"].values()) == {"host"}


def test_deferred_adam_stats_is_declared_bound_and_exported(native_lib):
    from wide_deep_b200 import _native
    assert "wd_deferred_adam_stats" in header_symbols()
    assert "wd_deferred_adam_stats" in _native.SYMBOLS
    assert hasattr(native_lib, "wd_deferred_adam_stats")
    out = (ctypes.c_int64 * 4)()
    assert native_lib.wd_deferred_adam_stats(None, out, 4, 0) == _native.EINVAL      # null model: refused without a device
