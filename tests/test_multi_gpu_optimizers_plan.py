"""Host side of Adam / RMSProp on the multi-GPU paths: Plan accepts them for row-sharded models and with the dense exchange of small
tables, for both optimizers.  (Adam with a host-placed shard is refused by the library when the model is created:
tests/test_gpu_multi_gpu_optimizers.py::test_adam_with_host_placed_shard_is_refused.)"""
import pytest

from tests.test_gpu_parity import small_conf
from wide_deep_b200.plan import Plan

OPTS = ["Adam", "RMSProp", "tf.train.AdamOptimizer(0.002, beta1=0.8)", "tf.train.RMSPropOptimizer(learning_rate=0.001,decay=0.8,momentum=0.5)"]


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("which", ["lin_opt", "dnn_opt"])
@pytest.mark.parametrize("kw", [dict(dense_exchange_max_rows=400), dict(dense_exchange_max_rows=400, shard_world=2, shard_rank=1)])
def test_plan_accepts_adam_and_rmsprop_on_multi_gpu_paths(opt, which, kw):
    fc, cross, model = small_conf(**{which: opt})
    plan = Plan(fc, cross, model, "wide_deep", max_batch=64, **kw)
    assert getattr(plan, which)["kind"] == ("adam" if "Adam" in opt else "rmsprop")
    assert plan.dense_exchange_max_rows == 400
    if "shard_world" in kw:
        assert any(plan.is_sharded_tensor(n) for n in plan.tensor_names)
