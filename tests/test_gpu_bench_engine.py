"""Parity of the engines bench.py runs (bf16x3, and the fp32-faithful tc3x) on the benchmark's own shape, at the north_star bar.

BASELINE.json north_star: fp32 logits within 1e-4 relative.  The benchmark model is the Criteo shape (845-wide deep input,
towers 1024-512-256, relu + BN affine, Adagrad / FTRL); here with every table scaled by 1e-3 so the oracle finishes in
seconds — the towers, the kernels and the tile shapes are the benchmark's.

  1. identical parameters: |gpu - oracle| <= 1e-4 * max(|oracle|, 1) on the logits of 3 x 2048 examples.
  2. 50 training steps in the settled regime ("warm": the oracle alone walks through the first ten steps, its state is copied
     to the GPU model, then both train 50 steps on the same batches): the loss of EVERY step within 1e-4 relative and the
     logits of a fresh batch after the run within 5e-4.
  3. 50 training steps from the TF initialisers ("init").  With the reference's SUM-reduced loss and Adagrad(0.05) the first
     steps of this synthetic configuration are a violent transient (oracle losses 1.5e3 -> 4.2e5 -> 1.6e4 -> 4.9e2 -> 4.7e3
     ...) that amplifies ANY rounding difference by three orders of magnitude: the exact-fp32 FFMA engine — which differs
     from the float64-accumulating oracle only in summation order — already drifts past 1e-4 on a step loss and on
     fresh logits (tests/engine_drift_report.py prints both).  No fp32 implementation can hold 1e-4 there, so the bound asserted for
     the tensor-core engines is relative to that floor: within 10x the drift the FFMA engine shows on the same run
     (the test prints both ratios) — bounded, not waived.
Both engines also assert that no GEMM fell back to the FFMA kernel."""
import numpy as np
import pytest

from oracle import model as OM
from tests.helpers import copy_params_to_product
from wide_deep_b200 import synthetic
from wide_deep_b200.model import Batch, WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu
B = 2048
_FC = None


def _conf():
    global _FC
    if _FC is None:
        _FC = synthetic.criteo_conf(scale=1e-3)
    return _FC


def _batch(step, zipf=None):
    fc = _conf()[0]
    cats = [f for f, c in fc.items() if c["type"] == "category"]
    dn = [f for f, c in fc.items() if c["type"] == "continuous"]
    keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=step, zipf=zipf)
    raw = {f: (np.arange(B + 1, dtype=np.int64), np.ascontiguousarray(keys[:, j])) for j, f in enumerate(cats)}
    for j, f in enumerate(dn):
        raw[f] = np.ascontiguousarray(dense[:, j])
    return raw, label, Batch(B, keys.reshape(-1), None, dense, label)


def _oracle(seed, warm=0):
    fc, cross, model, emb = _conf()
    om = OM.OracleModel(fc, cross, model, "wide_deep", embedding_dim_override=emb).init(seed)
    for s in range(warm):
        raw, label, _ = _batch(1000 + s)
        om.train_step(raw, label)
    return om


def _product(om, engine):
    fc, cross, model, emb = _conf()
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, gemm_engine=engine,
                max_nnz=B * (len(fc) + len(cross)), max_keys=B * n_cat)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    return pm


def _run50(engine, warm):
    """-> (worst relative step-loss error, max relative logit error on a fresh batch after the run)"""
    om = _oracle(11, warm)
    pm = _product(om, engine)
    worst = 0.0
    for step in range(50):
        raw, label, b = _batch(step)
        loss = pm.train_step(b)
        ref, _ = om.train_step(raw, label)
        worst = max(worst, abs(loss - ref) / max(abs(ref), 1.0))
    raw, label, b = _batch(999)
    logits, _ = pm.forward(b)
    _, cache = om.forward(raw)
    ref = cache["logits"]
    err = float((np.abs(logits - ref) / np.maximum(np.abs(ref), 1.0)).max())
    assert pm.gemm_fallback_count() == 0
    pm.close()
    return worst, err


@pytest.mark.parametrize("engine", ["bf16x3", "tc3x"])
def test_bench_shape_logits_at_the_bar(engine):
    om = _oracle(7)
    pm = _product(om, engine)
    worst = 0.0
    for step in (123, 124, 125):
        raw, label, b = _batch(step, zipf=1.1 if step == 124 else None)
        logits, _ = pm.forward(b)
        _, cache = om.forward(raw)
        ref = cache["logits"]
        worst = max(worst, float((np.abs(logits - ref) / np.maximum(np.abs(ref), 1.0)).max()))
    print("engine %s: max relative logit error %.3g on %d examples" % (engine, worst, 3 * B))
    assert worst <= 1e-4, worst
    assert pm.gemm_fallback_count() == 0


@pytest.mark.parametrize("engine", ["bf16x3", "tc3x"])
def test_bench_shape_50_step_drift_settled_regime(engine):
    worst, err = _run50(engine, warm=10)
    print("engine %s, 50 steps from a warmed-up state: worst step-loss error %.3g, fresh-batch logit error %.3g" % (engine, worst, err))
    assert worst <= 1e-4, worst
    assert err <= 5e-4, err


def test_bench_shape_50_step_drift_from_init_is_within_the_fp32_envelope():
    floor_loss, floor_err = _run50("ffma", warm=0)                 # exact fp32 products; differs from the oracle in summation order only
    print("ffma (fp32 floor), 50 steps from init: worst step-loss error %.3g, fresh-batch logit error %.3g" % (floor_loss, floor_err))
    for engine in ("tc3x", "bf16x3"):
        worst, err = _run50(engine, warm=0)
        print("engine %s, 50 steps from init: worst step-loss error %.3g (%.1fx the fp32 floor), fresh-batch logit error %.3g (%.1fx)" % (
            engine, worst, worst / max(floor_loss, 1e-12), err, err / max(floor_err, 1e-12)))
        assert worst <= max(1e-4, 10.0 * floor_loss), (engine, worst, floor_loss)
        assert err <= max(5e-4, 10.0 * floor_err), (engine, err, floor_err)


def test_bench_shape_parameters_after_two_steps():
    """Every trained tensor of the bf16x3 engine on the benchmark towers (B = 2048: the fused logits-layer / activation
    backward, and the activation / batch-norm backward of the other hidden layers) against the oracle: bias / gamma / beta
    gradients come from column partials, so a wrong partial shows up here at once."""
    om = _oracle(23, warm=3)
    pm = _product(om, "bf16x3")
    for step in range(2):
        raw, label, b = _batch(step)
        loss = pm.train_step(b)
        ref, _ = om.train_step(raw, label)
        assert abs(loss - ref) <= 1e-4 * max(abs(ref), 1.0), (step, loss, ref)
    worst = ("", 0.0)
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        scale = max(float(np.abs(exp).max()), 1e-3)
        err = float(np.max(np.abs(got - exp))) / scale
        if err > worst[1]:
            worst = (name, err)
        assert err <= 2e-3, "%s: %g of scale %g" % (name, err, scale)
    print("worst tensor after 2 steps: %s, %.3g of its scale" % worst)
    assert pm.gemm_fallback_count() == 0
