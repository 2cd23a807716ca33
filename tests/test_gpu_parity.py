"""GPU parity tests proper: the CUDA path (through the C-ABI) against the CPU oracle on the same seeded inputs.

Bars (BASELINE.json north_star): hashed-cross ids and bucketised ids BIT-EXACT; fp32 logits within 1e-4
relative.  "Relative" is implemented as |gpu - oracle| <= 1e-4 * max(|oracle|, 1) for logits (the head adds
O(1) terms, logits near zero have no meaningful relative error), and the same bound scaled by the tensor's
max magnitude for parameters after training steps.
"""
from collections import OrderedDict

import numpy as np
import pytest

from oracle import model as OM
from tests.helpers import copy_params_to_product, random_raw_batch, to_product_batch
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def small_conf(hidden=(64, 32), mode="simple", act="relu", bn=1, dnn_opt="Adagrad",
               lin_opt="tf.train.FtrlOptimizer(learning_rate=0.1,l1_regularization_strength=0.5,l2_regularization_strength=1)"):
    fc = OrderedDict()
    fc["h1"] = dict(type="category", transform="hash_bucket", parameter=1000)
    fc["h2"] = dict(type="category", transform="hash_bucket", parameter=37)
    fc["h3"] = dict(type="category", transform="hash_bucket", parameter=200000)
    fc["v1"] = dict(type="category", transform="vocab", parameter=[0, 1, 2, 3, 4])
    fc["v2"] = dict(type="category", transform="vocab", parameter=["male", "female"])
    fc["id1"] = dict(type="category", transform="identity", parameter=15)
    fc["x1"] = dict(type="continuous", transform="min_max", parameter=dict(normalization=[10, 90], boundaries=[15, 20, 25, 30, 35, 40, 45, 50]))
    fc["x2"] = dict(type="continuous", transform="standard", parameter=dict(normalization=[40.0, 30.0], boundaries=[-1, 0, 1]))
    fc["x3"] = dict(type="continuous", transform=None, parameter=dict(normalization=None, boundaries=None))
    cross = [(["h1", "h2"], 1000, 1), (["h1", "x1"], 500, 1), (["id1", "x1", "v2"], 100, 1), (["v1", "h3"], 2000, 0),
             (["h2", "id1"], 300, 1)]
    model = dict(linear_optimizer=lin_opt, linear_initial_learning_rate=0.05, dnn_hidden_units=list(hidden),
                 dnn_connected_mode=mode, dnn_optimizer=dnn_opt, dnn_initial_learning_rate=0.05,
                 dnn_activation_function=act, dnn_dropout=None, dnn_batch_normalization=bn)
    return fc, cross, model


def build_pair(fc, cross, model, model_type="wide_deep", B=96, seed=0, tf_compat_pad=False, emb_dim=None, max_batch=None, dense_rows=0,
               engine="ffma"):
    om = OM.OracleModel(fc, cross, model, model_type, embedding_dim_override=emb_dim, tf_compat_pad=tf_compat_pad).init(seed)
    plan = Plan(fc, cross, model, model_type, max_batch=max_batch or B, embedding_dim_override=emb_dim,
                tf_compat_pad=tf_compat_pad, max_nnz=(max_batch or B) * 64, max_keys=(max_batch or B) * 64, gemm_engine=engine,
                dense_exchange_max_rows=dense_rows)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    return om, plan, pm


def check_ids(om, plan, pm, raw, B):
    offs, ids = pm.column_ids()
    ref = om.transform(raw)
    C = len(plan.columns)
    checked = 0
    for ci, col in enumerate(plan.columns):
        if col.name not in ref:
            continue
        ro, ri = ref[col.name]
        for b in range(B):
            s, e = offs[b * C + ci], offs[b * C + ci + 1]
            got = ids[s:e]
            exp = ri[ro[b]:ro[b + 1]]
            assert np.array_equal(got, exp), "column %s row %d: gpu %s oracle %s" % (col.name, b, got, exp)
        checked += 1
    assert checked >= len(om.wide_cols) if om.use_wide else checked > 0


@pytest.mark.parametrize("tf_compat_pad", [False, True])
def test_column_ids_bit_exact(tf_compat_pad):
    fc, cross, model = small_conf()
    rng = np.random.default_rng(1)
    B = 96
    om, plan, pm = build_pair(fc, cross, model, B=B, tf_compat_pad=tf_compat_pad)
    raw = random_raw_batch(fc, B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    pm.forward(to_product_batch(plan, raw, label, tf_compat_pad=tf_compat_pad))
    check_ids(om, plan, pm, raw, B)


@pytest.mark.parametrize("mode", ["simple", "first_dense", "last_dense", "dense", "resnet"])
@pytest.mark.parametrize("model_type", ["wide_deep", "deep", "wide"])
def test_forward_logits(mode, model_type):
    if model_type == "wide" and mode != "simple":
        pytest.skip("wide has no towers")
    fc, cross, model = small_conf(hidden=(64, 48, 32), mode=mode)
    rng = np.random.default_rng(2)
    B = 200
    om, plan, pm = build_pair(fc, cross, model, model_type, B=B, seed=3)
    # give the zero-initialised wide weights some signal
    if om.use_wide:
        for c in om.wide_cols:
            om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
        copy_params_to_product(om, pm)
    raw = random_raw_batch(fc, B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    logits, loss = pm.forward(to_product_batch(plan, raw, label))
    ref, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
    ref_loss = om.loss(cache["logits"], label)
    assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0)
    if om.use_deep:
        X = pm.deep_input(B)
        for name, (lo, po, w) in plan.deep_layout.items():
            np.testing.assert_allclose(X[:, po:po + w], cache["X"][:, lo:lo + w], rtol=1e-5, atol=1e-6, err_msg=name)


def test_log_normaliser():
    """`transform: log` of a continuous feature (reference build_estimator.py:67-68: tf.log(x), natural log, fp32): the deep
    input column and — through its bucketized twin in the wide part — the logits, against the oracle on positive inputs."""
    fc, cross, model = small_conf(hidden=(64, 32))
    fc["x4"] = dict(type="continuous", transform="log", parameter=dict(normalization=[0, 1], boundaries=[0.5, 1.0, 2.0, 3.0, 4.0, 5.0]))   # (the reference needs a list here too: tuple(normalization), build_estimator.py:126)
    rng = np.random.default_rng(5)
    B = 128
    om, plan, pm = build_pair(fc, cross, model, "wide_deep", B=B, seed=9)
    for c in om.wide_cols:
        om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
    copy_params_to_product(om, pm)
    raw = random_raw_batch(fc, B, rng)
    raw["x4"] = np.exp(rng.uniform(-1.0, 6.0, size=B)).astype(np.float32)           # positive, three decades
    logits, _ = pm.forward(to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32)))
    _, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
    lo, po, w = plan.deep_layout["x4"]
    np.testing.assert_allclose(pm.deep_input(B)[:, po:po + w], cache["X"][:, lo:lo + w], rtol=2e-6, atol=1e-6)   # logf vs np.log: <= 2 ulp


@pytest.mark.parametrize("act", ["relu", "sigmoid", "tanh", "elu", "selu", "softplus", "softsign", "leaky_relu", "relu6", "crelu"])
def test_activations_train(act):
    fc, cross, model = small_conf(hidden=(32, 32), act=act)
    _train_compare(fc, cross, model, "wide_deep", steps=2, seed=5)


@pytest.mark.parametrize("engine", ["ffma", "tc3x", "bf16x3"])
@pytest.mark.parametrize("mode,bn,dnn_opt", [("simple", 1, "Adagrad"), ("dense", 0, "Adam"), ("first_dense", 1, "Ftrl")])
def test_crelu_train_parity(engine, mode, bn, dnn_opt):
    """dnn_activation_function crelu (reference model_util.py:45-50, tf.nn.crelu = concat(relu(z), relu(-z))): a layer of u units
    hands 2u features to dropout / batch norm / the next layers; the variables keep the reference's shapes (kernel [in, u],
    bias [u], gamma / beta [2u]).  Forward logits, per-step losses and the trained parameters + optimizer slots against the
    oracle (which concatenates explicitly); Adam and Ftrl move weights under a zero gradient, which the tied half must not see."""
    fc, cross, model = small_conf(hidden=(64, 48), mode=mode, act="crelu", bn=bn, dnn_opt=dnn_opt)
    B = 256
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(21)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, max_nnz=B * 64, max_keys=B * 64, gemm_engine=engine)
    pm = WideDeepModel(plan)
    assert plan.tensor_names["dnn/dnn_1/hiddenlayer_1/kernel"][3] == ((128 if mode == "simple" else plan.d0 + 128), 48)
    if bn:
        assert plan.tensor_names["dnn/dnn_1/hiddenlayer_1/batch_normalization/gamma"][3] == (96,)
    copy_params_to_product(om, pm)
    rng = np.random.default_rng(23)
    tol = 1 if engine != "bf16x3" else 5
    for step in range(3):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        batch = to_product_batch(plan, raw, label)
        if step == 0:
            logits, _ = pm.forward(batch)
            _, cache = om.forward(raw)
            np.testing.assert_array_less(np.abs(logits - cache["logits"]), tol * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
        loss = pm.train_step(batch)
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= tol * RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    ptol = 2e-4 if engine != "bf16x3" else 2e-3
    # Adam's early steps move a weight by lr * m / (sqrt(v) + 1e-8) ~ lr * g / (|g| + 1e-8): elements whose gradient is itself
    # ~1e-8 turn fp32 rounding of g into a visible fraction of lr (0.05 here), so a few elements per thousand may sit outside the
    # band (first GPU run: 3 of 4000 elements of one embedding table, 3.3e-4 of scale); everything else is held exactly to it
    frac = 2e-2 if engine == "bf16x3" else (2e-3 if plan.dnn_opt["kind"] == "adam" else 0.0)
    slot_keys = {"adagrad": ["acc"], "ftrl": ["n", "z"], "adam": ["m", "v"]}[plan.dnn_opt["kind"]]
    problems = []
    for name in pm.tensor_names():
        checks = [(0, None)]
        if name.startswith("dnn/dnn_1/"):
            checks += [(i + 1, k) for i, k in enumerate(slot_keys)]
        for slot, key in checks:
            got = pm.get_tensor(name, slot=slot)
            exp = om.params[name] if key is None else om.slots[name][key]
            assert got.shape == exp.shape, name
            scale = max(float(np.abs(exp).max()), 1e-3)
            err = np.abs(got - exp)
            bad = err > ptol * scale
            if bad.mean() > frac or err.max() > 0.05 * scale:
                problems.append("%s slot %d: %g of the tensor off, max %g (scale %g)" % (name, slot, bad.mean(), err.max(), scale))
    assert not problems, "\n".join(problems)
    # a fresh handle initialises the tied halves too: its first forward is finite and its kernels have the variable's shape
    pm2 = WideDeepModel(plan).init(3)
    assert pm2.get_tensor("dnn/dnn_1/hiddenlayer_0/kernel").shape == (plan.d0, 64)
    assert np.isfinite(pm2.forward(batch)[0]).all()


@pytest.mark.parametrize("mode", ["simple", "first_dense", "last_dense", "dense", "resnet"])
def test_train_steps_modes(mode):
    fc, cross, model = small_conf(hidden=(64, 48, 32), mode=mode)
    _train_compare(fc, cross, model, "wide_deep", steps=3, seed=7)


@pytest.mark.parametrize("model_type,dnn_opt,lin_opt,bn", [
    ("deep", "Adagrad", "Ftrl", 0),
    ("wide", "Adagrad", "Ftrl", 1),
    ("wide_deep", "tf.train.GradientDescentOptimizer(learning_rate=0.00002)", "Adagrad", 1),
    ("wide_deep", "tf.train.FtrlOptimizer(learning_rate=0.05,l1_regularization_strength=0.001,l2_regularization_strength=0.01)", "SGD", 1),
    ("wide_deep", "Adagrad", "tf.train.FtrlOptimizer(learning_rate=0.1,l1_regularization_strength=0.5,l2_regularization_strength=1)", 1),
    # the reference's remaining factory names (model_util.py:84-90): Adam (dense m / v decay over whole tables, TF's sparse Adam)
    # and RMSProp (touched rows only), by name and as tf.train expressions
    ("wide_deep", "Adam", "RMSProp", 1),
    ("deep", "tf.train.AdamOptimizer(learning_rate=0.001)", "Ftrl", 1),
    ("wide", "Adagrad", "Adam", 0),
    ("wide_deep", "tf.train.RMSPropOptimizer(learning_rate=0.001,decay=0.8,momentum=0.5)", "tf.train.AdamOptimizer(0.002, beta1=0.8)", 1),
])
def test_train_steps_optimizers(model_type, dnn_opt, lin_opt, bn):
    fc, cross, model = small_conf(hidden=(64, 32), dnn_opt=dnn_opt, lin_opt=lin_opt, bn=bn)
    _train_compare(fc, cross, model, model_type, steps=3, seed=11)


def test_multi_tower():
    fc, cross, model = small_conf()
    model["dnn_hidden_units"] = [[64, 32], [48, 16, 8]]
    model["dnn_connected_mode"] = ["simple", "dense"]
    _train_compare(fc, cross, model, "wide_deep", steps=2, seed=13)


def test_six_towers():
    """More towers than the four the head kernel once took: the logits layers of all six run in the one head kernel."""
    fc, cross, model = small_conf()
    model["dnn_hidden_units"] = [[64, 32], [48, 16, 8], [32], [40, 24], [16, 16], [24]]
    model["dnn_connected_mode"] = ["simple", "dense", "simple", "dense", "simple", "dense"]
    _train_compare(fc, cross, model, "wide_deep", steps=2, seed=13)


def test_more_than_eight_towers_is_rejected():
    from wide_deep_b200 import _native
    fc, cross, model = small_conf()
    model["dnn_hidden_units"] = [[16]] * 9
    model["dnn_connected_mode"] = "simple"
    plan = Plan(fc, cross, model, "wide_deep", max_batch=64, max_nnz=64 * 64, max_keys=64 * 64, gemm_engine="ffma")
    with pytest.raises(_native.NativeError) as e:
        WideDeepModel(plan)
    assert e.value.code == _native.EUNSUPPORTED
    assert "towers" in str(e.value)


def test_weighted_examples_and_ragged_batch():
    fc, cross, model = small_conf()
    _train_compare(fc, cross, model, "wide_deep", steps=2, seed=17, weighted=True, B=77, max_batch=128)


def _train_compare(fc, cross, model, model_type, steps, seed, weighted=False, B=160, max_batch=None, dense_rows=0):
    rng = np.random.default_rng(seed)
    om, plan, pm = build_pair(fc, cross, model, model_type, B=B, seed=seed, max_batch=max_batch, dense_rows=dense_rows)
    for step in range(steps):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        weight = (rng.random(B).astype(np.float32) + 0.5) if weighted else None
        loss = pm.train_step(to_product_batch(plan, raw, label, weight))
        ref_loss, _ = om.train_step(raw, label, weight)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    # parameters and optimizer state after the steps
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        scale = max(float(np.abs(exp).max()), 1e-3)
        assert np.max(np.abs(got - exp)) <= 2e-4 * scale, "%s: max abs diff %g (scale %g)" % (name, np.max(np.abs(got - exp)), scale)
        for si, key in enumerate([k for k in ("acc", "n", "z", "m", "v", "ms", "mom") if k in om.slots[name]]):
            g2, e2 = pm.get_tensor(name, slot=si + 1), om.slots[name][key]
            sc = max(float(np.abs(e2).max()), 1e-3)
            assert np.max(np.abs(g2 - e2)) <= 5e-4 * sc, "%s slot %s" % (name, key)
    # and a fresh forward agrees
    raw = random_raw_batch(fc, B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    logits, _ = pm.forward(to_product_batch(plan, raw, label))
    _, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), 5 * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))


@pytest.mark.parametrize("model_type,dense_rows", [("wide_deep", 1000), ("wide_deep", 10 ** 9), ("wide", 500), ("deep", 1000)])
def test_dense_exchange_of_small_tables(model_type, dense_rows):
    """dense_exchange_max_rows: tables / wide columns up to that size live at the end of the row space; their summed gradients
    leave the (row, gradient) lists for a dense block (what data-parallel runs all-reduce) and are applied from it.  Same results
    as the list path, checked against the oracle on one GPU (10**9: every table takes the dense route)."""
    fc, cross, model = small_conf()
    _train_compare(fc, cross, model, model_type, steps=3, seed=29, dense_rows=dense_rows)


def test_prefetched_slots_equal_direct_steps():
    """wd_batch_prefetch_slot (refill on the upload stream, step waits on the device) + wd_train_step_slot + wd_last_loss give
    exactly the losses of plain wd_train_step calls on the same batches, graphs included (8 steps over two alternating slots)."""
    fc, cross, model = small_conf()
    B = 128
    om, plan, pa = build_pair(fc, cross, model, B=B, seed=3)
    pb = WideDeepModel(plan)
    copy_params_to_product(om, pb)
    rng = np.random.default_rng(5)
    batches = []
    for _ in range(8):
        raw = random_raw_batch(fc, B, rng)
        batches.append(to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32)))
    direct = [pa.train_step(b) for b in batches]
    pb.prefetch_slot(2, batches[0])
    got = []
    for i in range(8):
        if i + 1 < 8:
            pb.prefetch_slot(2 + (i + 1) % 2, batches[i + 1])
        if i % 2:
            got.append(pb.train_step_slot(2 + i % 2, want_loss=True))
        else:
            pb.train_step_slot(2 + i % 2, want_loss=False)
            got.append(pb.last_loss())
    assert got == direct, (got, direct)
    for name in pa.tensor_names()[:8]:
        np.testing.assert_array_equal(pa.get_tensor(name), pb.get_tensor(name))


def test_run_to_run_bit_reproducible():
    fc, cross, model = small_conf()
    rng = np.random.default_rng(23)
    B = 128
    raws = [(random_raw_batch(fc, B, rng), (rng.random(B) < 0.3).astype(np.float32)) for _ in range(3)]
    outs = []
    for _ in range(2):
        om, plan, pm = build_pair(fc, cross, model, B=B, seed=29)
        for raw, label in raws:
            pm.train_step(to_product_batch(plan, raw, label))
        outs.append({n: pm.get_tensor(n) for n in pm.tensor_names()})
        pm.close()
    for n in outs[0]:
        assert np.array_equal(outs[0][n], outs[1][n]), n


def test_eval_metrics():
    from oracle.metrics import EvalAccumulator
    fc, cross, model = small_conf()
    rng = np.random.default_rng(31)
    B = 150
    om, plan, pm = build_pair(fc, cross, model, B=B, seed=37)
    acc = EvalAccumulator()
    pm.eval_reset()
    for _ in range(3):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.4).astype(np.float32)
        pm.eval_accumulate(to_product_batch(plan, raw, label))
        _, cache = om.forward(raw)
        acc.update(cache["logits"].astype(np.float32), label)
    got, exp = pm.eval_finish(), acc.result()
    for k in exp:
        assert abs(got[k] - exp[k]) <= 2e-4 * max(abs(exp[k]), 1.0), "%s: %g vs %g" % (k, got[k], exp[k])


# ------------------------------------------------------------------------------------ wgmma engines
def _engine_pair(engine, hidden, mode, B, seed):
    fc, cross, model = small_conf(hidden=hidden, mode=mode)
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(seed)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, max_nnz=B * 64, max_keys=B * 64, gemm_engine=engine)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    return fc, om, plan, pm


@pytest.mark.parametrize("engine", ["tc3x", "bf16x3"])
@pytest.mark.parametrize("mode", ["simple", "dense", "first_dense"])
def test_tc3x_engine_train_parity(mode, engine):
    """wgmma with the 3-pass hi/lo split.  tc3x (tf32, 2^-21 products) must meet the same bars as the fp32 FFMA
    engine.  bf16x3 (bf16 hi/lo copies written by the producing kernels, 2^-16 products) is the fast mode: its
    loss must still agree to 1e-4 and its logits to 5e-4 on these small, badly conditioned towers.  A 1e-5 pre-activation error flips the occasional relu gate (about one of the ~10^5
    activations of a step), which moves a handful of weight-gradient elements by a finite amount, so for bf16x3 the
    trained parameters are compared robustly (a flipped unit moves its whole weight column): 98 % of every tensor within
    2e-3 of its scale, nothing beyond 10 %."""
    B = 300
    ptol = 2e-4 if engine == "tc3x" else 2e-3
    fc, om, plan, pm = _engine_pair(engine, (128, 96, 64), mode, B, seed=41)
    rng = np.random.default_rng(43)
    # forward parity on identical parameters: the quantity the 1e-4 bar is about (bf16x3 on these towers: within 5e-4)
    rng0 = np.random.default_rng(101)                    # (own generator: the training batches below stay what they were)
    raw = random_raw_batch(fc, B, rng0)
    logits, _ = pm.forward(to_product_batch(plan, raw, (rng0.random(B) < 0.3).astype(np.float32)))
    _, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), (1 if engine == "tc3x" else 5) * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
    for step in range(3):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        loss = pm.train_step(to_product_batch(plan, raw, label))
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        scale = max(float(np.abs(exp).max()), 1e-3)
        if engine == "tc3x":
            assert np.max(np.abs(got - exp)) <= ptol * scale, "%s: %g (scale %g)" % (name, np.max(np.abs(got - exp)), scale)
        else:
            bad = np.abs(got - exp) > ptol * scale
            assert bad.mean() <= 2e-2 and np.max(np.abs(got - exp)) <= 0.1 * scale, "%s: %g of the tensor off, max %g (scale %g)" % (
                name, bad.mean(), np.max(np.abs(got - exp)), scale)
    if engine != "tc3x":
        return            # after gate flips the two trained states are different models; their logits are not comparable at 1e-4
    raw = random_raw_batch(fc, B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    logits, _ = pm.forward(to_product_batch(plan, raw, label))
    _, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), 5 * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))


def test_tc1x_engine_is_close_but_not_parity_grade():
    """Single-pass tf32 is offered as a fast mode only: it must be roughly right (1e-2) — and the test documents
    that it does not meet the parity bar, which is why bench.py never uses it."""
    B = 256
    fc, om, plan, pm = _engine_pair("tc1x", (128, 64), "simple", B, seed=47)
    rng = np.random.default_rng(49)
    raw = random_raw_batch(fc, B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    logits, _ = pm.forward(to_product_batch(plan, raw, label))
    _, cache = om.forward(raw)
    err = np.abs(logits - cache["logits"]) / np.maximum(np.abs(cache["logits"]), 1.0)
    assert err.max() < 2e-2


@pytest.mark.parametrize("engine", ["tc3x", "bf16x3"])
def test_hidden_widths_over_128_with_presplit_weights(engine):
    """Hidden widths of 512 and 256: several 128 x 128 output tiles per layer, and the forward and data-gradient GEMMs read the
    weights as pre-split hi / lo copies; B = 700 leaves a ragged last row tile."""
    B = 700
    ptol = 2e-4 if engine == "tc3x" else 2e-3
    fc, om, plan, pm = _engine_pair(engine, (512, 256), "simple", B, seed=53)
    rng = np.random.default_rng(59)
    for step in range(2):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        loss = pm.train_step(to_product_batch(plan, raw, label))
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        scale = max(float(np.abs(exp).max()), 1e-3)
        assert np.max(np.abs(got - exp)) <= ptol * scale, "%s: %g (scale %g)" % (name, np.max(np.abs(got - exp)), scale)


def test_criteo_shape_scaled_down():
    """The benchmark configuration (BASELINE.json configs[1]) with every table scaled by 1e-3: single-valued 32-wide
    embedding bags -> exercises the short-bag gather (emb_pool_fwd_rows_kernel), the pre-split-weight GEMMs and the chunked
    hot-row gradient sums, against the oracle."""
    from wide_deep_b200 import synthetic
    from wide_deep_b200.model import Batch
    fc, cross, model, emb = synthetic.criteo_conf(scale=1e-3, hidden=(256, 128, 64))
    B = 1024
    om = OM.OracleModel(fc, cross, model, "wide_deep", embedding_dim_override=emb).init(61)
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, max_nnz=B * (len(fc) + len(cross)), max_keys=B * n_cat)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    cats = [f for f, c in fc.items() if c["type"] == "category"]
    dense_names = [f for f, c in fc.items() if c["type"] == "continuous"]
    for step in range(3):
        keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=step, zipf=1.2 if step == 1 else None)
        raw = {f: (np.arange(B + 1, dtype=np.int64), np.ascontiguousarray(keys[:, j])) for j, f in enumerate(cats)}
        for j, f in enumerate(dense_names):
            raw[f] = np.ascontiguousarray(dense[:, j])
        loss = pm.train_step(Batch(B, keys.reshape(-1), None, dense, label))
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    # Parameters: Adagrad's g/sqrt(acc) amplifies fp32 summation noise of near-cancelling gradients (batch-sum loss over
    # 1024 examples), so the bound is a fraction of one learning-rate step rather than of the weight scale ...
    lr = 0.05
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        assert np.max(np.abs(got - exp)) <= 0.03 * lr, "%s: %g" % (name, np.max(np.abs(got - exp)))
    # ... while the quantity the parity bar is about, the logits of a fresh batch, still agrees to 1e-4-level
    keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=99)
    raw = {f: (np.arange(B + 1, dtype=np.int64), np.ascontiguousarray(keys[:, j])) for j, f in enumerate(cats)}
    for j, f in enumerate(dense_names):
        raw[f] = np.ascontiguousarray(dense[:, j])
    logits, _ = pm.forward(Batch(B, keys.reshape(-1), None, dense, label))
    _, cache = om.forward(raw)
    np.testing.assert_array_less(np.abs(logits - cache["logits"]), 5 * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))


def test_long_multihot_bags_resdnn():
    """BASELINE.json configs[3] in miniature: one hashed multihot slot (Poisson(30) ids per row, clipped to [1, 96]),
    64-wide embedding, ResDnn 4 x 64 ('resnet' connections).  Exercises the full-warp gather with the warp-shuffle
    segmented mean, duplicate ids inside a bag, and the chunked hot-row gradient sums."""
    from oracle import hashing as OH
    from wide_deep_b200.model import Batch
    fc = OrderedDict()
    fc["tags"] = dict(type="category", transform="hash_bucket", parameter=5000)
    fc["x"] = dict(type="continuous", transform="standard", parameter=dict(normalization=[0.0, 1.0], boundaries=[-1, 0, 1]))
    model = dict(linear_optimizer="Ftrl", linear_initial_learning_rate=0.05, dnn_hidden_units=[64, 64, 64, 64],
                 dnn_connected_mode="resnet", dnn_optimizer="Adagrad", dnn_initial_learning_rate=0.05,
                 dnn_activation_function="relu", dnn_dropout=None, dnn_batch_normalization=1)
    B = 256
    om = OM.OracleModel(fc, [], model, "wide_deep", embedding_dim_override=64).init(71)
    plan = Plan(fc, [], model, "wide_deep", max_batch=B, embedding_dim_override=64, max_nnz=B * 128, max_keys=B * 128)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    rng = np.random.default_rng(73)
    vocab = OH.fingerprint64_tokens(["t%d" % i for i in range(2000)])
    for step in range(3):
        lens = np.clip(rng.poisson(30, size=B), 1, 96)
        offs = np.zeros(B + 1, dtype=np.int64)
        offs[1:] = np.cumsum(lens)
        zipf = (rng.zipf(1.3, size=int(offs[-1])) - 1) % len(vocab)          # skewed: hot rows + duplicates inside bags
        fps = vocab[zipf]
        x = rng.standard_normal(B).astype(np.float32)
        label = (rng.random(B) < 0.3).astype(np.float32)
        raw = {"tags": (offs, fps), "x": x}
        batch = Batch(B, fps, offs.astype(np.int32), x.reshape(B, 1), label)
        if step == 0:
            logits, _ = pm.forward(batch)
            _, cache = om.forward(raw)
            np.testing.assert_array_less(np.abs(logits - cache["logits"]), RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
            X = pm.deep_input(B)
            lo, po, w = plan.deep_layout["tags_embedding"]
            np.testing.assert_allclose(X[:, po:po + w], cache["X"][:, lo:lo + w], rtol=1e-5, atol=1e-6)
        loss = pm.train_step(batch)
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    name = "dnn/input_from_feature_columns/input_layer/tags_embedding/embedding_weights"
    got, exp = pm.get_tensor(name), om.params[name]
    assert np.max(np.abs(got - exp)) <= 0.03 * 0.05


@pytest.mark.parametrize("nnz_cap,digit_bits", [(2048 * 32, None), (2 << 20, None), (2 << 20, 10), (2048 * 32, 10)])
def test_wide_only_hashed_crosses_ftrl(nnz_cap, digit_bits, monkeypatch):
    """BASELINE.json configs[4] in miniature: model_type 'wide', many hashed crosses into large bucket spaces, FTRL.
    The pure sparse-linear path: cross ids bit-exact, FTRL state (w, n, z) after three steps.  An id capacity of 2 M and more
    selects the radix sort's big-list kernels (4096-key tiles reordered in shared memory, sort.cu radix_sort_pairs: what the
    5.4 M-key lists of the wide-only benchmark use); WD_SORT_DIGIT_BITS=10 runs them with the 1024 bins the benchmark's 125 M
    buckets need, which these small tables would not reach."""
    if digit_bits:
        monkeypatch.setenv("WD_SORT_DIGIT_BITS", str(digit_bits))
    fc = OrderedDict()
    for i in range(6):
        fc["k%d" % i] = dict(type="category", transform="hash_bucket", parameter=1000 + 17 * i)
    cross = [(["k%d" % a, "k%d" % b], 200000 + 1000 * (a + b), 0) for a in range(6) for b in range(a + 1, 6)]      # 15 crosses
    model = dict(linear_optimizer="tf.train.FtrlOptimizer(learning_rate=0.1,l1_regularization_strength=0.5,l2_regularization_strength=1)",
                 linear_initial_learning_rate=0.05, dnn_hidden_units=[8], dnn_connected_mode="simple", dnn_optimizer="Adagrad",
                 dnn_initial_learning_rate=0.05, dnn_activation_function="relu", dnn_dropout=None, dnn_batch_normalization=0)
    B = 2048
    rng = np.random.default_rng(81)
    om = OM.OracleModel(fc, cross, model, "wide").init(83)
    plan = Plan(fc, cross, model, "wide", max_batch=B, max_nnz=nnz_cap, max_keys=B * 8)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    for step in range(3):
        raw = random_raw_batch(fc, B, rng, multihot_max=1, na_rate=0.05)
        label = (rng.random(B) < 0.3).astype(np.float32)
        batch = to_product_batch(plan, raw, label)
        if step == 0:
            pm.forward(batch)
            check_ids(om, plan, pm, raw, B)
        loss = pm.train_step(batch)
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    for name in pm.tensor_names():
        for slot, key in ((0, None), (1, "n"), (2, "z")):
            got = pm.get_tensor(name, slot=slot)
            exp = om.params[name] if key is None else om.slots[name][key]
            sc = max(float(np.abs(exp).max()), 1e-3)
            assert np.max(np.abs(got - exp)) <= 5e-4 * sc, "%s slot %d: %g (scale %g)" % (name, slot, np.max(np.abs(got - exp)), sc)


@pytest.mark.parametrize("engine", ["ffma", "tc3x", "bf16x3"])
@pytest.mark.parametrize("mode,bn", [("simple", 1), ("dense", 0)])
def test_dropout_train_parity(engine, mode, bn):
    """dnn_dropout (reference dnn.py:111-112: tf.layers.dropout after every hidden layer's activation, TRAIN only): the keep mask
    is the counter-based one both sides define (oracle.model.drop_keep / csrc/gemm.cuh), so losses and trained parameters must
    agree like without dropout; the mask changes every step (device-side step counter) and evaluation applies no dropout."""
    fc, cross, model = small_conf(hidden=(128, 64), mode=mode, bn=bn)
    model["dnn_dropout"] = 0.25
    B = 256
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(91)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, max_nnz=B * 64, max_keys=B * 64, gemm_engine=engine)
    pm = WideDeepModel(plan)
    copy_params_to_product(om, pm)
    rng = np.random.default_rng(93)
    tol = 1 if engine != "bf16x3" else 5
    for step in range(3):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        batch = to_product_batch(plan, raw, label)
        if step == 1:                                    # evaluation in between: no dropout, and it must not advance the mask counter
            logits, _ = pm.forward(batch)
            _, cache = om.forward(raw)
            np.testing.assert_array_less(np.abs(logits - cache["logits"]), tol * RTOL * np.maximum(np.abs(cache["logits"]), 1.0))
        loss = pm.train_step(batch)
        ref_loss, _ = om.train_step(raw, label)
        assert abs(loss - ref_loss) <= tol * RTOL * max(abs(ref_loss), 1.0), "step %d loss %g vs %g" % (step, loss, ref_loss)
    ptol = 2e-4 if engine != "bf16x3" else 2e-3
    for name in pm.tensor_names():
        got, exp = pm.get_tensor(name), om.params[name]
        scale = max(float(np.abs(exp).max()), 1e-3)
        bad = np.abs(got - exp) > ptol * scale
        assert bad.mean() <= (0.0 if engine != "bf16x3" else 2e-2), "%s: %g of the tensor off, max %g (scale %g)" % (name, bad.mean(), np.max(np.abs(got - exp)), scale)
