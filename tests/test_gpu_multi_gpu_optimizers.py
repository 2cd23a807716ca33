"""Adam and RMSProp on the multi-GPU paths: row-sharded tables (LocalShardGroup and the multi-process driver) and the data-parallel
list exchange with and without the dense block.  Each must compute what one GPU of this library computes on the concatenated
batch.  TensorFlow's sparse Adam moves every row of a table on every step: a row that no rank touched must still move, by the scalar
formula, and by exactly one rank (each replicated tensor stays byte-identical across ranks)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import model as OM
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_CHUNK = 16                        # occurrences per chunk of a hot row's gradient sum (sparse_dev.cuh kChunk)
STEPS = 4
ADAM_FRAC = 2e-3                    # test_gpu_parity's allowance for Adam: elements with a gradient ~0 move by ~lr * sign(g)
FTRL = "tf.train.FtrlOptimizer(learning_rate=0.1,l1_regularization_strength=0.5,l2_regularization_strength=1)"
PAIRS = {                           # (linear_optimizer, dnn_optimizer)
    "adam-adam": ("Adam", "Adam"),
    "ftrl-adam": (FTRL, "Adam"),
    "rmsprop-rmsprop": ("RMSProp", "RMSProp"),
    "adam-rmsprop": ("tf.train.AdamOptimizer(0.002, beta1=0.8)", "RMSProp"),
}
H3 = "dnn/input_from_feature_columns/input_layer/h3_embedding/embedding_weights"


def _conf(pair):
    lin, dnn = PAIRS[pair]
    return small_conf(hidden=(64, 32), dnn_opt=dnn, lin_opt=lin)


def _oracle(fc, cross, model, model_type, seed, rng):
    om = OM.OracleModel(fc, cross, model, model_type).init(seed)
    if om.use_wide:                                   # zero-initialised wide weights carry no signal: give them some
        for c in om.wide_cols:
            om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
    return om


def _set_all(set_tensor, names, om):
    for name in names:
        set_tensor(name, om.params[name], 0)
        for s, v in enumerate(om.slots[name].values()):
            set_tensor(name, v, s + 1)


def _single(fc, cross, model, model_type, B, om):
    plan = Plan(fc, cross, model, model_type, max_batch=B, max_nnz=B * 64, max_keys=B * 64, gemm_engine="ffma")
    pm = WideDeepModel(plan)
    _set_all(lambda n, v, s: pm.set_tensor(n, v, slot=s), pm.tensor_names(), om)
    return pm


def _group(fc, cross, model, model_type, G, per, om, dense_rows=400):
    models = [WideDeepModel(Plan(fc, cross, model, model_type, max_batch=per, max_nnz=per * 64, max_keys=per * 64, gemm_engine="ffma",
                                 dense_exchange_max_rows=dense_rows, shard_world=G, shard_rank=r, shard_slack=float(G)))
              for r in range(G)]
    grp = LocalShardGroup(models)
    _set_all(lambda n, v, s: grp.set_tensor(n, v, slot=s), models[0].tensor_names(), om)
    return grp


def _is_adam(plan, name):
    return (plan.lin_opt if name.startswith("linear/") else plan.dnn_opt)["kind"] == "adam"


def compare_to_single(get, names, n_slots, single, plan):
    """test_gpu_sharded.compare_params' bar (2e-4 of each tensor's scale, 5e-4 for slots) against the single-GPU model; a tensor
    of an Adam optimizer may have up to ADAM_FRAC of its elements outside it."""
    for name in names:
        for s in range(n_slots(name) + 1):
            got, exp = get(name, s), single.get_tensor(name, slot=s)
            scale = max(float(np.abs(exp).max()), 1e-3)
            bad = np.abs(got - exp) > (2e-4 if s == 0 else 5e-4) * scale
            frac = ADAM_FRAC if _is_adam(plan, name) else 0.0
            assert bad.mean() <= frac, "%s slot %d: %d of %d elements off (max %g, scale %g)" % (
                name, s, bad.sum(), bad.size, np.abs(got - exp).max(), scale)


def _table_ids(pm, table):
    """Rows of embedding table `table` in the batch `pm` ran last, with their occurrence counts."""
    plan = pm.plan
    t = [i for i, x in enumerate(plan.tables) if x["name"] == table][0]
    ci = [i for i, c in enumerate(plan.columns) if c.emb_table == t][0]
    C = len(plan.columns)
    offs, ids = pm.column_ids()
    col = np.repeat(np.tile(np.arange(C), (len(offs) - 1) // C), np.diff(offs))
    ids = ids[(col == ci) & (ids >= 0)]
    return np.bincount(ids, minlength=plan.tables[t]["rows"])


def adam_untouched_expect(w, m, v, opt, t):
    """TensorFlow's sparse Adam on a row without gradient at step t (1-based), in fp32 as the library computes it: beta powers
    multiplied up in fp32, lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t), decay, step."""
    f = np.float32
    b1, b2 = f(opt["beta1"]), f(opt["beta2"])
    p1, p2 = b1, b2
    for _ in range(t - 1):
        p1, p2 = f(p1 * b1), f(p2 * b2)
    lr_t = f(f(f(opt["lr"]) * np.sqrt(f(1) - p2)) / f(f(1) - p1))
    m2, v2 = (m * b1).astype(f), (v * b2).astype(f)
    return (w - (lr_t * m2) / (np.sqrt(v2) + f(opt["epsilon"]))).astype(f), m2, v2


def check_untouched_rows(before, after, counts, opt, t):
    """Rows of H3 no rank touched in step t moved exactly as adam_untouched_expect says; there are such rows that had moments."""
    (w0, m0, v0), (w1, m1, v1) = before, after
    idle = counts == 0
    ew, em, ev = adam_untouched_expect(w0[idle], m0[idle], v0[idle], opt, t)
    np.testing.assert_array_equal(m1[idle], em)
    np.testing.assert_array_equal(v1[idle], ev)
    np.testing.assert_allclose(w1[idle], ew, rtol=1e-6, atol=1e-9)
    moved = idle & (np.abs(m0).max(axis=1) > 0)
    assert moved.sum() > 0, "no untouched row with moments"
    assert (w1[moved] != w0[moved]).any(axis=1).all(), "an untouched row with moments did not move"


def _batches(fc, B, rng, n=STEPS):
    """n batches; the last one has no h3 ids (every bag empty), so the h3 rows earlier steps touched sit it out"""
    out = []
    for i in range(n):
        raw = random_raw_batch(fc, B, rng)
        if i == n - 1:
            raw["h3"] = (np.zeros(B + 1, dtype=np.int64), np.zeros(0, dtype=np.uint64))
        out.append((raw, (rng.random(B) < 0.3).astype(np.float32)))
    return out


def _shards(plan, raw, label, G, per):
    return [to_product_batch(plan, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]


def _replicas_identical(models):
    for name in models[0].tensor_names():
        if models[0].plan.is_sharded_tensor(name):
            continue
        for s in range(models[0].n_slots(name) + 1):
            ref = models[0].get_tensor(name, slot=s).tobytes()
            for m in models[1:]:
                assert m.get_tensor(name, slot=s).tobytes() == ref, "%s slot %d differs between ranks" % (name, s)


@pytest.mark.parametrize("pair", sorted(PAIRS))
@pytest.mark.parametrize("model_type", ["wide_deep", "deep", "wide"])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_local_shard_group_matches_single_gpu(G, model_type, pair):
    fc, cross, model = _conf(pair)
    per = 384 // G
    B = per * G
    rng = np.random.default_rng(40 + G)
    om = _oracle(fc, cross, model, model_type, 9 + G, rng)
    grp = _group(fc, cross, model, model_type, G, per, om)
    single = _single(fc, cross, model, model_type, B, om)
    plan0 = grp.models[0].plan
    names = grp.models[0].tensor_names()
    assert any(plan0.is_sharded_tensor(n) for n in names)
    check_h3 = model_type != "wide" and plan0.dnn_opt["kind"] == "adam"
    for step, (raw, label) in enumerate(_batches(fc, B, rng)):
        if check_h3 and step == STEPS - 1:
            before = tuple(grp.get_tensor(H3, slot=s) for s in range(3))
        loss = grp.train_step(_shards(plan0, raw, label, G, per))
        ref = single.train_step(to_product_batch(single.plan, raw, label))
        assert abs(loss - ref) <= 1e-4 * max(abs(ref), 1.0), "step %d: loss %g vs single GPU %g" % (step, loss, ref)
        if model_type != "wide" and step == 0:
            assert _table_ids(single, "h2_embedding").max() > K_CHUNK
    compare_to_single(lambda n, s: grp.get_tensor(n, slot=s), names, grp.models[0].n_slots, single, plan0)
    _replicas_identical(grp.models)
    if check_h3:
        assert plan0.is_sharded_tensor(H3)
        after = tuple(grp.get_tensor(H3, slot=s) for s in range(3))
        check_untouched_rows(before, after, _table_ids(single, "h3_embedding"), plan0.dnn_opt, STEPS)
    single.close()


def _list_pair(fc, cross, model, per, dense_rows, om):
    models = []
    for _ in range(2):
        plan = Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * 64 * 2, max_keys=per * 64, gemm_engine="ffma",
                    dense_exchange_max_rows=dense_rows)
        pm = WideDeepModel(plan)
        _set_all(lambda n, v, s, pm=pm: pm.set_tensor(n, v, slot=s), pm.tensor_names(), om)
        models.append(pm)
    return models


def _list_step(models, shards, K):
    """One data-parallel step of two replicas on one GPU: the fixed-size list exchange and the dense all-reduce done with torch."""
    import torch
    from wide_deep_b200.parallel import wrap_device
    dev = torch.device("cuda", models[0].device)
    loss = 0.0
    for pm, b in zip(models, shards):
        loss += pm.step_backward(b)
    for pm in models:
        pm.sync()
    keep = []
    for w in (0, 1):
        parts_r, parts_g = [], []
        for pm in models:
            rows_ptr, grads_ptr, _, width, cap = pm.sparse_grads(w, want_count=False)
            parts_r.append(wrap_device(rows_ptr, (cap,), torch.int32, dev)[:K])
            parts_g.append(wrap_device(grads_ptr, (cap, width), torch.float32, dev)[:K])
        keep.append((torch.cat(parts_r).contiguous(), torch.cat(parts_g).contiguous()))
    dg = [wrap_device(pm.dense_grad()[0], (pm.dense_grad()[1],), torch.float32, dev) for pm in models]
    total = dg[0] + dg[1]
    for d in dg:
        d.copy_(total)
    torch.cuda.synchronize()
    for pm in models:
        for w, (r, g) in enumerate(keep):
            pm.sparse_set_sorted(w, r.data_ptr(), g.data_ptr(), 2, K)
        pm.step_apply()
    for pm in models:
        pm.sync()
    return loss


@pytest.mark.parametrize("pair", sorted(PAIRS))
@pytest.mark.parametrize("dense_rows", [0, 400])
def test_list_exchange_matches_single_gpu(dense_rows, pair):
    fc, cross, model = _conf(pair)
    per = 192
    rng = np.random.default_rng(7)
    om = _oracle(fc, cross, model, "wide_deep", 21, rng)
    models = _list_pair(fc, cross, model, per, dense_rows, om)
    single = _single(fc, cross, model, "wide_deep", 2 * per, om)
    plan0 = models[0].plan
    for step, (raw, label) in enumerate(_batches(fc, 2 * per, rng)):
        loss = _list_step(models, _shards(plan0, raw, label, 2, per), per * 64)
        ref = single.train_step(to_product_batch(single.plan, raw, label))
        assert abs(loss - ref) <= 1e-4 * max(abs(ref), 1.0), "step %d: loss %g vs single GPU %g" % (step, loss, ref)
    compare_to_single(lambda n, s: models[0].get_tensor(n, slot=s), models[0].tensor_names(), models[0].n_slots, single, plan0)
    _replicas_identical(models)
    for pm in models + [single]:
        pm.close()


def test_resume_is_byte_identical():
    """k steps, every tensor and slot saved with global_step, a fresh group restored from them (set_opt_step on every rank), the
    rest of the steps: byte-identical to the uninterrupted run."""
    fc, cross, model = _conf("adam-adam")
    G, per, k = 2, 128, 2
    rng = np.random.default_rng(3)
    om = _oracle(fc, cross, model, "wide_deep", 5, rng)
    batches = _batches(fc, G * per, rng)
    full = _group(fc, cross, model, "wide_deep", G, per, om)
    plan0 = full.models[0].plan
    for raw, label in batches:
        full.train_step(_shards(plan0, raw, label, G, per))
    first = _group(fc, cross, model, "wide_deep", G, per, om)
    for raw, label in batches[:k]:
        first.train_step(_shards(plan0, raw, label, G, per))
    names = first.models[0].tensor_names()
    saved = {(n, s): first.get_tensor(n, slot=s) for n in names for s in range(first.models[0].n_slots(n) + 1)}
    step = first.models[0].global_step
    assert step == k
    del first
    resumed = _group(fc, cross, model, "wide_deep", G, per, om)
    for m in resumed.models:
        m.global_step = step
        m.set_opt_step(step)
    for (n, s), v in saved.items():
        resumed.set_tensor(n, v, slot=s)
    for raw, label in batches[k:]:
        resumed.train_step(_shards(plan0, raw, label, G, per))
    for (n, s) in saved:
        assert resumed.get_tensor(n, slot=s).tobytes() == full.get_tensor(n, slot=s).tobytes(), (n, s)


def test_multi_process_shard_driver_with_adam():
    """wd_shard_train_step_slot under flag barriers and graph replay, two processes sharing cuda:0 (and one process per GPU
    when there are two): Adam / Adam and RMSProp / RMSProp against a single-GPU model, untouched rows by the formula."""
    import torch
    runs = [(2, True)] + ([(2, False)] if torch.cuda.device_count() >= 2 else [])
    for world, same_gpu in runs:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
               "--master-port", "29657", os.path.join(ROOT, "tests", "_shard_adam_worker.py")]
        env = dict(os.environ)
        if same_gpu:
            env["WD_SHARD_SAME_GPU"] = "1"
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
        assert r.returncode == 0 and "SHARD_ADAM_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_adam_with_host_placed_shard_is_refused():
    """Adam's untouched pass would stream a whole host-placed shard over PCIe every step: refused when the model is created;
    RMSProp (row-local) may keep its shard on the host."""
    from wide_deep_b200 import _native
    for pair, refused in (("adam-adam", True), ("rmsprop-rmsprop", False)):
        fc, cross, model = _conf(pair)
        plan = Plan(fc, cross, model, "wide_deep", max_batch=64, max_nnz=64 * 64, max_keys=64 * 64, gemm_engine="ffma",
                    dense_exchange_max_rows=400, shard_world=2, shard_rank=0, shard_slack=2.0, host_tables=["h3_embedding"])
        assert plan.is_sharded_tensor(H3)
        if refused:
            with pytest.raises(_native.NativeError) as e:
                WideDeepModel(plan)
            assert e.value.code == _native.EUNSUPPORTED
        else:
            pm = WideDeepModel(plan)
            assert pm.memory_usage()[1] > 0
            pm.close()
