"""Adam on host-placed embedding tables by deferral (Plan(defer_adam=True), WD_PLACE_DEFER_ADAM).

Sparse Adam moves every row of a table every step.  A deferred host table skips that untouched pass and replays the steps a row
missed when the row is next staged (or when the whole table is read), with the same fp32 operations in the same order, so the
model must compute exactly what the same model computes with every table in HBM: that model is the oracle and every comparison is
byte for byte.  Long gaps are checked against the float32 emulation in tests/adam_replay_ref.py.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.adam_replay_ref import lr_t_table, replay
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200 import _native
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import T_EMB_TABLE, Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAM = "Adam"
ADAM_FAST = "tf.train.AdamOptimizer(learning_rate=0.05,beta1=0.5,beta2=0.9)"     # lr_t reaches lr after ~165 steps
ADAM_HALF = "tf.train.AdamOptimizer(learning_rate=0.05,beta1=0.5,beta2=0.5)"
# h2_embedding (37 rows) has hot rows (the chunked combine runs before the staged apply); h3_embedding (200000 x 16) is the large
# one; h1_X_h2_embedding (1000 rows) sees most of its rows come back after gaps (the random batches draw h1 / h3 from 50 tokens)
SUBSET = ["h2_embedding", "h3_embedding", "h1_X_h2_embedding"]
SMALL = ["h2_embedding", "h1_embedding", "id1_X_v2_X_x1_bucketized_embedding"]   # small enough for the numpy emulation


def _plan(dnn_opt, B, gather, host_tables, defer=True, **kw):
    fc, cross, model = small_conf(dnn_opt=dnn_opt)
    keys = B * (18 if gather == "rows" else 64)
    return Plan(fc, cross, model, "wide_deep", max_batch=B, max_nnz=B * 320, max_keys=keys, gemm_engine="ffma",
                host_tables=host_tables, defer_adam=defer, **kw)


def _batches(plan, B, n, seed, gather="rows"):
    fc = small_conf()[0]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        raw = random_raw_batch(fc, B, rng, multihot_max=3 if gather == "rows" else 10)
        out.append(to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32)))
    return out


def _all_tensors(pm):
    out = {}
    for name in pm.tensor_names():
        for s in range(pm.n_slots(name) + 1):
            out["%s/slot%d" % (name, s)] = pm.get_tensor(name, slot=s)
    return out


def _assert_bytes_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def _train(pm, batches, steps=None):
    """Two alternating prefetched slots: per slot two eager steps, then the captured step graph, then its replays."""
    steps = steps or len(batches)
    losses = []
    pm.prefetch_slot(0, batches[0])
    for i in range(steps):
        if i + 1 < steps:
            pm.prefetch_slot((i + 1) % 2, batches[(i + 1) % len(batches)])
        losses.append(pm.train_step_slot(i % 2, want_loss=True))
    return np.float32(losses)


def _compare_after_training(host, ref, test):
    for b in test:
        lh, ll = host.forward(b)
        rh, rl = ref.forward(b)
        assert lh.tobytes() == rh.tobytes() and ll == rl
    for pm in (host, ref):
        pm.eval_reset()
        for b in test:
            pm.eval_accumulate(b)
    # (the logits are byte-equal above; the metric sums are double atomics, whose order may move the last bit)
    eh, er = host.eval_finish(), ref.eval_finish()
    assert eh.keys() == er.keys() and all(abs(eh[k] - er[k]) <= 1e-12 * max(1.0, abs(er[k])) for k in er), (eh, er)
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))


@pytest.mark.parametrize("cache", [0, 1 << 16])
@pytest.mark.parametrize("placement", ["all", "subset"])
@pytest.mark.parametrize("gather", ["rows", "warp"])
def test_deferred_host_tables_train_bit_identical(gather, placement, cache):
    B = 128
    ref_plan = _plan(ADAM, B, gather, [], defer=False)
    host_plan = _plan(ADAM, B, gather, "all" if placement == "all" else SUBSET, host_cache_bytes=cache)
    ref, host = WideDeepModel(ref_plan).init(11), WideDeepModel(host_plan).init(11)
    assert ref.memory_usage()[1] == 0 and host.memory_usage()[1] > 0
    batches = _batches(ref_plan, B, 8, 5, gather)
    lh, lr = _train(host, batches), _train(ref, batches)
    assert np.isfinite(lr).all() and lh.tobytes() == lr.tobytes(), (lh, lr)
    st = host.deferred_adam_stats()
    assert st["rows"] > 0 and st["replayed"] > 0 and st["max_gap"] >= 1, st
    assert ref.deferred_adam_stats() == dict(rows=0, replayed=0, skipped=0, max_gap=0)
    if cache:
        assert host.host_cache_stats()["evictions"] > 0          # records with their stamps went home from the cache
    _compare_after_training(host, ref, _batches(ref_plan, B, 2, 6, gather))


def test_long_run_crosses_the_end_of_the_lr_t_table():
    """400 steps at betas (0.5, 0.9): lr_t reaches lr after ~165 steps, rows come back after gaps on both sides of that step."""
    B = 128
    ref_plan = _plan(ADAM_FAST, B, "rows", [], defer=False)
    ref, host = WideDeepModel(ref_plan).init(3), WideDeepModel(_plan(ADAM_FAST, B, "rows", SUBSET)).init(3)
    batches = _batches(ref_plan, B, 24, 9)
    lh, lr = _train(host, batches, 400), _train(ref, batches, 400)
    assert np.isfinite(lr).all() and lh.tobytes() == lr.tobytes()
    _compare_after_training(host, ref, _batches(ref_plan, B, 2, 10))
    assert host.deferred_adam_stats()["skipped"] > 0                # rows idle past the table's end stopped early


def _deferred_state(pm, names):
    return {n: tuple(pm.get_tensor(n, slot=s) for s in range(3)) for n in names}


@pytest.mark.parametrize("opt,gaps", [(ADAM, "ladder"), (ADAM_HALF, "huge")])
def test_long_gaps_match_the_emulation(opt, gaps):
    """Read every tensor at step g (settling the deferred rows), move the step count to g + k, read again: each deferred row
    replays exactly steps g+1 .. g+k (until its values stop changing past the lr_t table's end)."""
    B = 128
    plan = _plan(opt, B, "rows", SMALL)
    pm = WideDeepModel(plan).init(21)
    _train(pm, _batches(plan, B, 5, 22))
    g = 5
    o = plan.dnn_opt
    lr, b1, b2, eps = o["lr"], o["beta1"], o["beta2"], o["epsilon"]
    table = lr_t_table(lr, b1, b2)
    last = table[1]
    rows = sum(t["rows"] for t in plan.tables if t["name"] in SMALL)
    def deferred(n):
        kind, index = plan.tensor_names[n][:2]
        return kind == T_EMB_TABLE and plan.tables[index]["name"] in SMALL
    names = [n for n in pm.tensor_names() if deferred(n)]
    others = [n for n in pm.tensor_names() if not deferred(n)]
    assert len(names) == len(SMALL)
    before = _deferred_state(pm, names)
    rest = {n: pm.get_tensor(n) for n in others}
    ks = [1, 17, 5000, last, last + 1] if gaps == "ladder" else [10 ** 6]
    for k in ks:
        pm.deferred_adam_stats(reset=True)
        pm.set_opt_step(g + k)
        after = _deferred_state(pm, names)
        st = pm.deferred_adam_stats()
        for n in names:
            w, m, v, _ = replay(*before[n], g, g + k, lr, b1, b2, eps, table=table)
            assert after[n][0].tobytes() == w.tobytes(), (n, k)
            assert after[n][1].tobytes() == m.tobytes(), (n, k)
            assert after[n][2].tobytes() == v.tobytes(), (n, k)
        assert st["rows"] == rows and st["max_gap"] == k, (k, st)
        assert st["replayed"] + st["skipped"] == rows * k, (k, st)
        if g + k <= last:
            assert st["replayed"] == rows * k and st["skipped"] == 0, (k, st)
        if k == 10 ** 6:
            assert st["skipped"] > 0 and st["replayed"] < rows * 2000, st
        for n in others:
            assert pm.get_tensor(n).tobytes() == rest[n].tobytes(), n
        # a second read finds every row current
        pm.deferred_adam_stats(reset=True)
        _deferred_state(pm, names)
        assert pm.deferred_adam_stats()["rows"] == 0
        before, g = after, g + k
    # training continues from the settled rows
    assert np.isfinite(_train(pm, _batches(plan, B, 3, 23))).all()


def _restore(dst, src_tensors, steps):
    dst.set_opt_step(steps)
    for key, val in src_tensors.items():
        name, s = key.rsplit("/slot", 1)
        dst.set_tensor(name, val, slot=int(s))


def test_checkpoints_move_between_deferred_host_and_hbm_placement():
    """set_opt_step + set_tensor (a checkpoint restore) leaves every row current: deferred -> HBM -> deferred."""
    B = 128
    ref_plan = _plan(ADAM, B, "rows", [], defer=False)
    batches = _batches(ref_plan, B, 12, 31)
    a = WideDeepModel(_plan(ADAM, B, "rows", "all")).init(4)
    _train(a, batches[:4])
    hbm = WideDeepModel(ref_plan)
    _restore(hbm, _all_tensors(a), 4)
    _train(a, batches[4:8])
    _train(hbm, batches[4:8])
    _assert_bytes_equal(_all_tensors(a), _all_tensors(hbm))
    b = WideDeepModel(_plan(ADAM, B, "rows", "all", host_cache_bytes=1 << 16))
    _restore(b, _all_tensors(hbm), 8)
    _train(b, batches[8:])
    _train(hbm, batches[8:])
    _assert_bytes_equal(_all_tensors(b), _all_tensors(hbm))


def test_refusals_and_other_optimizers():
    B = 64
    pm = WideDeepModel(_plan(ADAM, B, "rows", SUBSET))
    pm.init(1)
    b = _batches(pm.plan, B, 1, 2)[0]
    with pytest.raises(_native.NativeError) as e:
        pm.step_backward(b)
    assert e.value.code == _native.EUNSUPPORTED
    with pytest.raises(_native.NativeError) as e:                     # without the flag Adam stays refused on the host
        WideDeepModel(_plan(ADAM, B, "rows", SUBSET, defer=False))
    assert e.value.code == _native.EUNSUPPORTED
    auto = WideDeepModel(_plan(ADAM, B, "rows", None))                 # auto + defer: fits in HBM, stays there
    assert auto.memory_usage()[1] == 0
    # the flag with another optimizer is plain host placement: same records, same results
    plain, flagged = (WideDeepModel(_plan("Adagrad", B, "rows", SUBSET, defer=d)).init(5) for d in (False, True))
    assert plain.memory_usage() == flagged.memory_usage()
    batches = _batches(plain.plan, B, 4, 6)
    assert _train(plain, batches).tobytes() == _train(flagged, batches).tobytes()
    _assert_bytes_equal(_all_tensors(plain), _all_tensors(flagged))
    assert flagged.deferred_adam_stats()["rows"] == 0


# ---------------------------------------------------------------------------------------------------------- row-sharded
DENSE_ROWS = 30


def _sharded_plans(G, per, host_tables, defer, **kw):
    fc, cross, model = small_conf(dnn_opt=ADAM)
    return [Plan(fc, cross, model, "wide_deep", max_batch=per, gemm_engine="ffma", max_nnz=per * 64, max_keys=per * 64,
                 dense_exchange_max_rows=DENSE_ROWS, shard_world=G, shard_rank=r, shard_slack=float(G), host_tables=host_tables,
                 defer_adam=defer, **kw) for r in range(G)]


def _sharded_all(grp):
    out = {}
    m0 = grp.models[0]
    for name in m0.tensor_names():
        for s in range(m0.n_slots(name) + 1):
            out["%s/slot%d" % (name, s)] = grp.get_tensor(name, slot=s)
    return out


@pytest.mark.parametrize("cache", [0, 1 << 15])
@pytest.mark.parametrize("G", [2, 3])
def test_sharded_deferred_host_tables_bit_identical(G, cache):
    per = 384 // G
    B = per * G
    ref_plans = _sharded_plans(G, per, [], False)
    host = [t["name"] for t in ref_plans[0].tables if t["sharded"]]
    kw = dict(shard_cache_bytes=cache) if cache else {}
    ref = LocalShardGroup([WideDeepModel(p).init(7) for p in ref_plans])
    hst = LocalShardGroup([WideDeepModel(p).init(7) for p in _sharded_plans(G, per, host, True, **kw)])
    assert all(m.memory_usage()[1] > 0 for m in hst.models)
    fc = small_conf()[0]
    rng = np.random.default_rng(41 + G)
    plan0 = ref_plans[0]

    def shards():
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        return [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]

    lr, lh = [], []
    for _ in range(6):
        s = shards()
        lr.append(ref.train_step(s))
        lh.append(hst.train_step(s))
    lr, lh = np.float32(lr), np.float32(lh)
    assert np.isfinite(lr).all() and lh.tobytes() == lr.tobytes(), (lh, lr)
    s = shards()
    assert np.concatenate(hst.forward(s)).tobytes() == np.concatenate(ref.forward(s)).tobytes()
    _assert_bytes_equal(_sharded_all(hst), _sharded_all(ref))
    assert sum(st["rows"] for st in hst.deferred_adam_stats()) > 0
    if cache:
        assert sum(c["loads"] for c in hst.host_cache_stats()) > 0


def test_sharded_deferred_host_tables_in_separate_processes():
    """The multi-process driver (CUDA IPC, flag barriers, step graph replay), two ranks on one GPU."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29667", os.path.join(ROOT, "tests", "_shard_defer_adam_worker.py")]
    env = dict(os.environ)
    env["WD_SHARD_SAME_GPU"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0 and "SHARD_DEFER_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
