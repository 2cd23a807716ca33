"""The owner's HBM cache of its host-placed shard records (Plan(shard_cache_bytes=...), wd_shard_cache_enable).

Each rank of a row-sharded model with host-placed shards may keep the most recently used records of the rows it owns in its own
HBM.  A cached record is an exact copy of its host record and every kernel after the stage-in sees the same values in the same
order, so the cached model must compute exactly what the same G-rank model computes with every shard in HBM, and what it computes
with the shards on the host and no cache: both are oracles here and every comparison is byte for byte.  Each rank's counters are
predicted exactly by the single-GPU policy restatement (tests/test_gpu_host_cache.CachePolicy) fed with the rows that rank owns.
The G ranks are G handles in one process (`LocalShardGroup`); tests/_shard_cache_worker.py runs the multi-process driver.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import hashing as OH
from oracle import model as OM
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_host_cache import WAYS, CachePolicy
from tests.test_gpu_parity import small_conf
from tests.test_gpu_sharded_host_tables import K_CHUNK, SUBSET, _all_tensors, _assert_bytes_equal, _max_occurrences, _sharded_tables
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200 import _native
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (plain SGD diverges on the sum-reduced loss at the conf's 0.05, quirk Q11; test_gpu_host_tables uses the same 2e-5)
OPTS = {"Adagrad": "Adagrad", "Ftrl": "Ftrl", "RMSProp": "RMSProp", "SGD": "tf.train.GradientDescentOptimizer(learning_rate=0.00002)"}
DENSE_ROWS = 30                    # tables of more rows are row-sharded (as in test_gpu_sharded_host_tables)
MAX_IDS = 64
STEPS = 4


def _plans(fc, cross, model, G, per, host_tables, **kw):
    return [Plan(fc, cross, model, "wide_deep", max_batch=per, gemm_engine="ffma", max_nnz=per * MAX_IDS, max_keys=per * MAX_IDS,
                 dense_exchange_max_rows=DENSE_ROWS, shard_world=G, shard_rank=r, shard_slack=float(G), host_tables=host_tables, **kw)
            for r in range(G)]


def _oracle(fc, cross, model, seed, rng):
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(seed)
    for c in om.wide_cols:                            # zero-initialised wide weights carry no signal: give them some
        om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
    return om


def _group(plans, om):
    grp = LocalShardGroup([WideDeepModel(p) for p in plans])
    for name in grp.models[0].tensor_names():
        grp.set_tensor(name, om.params[name])
        for s, v in enumerate(om.slots[name].values()):
            grp.set_tensor(name, v, slot=s + 1)
    return grp


def _stride(plan, host):
    """Floats per staged shard record: the widest host record [w | slots]."""
    nslots = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan.dnn_opt["kind"]]
    return max(((t["dim"] + 3) // 4 * 4) * (1 + nslots) for t in plan.tables if t["name"] in host)


def _bytes_for(plan, host, set_bits):
    return WAYS * (1 << set_bits) * _stride(plan, host) * 4


def _owned_rows(grp, host):
    """Per rank: sorted unique rows it owns of the host tables in the call just run, in its shard row space (slot bases of
    ceil(rows / G) rows in table order, global row r at local row r // G of rank r mod G), from every rank's column ids."""
    plan, G = grp.models[0].plan, grp.G
    base, acc = {}, 0
    for t, tb in enumerate(plan.tables):
        if tb["sharded"]:
            base[t] = acc
            acc += (tb["rows"] + G - 1) // G
    C = len(plan.columns)
    per_table = {}
    for m in grp.models:
        offs, ids = m.column_ids()
        col = np.repeat(np.tile(np.arange(C), (len(offs) - 1) // C), np.diff(offs))
        for ci, c in enumerate(plan.columns):
            t = c.emb_table
            if t < 0 or plan.tables[t]["name"] not in host:
                continue
            v = ids[col == ci]
            per_table.setdefault(t, []).append(v[(v >= 0) & (v < plan.tables[t]["rows"])])
    uniq = {t: np.unique(np.concatenate(vs)) for t, vs in per_table.items()}
    out = []
    for r in range(G):
        rows = [base[t] + v[v % G == r] // G for t, v in uniq.items()]
        out.append(np.unique(np.concatenate(rows)) if rows else np.zeros(0, np.int64))
    return out


def _simulate(calls, G, bits):
    pols = [CachePolicy(bits) for _ in range(G)]
    for rows, train in calls:
        for r in range(G):
            pols[r].call(rows[r], train)
    return [p.c for p in pols]


def _pick_bits(calls, G, want):
    """Smallest set count whose simulated run shows `want` on the ranks: no overflow and some rank evicting (medium), or no
    overflow and nothing evicted on any rank (large)."""
    for bits in range(1, 18):
        cs = _simulate(calls, G, bits)
        if all(c["overflow"] == 0 for c in cs) and any(c["evictions"] > 0 for c in cs) == (want == "medium"):
            return bits
    raise AssertionError("no cache size gives a %s cache for these calls" % want)


def _batches(fc, plan0, G, per, n, rng):
    """Multihot bags (h2's 37 rows take more than a 16-occurrence chunk per row); h1 and h3 draw from 2^20 tokens, so the large
    tables see new rows every step and a cache that holds one step's rows still has to evict over the run."""
    out = []
    for _ in range(n):
        raw = random_raw_batch(fc, G * per, rng, multihot_max=3)
        for f in ("h1", "h3"):
            offs, fp = raw[f]
            raw[f] = (offs, OH.fingerprint64_tokens(["w%d" % rng.integers(0, 1 << 20) for _ in range(len(fp))]))
        label = (rng.random(G * per) < 0.3).astype(np.float32)
        out.append([to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)])
    return out


@pytest.mark.parametrize("placement", ["all", "subset"])
@pytest.mark.parametrize("opt", sorted(OPTS))
@pytest.mark.parametrize("G", [2, 3, 4])
def test_cached_sharded_training_is_bit_identical(G, opt, placement):
    """4 train steps of 512 examples and a forward on three cache sizes (one set: overflow rows; medium: evictions without
    overflow; large: nothing evicted): losses, logits, every parameter and optimizer slot byte-equal to the HBM-sharded and the
    uncached host-sharded model, and every rank's counters equal to the policy's after every call."""
    fc, cross, model = small_conf(dnn_opt=OPTS[opt])
    per = 512 // G
    rng = np.random.default_rng(31 + G)
    om = _oracle(fc, cross, model, 7 + G, rng)
    ref_plans = _plans(fc, cross, model, G, per, [])
    host = _sharded_tables(ref_plans[0]) if placement == "all" else SUBSET
    if placement == "subset":
        assert set(_sharded_tables(ref_plans[0])) - set(host)
    batches = _batches(fc, ref_plans[0], G, per, STEPS + 1, rng)
    ref = _group(ref_plans, om)
    unc = _group(_plans(fc, cross, model, G, per, host), om)
    lr, lu, calls = [], [], []
    for i, shards in enumerate(batches[:STEPS]):
        lr.append(ref.train_step(shards))
        lu.append(unc.train_step(shards))
        calls.append((_owned_rows(ref, host), True))
        if i == 0:                                    # the chunked combine of hot rows runs before a staged apply
            assert _max_occurrences(ref, "h2_embedding") > K_CHUNK
    logits_ref = np.concatenate(ref.forward(batches[STEPS]))
    calls.append((_owned_rows(ref, host), False))
    assert np.concatenate(unc.forward(batches[STEPS])).tobytes() == logits_ref.tobytes()
    lr, lu = np.float32(lr), np.float32(lu)
    assert np.isfinite(lr).all() and lu.tobytes() == lr.tobytes()
    want = _all_tensors(ref)
    _assert_bytes_equal(_all_tensors(unc), want)
    for g in (ref, unc):
        for m in g.models:
            m.close()
    sizes = {"one set": 0, "medium": _pick_bits(calls, G, "medium"), "large": _pick_bits(calls, G, "large")}
    for size, bits in sizes.items():
        cached = _group(_plans(fc, cross, model, G, per, host, shard_cache_bytes=_bytes_for(ref_plans[0], host, bits)), om)
        assert [c["capacity"] for c in cached.host_cache_stats()] == [WAYS << bits] * G
        pols = [CachePolicy(bits) for _ in range(G)]
        lc = []
        for (rows, train), shards in zip(calls, batches):
            if train:
                lc.append(cached.train_step(shards))
            else:
                assert np.concatenate(cached.forward(shards)).tobytes() == logits_ref.tobytes(), size
            for r in range(G):
                pols[r].call(rows[r], train)
            got = cached.host_cache_stats()
            assert got == [dict(capacity=WAYS << bits, **p.c) for p in pols], (size, got, [p.c for p in pols])
        assert np.float32(lc).tobytes() == lr.tobytes(), (size, lc, lr)
        got = cached.host_cache_stats()
        if size == "one set":
            assert all(c["overflow"] > 0 for c in got), got
        elif size == "medium":
            assert all(c["overflow"] == 0 for c in got) and any(c["evictions"] > 0 for c in got), got
        else:
            assert all(c["overflow"] == 0 and c["evictions"] == 0 and c["hits"] > 0 for c in got), got
        _assert_bytes_equal(_all_tensors(cached), want)          # (reads flush the dirty slots)
        for m in cached.models:
            m.close()


def test_eval_and_forward_of_a_fresh_cached_model_leave_nothing_dirty():
    """Forward-only calls and LocalShardGroup.evaluate load slots but mark none dirty: nothing is evicted, the host records do not
    change, and the metrics equal the uncached model's."""
    G, per = 2, 96
    fc, cross, model = small_conf()
    rng = np.random.default_rng(17)
    om = _oracle(fc, cross, model, 13, rng)
    ref_plans = _plans(fc, cross, model, G, per, [])
    host = _sharded_tables(ref_plans[0])
    unc = _group(_plans(fc, cross, model, G, per, host), om)
    cached = _group(_plans(fc, cross, model, G, per, host, shard_cache_bytes=_bytes_for(ref_plans[0], host, 1)), om)
    before = _all_tensors(cached)
    batches = _batches(fc, ref_plans[0], G, per, 4, rng)
    for shards in batches[:2]:
        assert np.concatenate(cached.forward(shards)).tobytes() == np.concatenate(unc.forward(shards)).tobytes()
    nv = [[b.batch_size - 5 * r for b in [s[r] for s in batches]] for r in range(G)]
    per_rank = [[s[r] for s in batches] for r in range(G)]
    assert cached.evaluate(per_rank, nv) == unc.evaluate(per_rank, nv)
    got = cached.host_cache_stats()
    assert all(c["loads"] > 0 and c["overflow"] > 0 and c["evictions"] == 0 for c in got), got    # 2 sets: slots reused, none dirty
    _assert_bytes_equal(_all_tensors(cached), before)


def test_tensor_io_reinit_and_set_tensor_see_the_cache():
    """Reads after training flush dirty slots; set_tensor and re-init rewrite the host records and empty the cache; training
    afterwards equals the HBM model doing the same."""
    G, per = 3, 128
    fc, cross, model = small_conf(dnn_opt=OPTS["Ftrl"])
    rng = np.random.default_rng(2)
    om = _oracle(fc, cross, model, 2, rng)
    ref_plans = _plans(fc, cross, model, G, per, [])
    ref = _group(ref_plans, om)
    cached = _group(_plans(fc, cross, model, G, per, SUBSET, shard_cache_bytes=_bytes_for(ref_plans[0], SUBSET, 3)), om)
    batches = _batches(fc, ref_plans[0], G, per, 9, rng)

    def train(steps):
        for shards in batches[steps]:
            assert np.float32(cached.train_step(shards)).tobytes() == np.float32(ref.train_step(shards)).tobytes()

    train(slice(0, 3))
    _assert_bytes_equal(_all_tensors(cached), _all_tensors(ref))
    for name in ("h2_embedding", "h3_embedding"):
        full = [n for n in ref.models[0].tensor_names() if n.endswith("/" + name + "/embedding_weights")]
        assert len(full) == 1, name
        w = rng.standard_normal(ref.get_tensor(full[0]).shape).astype(np.float32)
        n = np.abs(rng.standard_normal(w.shape)).astype(np.float32) + 0.1
        for g in (cached, ref):
            g.set_tensor(full[0], w)
            g.set_tensor(full[0], n, slot=1)
    train(slice(3, 6))
    _assert_bytes_equal(_all_tensors(cached), _all_tensors(ref))
    for g in (cached, ref):
        for m in g.models:
            m.init(7)                                 # re-init empties the cache
    train(slice(6, 9))
    _assert_bytes_equal(_all_tensors(cached), _all_tensors(ref))
    assert all(c["hits"] > 0 for c in cached.host_cache_stats())


def test_refusals():
    G, per = 2, 64
    fc, cross, model = small_conf()
    rng = np.random.default_rng(3)
    om = _oracle(fc, cross, model, 3, rng)
    plans = _plans(fc, cross, model, G, per, SUBSET)
    budget = _bytes_for(plans[0], SUBSET, 2)
    # after a step or forward
    grp = _group(plans, om)
    grp.train_step(_batches(fc, plans[0], G, per, 1, rng)[0])
    assert grp.models[0]._lib.wd_shard_cache_enable(grp.models[0]._h, budget) == _native.ESTATE
    for m in grp.models:
        m.close()
    # twice, and a negative budget
    pm = WideDeepModel(_plans(fc, cross, model, G, per, SUBSET, shard_cache_bytes=budget)[0])
    assert pm._lib.wd_shard_cache_enable(pm._h, budget) == _native.ESTATE
    pm.close()
    pm = WideDeepModel(plans[0])
    assert pm._lib.wd_shard_cache_enable(pm._h, -1) == _native.EINVAL
    # the single-GPU cache stays refused on host shards, and its message names the owner's cache
    with pytest.raises(_native.NativeError) as e:
        WideDeepModel(_plans(fc, cross, model, G, per, SUBSET, host_cache_bytes=budget)[0])
    assert e.value.code == _native.EUNSUPPORTED and "wd_shard_cache_enable" in str(e.value)
    # one GPU: the owner's cache does not apply
    single = Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * MAX_IDS, max_keys=per * MAX_IDS, gemm_engine="ffma",
                  host_tables="all")
    ps = WideDeepModel(single)
    assert ps._lib.wd_shard_cache_enable(ps._h, budget) == _native.EUNSUPPORTED
    ps.close()
    # no host shard on the rank, or a budget below one set: capacity 0, nothing allocated
    hbm = WideDeepModel(_plans(fc, cross, model, G, per, [])[0])
    hbm2 = WideDeepModel(_plans(fc, cross, model, G, per, [], shard_cache_bytes=1 << 24)[0])
    assert hbm2.memory_usage() == hbm.memory_usage() and hbm2.host_cache_stats()["capacity"] == 0
    small = WideDeepModel(_plans(fc, cross, model, G, per, SUBSET, shard_cache_bytes=_bytes_for(plans[0], SUBSET, 0) - 1)[0])
    assert small.memory_usage() == pm.memory_usage() and small.host_cache_stats() == dict.fromkeys(
        ("capacity", "hits", "loads", "overflow", "evictions"), 0)
    for m in (pm, hbm, hbm2, small):
        m.close()


def test_cache_memory_accounting():
    """HBM grows by the slots and their metadata (as test_gpu_host_cache.test_cache_memory_accounting counts them for one GPU,
    with max_nnz + 1 per-row entries: the owner staging buffer's spare row); budgets beyond HBM or 31-bit staging rows are
    refused."""
    G, per = 3, 64
    fc, cross, model = small_conf()
    plans = _plans(fc, cross, model, G, per, SUBSET)
    bits = 3
    S, C, nnz = _stride(plans[0], SUBSET), WAYS << bits, per * MAX_IDS * G       # max_nnz x shard_slack
    meta = C * (4 + 4 + 1) + 4 + 4 * 8 + (nnz + 1) * (4 + 4 + 1) + 4 * (nnz + 8) * 4
    for r in range(G):
        base = WideDeepModel(plans[r])
        cached = WideDeepModel(_plans(fc, cross, model, G, per, SUBSET, shard_cache_bytes=_bytes_for(plans[0], SUBSET, bits))[r])
        assert cached.memory_usage()[0] - base.memory_usage()[0] == C * S * 4 + meta, r
        assert cached.memory_usage()[1] == base.memory_usage()[1]
        base.close()
        cached.close()
    big = next(k for k in range(40) if _bytes_for(plans[0], SUBSET, k) > 96e9)
    assert (WAYS << big) + nnz + 1 < 2 ** 31
    for k, code in ((big, _native.ENOMEM), (28, _native.EINVAL)):
        with pytest.raises(_native.NativeError) as e:
            WideDeepModel(_plans(fc, cross, model, G, per, SUBSET, shard_cache_bytes=_bytes_for(plans[0], SUBSET, k))[0])
        assert e.value.code == code, k


@pytest.mark.parametrize("same_gpu", [True, False])
def test_shard_cache_in_separate_processes(same_gpu):
    """The multi-process driver (CUDA IPC, flag barriers, step graph replay, graphed eval accumulate): every rank trains an
    uncached and a cached host-sharded model on the same batches and compares them byte for byte; then a checkpoint saved by the
    estimator from a cached sharded model restores bit-identically into an HBM-sharded one."""
    import torch
    n = torch.cuda.device_count()
    if not same_gpu and n < 2:
        pytest.skip("needs 2 GPUs")
    world = 2 if same_gpu else min(n, 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", "29681" if same_gpu else "29682", os.path.join(ROOT, "tests", "_shard_cache_worker.py")]
    env = dict(os.environ)
    if same_gpu:
        env["WD_SHARD_SAME_GPU"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0 and "SHARD_CACHE_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
