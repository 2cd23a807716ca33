"""Row-sharded embedding tables whose shards live in page-locked host memory (Plan(host_tables=[...]) with shard_world > 1).

Each owner groups the rows it received, stages the records of its host rows into HBM, serves and updates them there and writes
them back, so a host-placed sharded model must compute exactly what the same G-rank model computes with every shard in HBM: that
model is the oracle here and every comparison is byte for byte.  The G ranks are G handles in one process (`LocalShardGroup`);
tests/_shard_host_worker.py runs the multi-process driver (CUDA IPC, flag barriers, graph replay).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import model as OM
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200 import _native
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (plain SGD diverges on the sum-reduced loss at the conf's 0.05, quirk Q11; test_gpu_host_tables uses the same 2e-5)
OPTS = {"Adagrad": "Adagrad", "Ftrl": "Ftrl", "SGD": "tf.train.GradientDescentOptimizer(learning_rate=0.00002)"}
DENSE_ROWS = 30                    # tables of more rows are row-sharded: h2_embedding (37 rows) among them
SUBSET = ["h2_embedding", "h3_embedding"]   # the other sharded tables stay in HBM: host and HBM slots in one space
K_CHUNK = 16                       # occurrences per chunk of a hot row's gradient sum (sparse_dev.cuh kChunk)


def _plans(fc, cross, model, model_type, G, per, max_ids, host_tables, emb_dim=None, **kw):
    return [Plan(fc, cross, model, model_type, max_batch=per, embedding_dim_override=emb_dim, gemm_engine="ffma",
                 max_nnz=per * max_ids, max_keys=per * max_ids, dense_exchange_max_rows=DENSE_ROWS, shard_world=G, shard_rank=r,
                 shard_slack=float(G), host_tables=host_tables, **kw) for r in range(G)]


def _sharded_tables(plan):
    return [t["name"] for t in plan.tables if t["sharded"]]


def _group(plans, om):
    grp = LocalShardGroup([WideDeepModel(p) for p in plans])
    for name in grp.models[0].tensor_names():
        grp.set_tensor(name, om.params[name])
        slots = om.slots[name]
        if "acc" in slots:
            grp.set_tensor(name, slots["acc"], slot=1)
        if "n" in slots:
            grp.set_tensor(name, slots["n"], slot=1)
            grp.set_tensor(name, slots["z"], slot=2)
    return grp


def _all_tensors(grp):
    out = {}
    m0 = grp.models[0]
    for name in m0.tensor_names():
        for s in range(m0.n_slots(name) + 1):
            out["%s/slot%d" % (name, s)] = grp.get_tensor(name, slot=s)
    return out


def _assert_bytes_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def _max_occurrences(grp, table):
    """Most occurrences of one row of `table` in the step just run, over every rank's ids."""
    plan = grp.models[0].plan
    t = [i for i, x in enumerate(plan.tables) if x["name"] == table][0]
    ci = [i for i, c in enumerate(plan.columns) if c.emb_table == t][0]
    C = len(plan.columns)
    ids = []
    for m in grp.models:
        offs, col_ids = m.column_ids()
        col = np.repeat(np.tile(np.arange(C), (len(offs) - 1) // C), np.diff(offs))
        ids.append(col_ids[col == ci])
    ids = np.concatenate(ids)
    ids = ids[ids >= 0]
    return int(np.bincount(ids).max()) if len(ids) else 0


def _run_pair(model_type, opt, G, placement, emb_dim=None, multihot_max=3, max_ids=64, per=None):
    fc, cross, model = small_conf(dnn_opt=OPTS[opt])
    per = per or 512 // G
    B = per * G
    om = OM.OracleModel(fc, cross, model, model_type, embedding_dim_override=emb_dim).init(7 + G)
    rng = np.random.default_rng(31 + G)
    if om.use_wide:
        for c in om.wide_cols:
            om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
    ref_plans = _plans(fc, cross, model, model_type, G, per, max_ids, [], emb_dim)
    host = _sharded_tables(ref_plans[0]) if placement == "all" else SUBSET
    assert set(host) <= set(_sharded_tables(ref_plans[0]))
    if placement == "subset":
        assert set(_sharded_tables(ref_plans[0])) - set(host)
    ref = _group(ref_plans, om)
    hst = _group(_plans(fc, cross, model, model_type, G, per, max_ids, host, emb_dim), om)
    assert all(m.memory_usage()[1] == 0 for m in ref.models) and all(m.memory_usage()[1] > 0 for m in hst.models)
    plan0 = ref.models[0].plan
    lr, lh = [], []
    for step in range(4):
        raw = random_raw_batch(fc, B, rng, multihot_max=multihot_max)
        label = (rng.random(B) < 0.3).astype(np.float32)
        shards = [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
        lr.append(ref.train_step(shards))
        lh.append(hst.train_step(shards))
        if step == 0:                              # the chunked combine of hot rows runs before a staged apply
            assert _max_occurrences(hst, "h2_embedding") > K_CHUNK
    lr, lh = np.float32(lr), np.float32(lh)
    assert np.isfinite(lr).all() and lh.tobytes() == lr.tobytes(), (lh, lr)
    _assert_bytes_equal(_all_tensors(hst), _all_tensors(ref))
    raw = random_raw_batch(fc, B, rng, multihot_max=multihot_max)
    label = (rng.random(B) < 0.3).astype(np.float32)
    shards = [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
    assert np.concatenate(hst.forward(shards)).tobytes() == np.concatenate(ref.forward(shards)).tobytes()


@pytest.mark.parametrize("placement", ["all", "subset"])
@pytest.mark.parametrize("opt", sorted(OPTS))
@pytest.mark.parametrize("model_type", ["wide_deep", "deep"])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_sharded_host_tables_bit_identical(G, model_type, opt, placement):
    """4 train steps of 512 examples with multihot bags, empty bags and dropped ids, then a forward: losses, logits, every
    parameter and optimizer slot byte-equal to the HBM-sharded model."""
    _run_pair(model_type, opt, G, placement)


@pytest.mark.parametrize("G", [2, 4])
def test_sharded_host_tables_wide_records(G):
    """64-wide embeddings (Adagrad record of 128 floats) and bags of up to 10 ids."""
    _run_pair("wide_deep", "Adagrad", G, "subset", emb_dim=64, multihot_max=10, max_ids=320)


def test_forward_of_a_fresh_sharded_host_model():
    """Forward-only calls group and stage the owned host rows themselves and write nothing back."""
    G, per = 2, 96
    fc, cross, model = small_conf()
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(13)
    ref_plans = _plans(fc, cross, model, "wide_deep", G, per, 64, [])
    ref = _group(ref_plans, om)
    hst = _group(_plans(fc, cross, model, "wide_deep", G, per, 64, _sharded_tables(ref_plans[0])), om)
    before = _all_tensors(hst)
    rng = np.random.default_rng(17)
    for _ in range(3):
        raw = random_raw_batch(fc, G * per, rng)
        label = (rng.random(G * per) < 0.3).astype(np.float32)
        shards = [to_product_batch(ref_plans[0], slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
        assert np.concatenate(hst.forward(shards)).tobytes() == np.concatenate(ref.forward(shards)).tobytes()
    _assert_bytes_equal(_all_tensors(hst), before)
    _assert_bytes_equal(_all_tensors(hst), _all_tensors(ref))


@pytest.mark.parametrize("same_gpu", [True, False])
def test_sharded_host_tables_in_separate_processes(same_gpu):
    """The multi-process driver (CUDA IPC, flag barriers, step graph replay): every rank trains an HBM-sharded and a
    host-sharded model on the same batches and compares them byte for byte."""
    import torch
    n = torch.cuda.device_count()
    if not same_gpu and n < 2:
        pytest.skip("needs 2 GPUs")
    world = 2 if same_gpu else min(n, 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", "29661", os.path.join(ROOT, "tests", "_shard_host_worker.py")]
    env = dict(os.environ)
    if same_gpu:
        env["WD_SHARD_SAME_GPU"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0 and "SHARD_HOST_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_memory_usage_per_rank():
    """Each rank reports its own host shards; its HBM falls by them, less the owner staging buffer."""
    G, per, max_ids = 3, 64, 64
    fc, cross, model = small_conf()
    ref_plans = _plans(fc, cross, model, "wide_deep", G, per, max_ids, [])
    host_plans = _plans(fc, cross, model, "wide_deep", G, per, max_ids, SUBSET)
    nslots = 1                                                         # Adagrad
    by_name = {t["name"]: t for t in ref_plans[0].tables}
    stride = {n: ((by_name[n]["dim"] + 3) // 4 * 4) * (1 + nslots) for n in SUBSET}
    # the owner staging buffer: one row of the widest host record per id a rank can receive (max_nnz x shard_slack), plus one
    stage = (per * max_ids * G + 1) * max(stride.values()) * 4
    for r in range(G):
        ref, hst = WideDeepModel(ref_plans[r]), WideDeepModel(host_plans[r])
        table_bytes = sum((by_name[n]["rows"] - r + G - 1) // G * stride[n] * 4 for n in SUBSET)     # rows r, r + G, ...
        dev_ref, host_ref = ref.memory_usage()
        dev_host, host_host = hst.memory_usage()
        assert host_ref == 0 and host_host == table_bytes, (r, host_host, table_bytes)
        assert abs((dev_ref - dev_host) - (table_bytes - stage)) < 4096, (r, dev_ref, dev_host, table_bytes, stage)
        ref.close()
        hst.close()


def test_refusals_and_auto_placement():
    G, per = 2, 64
    fc, cross, model = small_conf()
    # a replicated table (h1 has 1000 rows <= dense_exchange_max_rows 4000) forced to the host
    plan = Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * 64, max_keys=per * 64, gemm_engine="ffma",
                dense_exchange_max_rows=4000, shard_world=G, shard_rank=0, shard_slack=float(G), host_tables=["h1_embedding"])
    assert not [t for t in plan.tables if t["name"] == "h1_embedding"][0]["sharded"]
    with pytest.raises(_native.NativeError) as e:
        WideDeepModel(plan)
    assert e.value.code == _native.EUNSUPPORTED
    # the HBM cache stays a single-GPU feature
    with pytest.raises(_native.NativeError) as e:
        WideDeepModel(_plans(fc, cross, model, "wide_deep", G, per, 64, SUBSET, host_cache_bytes=1 << 20)[0])
    assert e.value.code == _native.EUNSUPPORTED
    # auto: every table fits, nothing goes to the host on any rank
    for p in _plans(fc, cross, model, "wide_deep", G, per, 64, None):
        pm = WideDeepModel(p)
        assert pm.memory_usage()[1] == 0
        pm.close()
