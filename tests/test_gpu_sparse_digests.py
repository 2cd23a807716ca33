"""Sparse gradient sums and row updates (csrc/sparse.cu, shard.cu, sparse_dev.cuh) held bit for bit.

Whether the updates are right is tests/test_gpu_optimizer_parity.py's question: it holds every element of every update kernel to a
float64 reference under a derived bound.  These digests catch a change, not an error.  The other bitwise tests compare two models
that run the same sparse kernels (host against HBM tables, host against HBM shards), so a rounding change shared by both would
pass them.  These cases hold the losses and every trained tensor and optimizer slot
after four train steps to SHA-256 digests recorded on an H100 80GB HBM3, per rank for the sharded runs.  Every case has rows
touched more than kChunk = 16 times in a step, so both the direct sums and the chunked hot-row combine run:

  adagrad_ftrl      fused single-GPU update: emb_grad_sum<true>, chunk_combine<1>, wide_grad_sum<true>, chunk_combine<2>
  rmsprop_dim64     the same on 64-wide embeddings (other lane widths) with RMSProp
  adam              unfused emb_apply / wide_apply, the dense Adam passes, chunk_combine<0>
  dense_exchange    small tables through the dense block: small_scatter_* / small_apply_*
  split_sorted,     the split step with a world-1 exchange merged by wd_sparse_set_sorted / wd_sparse_set, then the unfused apply
  split_counted
  host_tables       every table in host memory without a cache: staged fused updates, uslot null
  host_cache        the same with a small HBM cache that both hits and overflows: uslot non-null
  shard_g2          LocalShardGroup of 2 ranks, all shards in HBM: peer sums, shard chunk combine, owner apply
  shard_g3_mixed    3 ranks with host and HBM shards in one space: staged owner apply

Several single-GPU cases share a digest: they train the same model along different routes, which must agree bit for bit.
`python -m tests.test_gpu_sparse_digests` prints the digests of the current build and what each case checks."""
import hashlib

import numpy as np
import pytest

from oracle import model as OM
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_host_cache import _bytes_for
from tests.test_gpu_host_tables import _batches, _plan, _train
from tests.test_gpu_parity import small_conf
from tests.test_gpu_sharded_host_tables import K_CHUNK, SUBSET, _group, _max_occurrences, _plans
from tests.test_gpu_step_graphs import split_train
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200.model import WideDeepModel

pytestmark = pytest.mark.gpu

B = 128
STEPS = 4
RMSPROP = "tf.train.RMSPropOptimizer(learning_rate=0.05,momentum=0.5)"
# name -> (small_conf arguments, Plan arguments, host tables, how the steps run)
SINGLE = {
    "adagrad_ftrl": ({}, {}, [], "slots"),
    "rmsprop_dim64": (dict(dnn_opt=RMSPROP, lin_opt="RMSProp"), dict(embedding_dim_override=64), [], "slots"),
    "adam": (dict(dnn_opt="Adam", lin_opt="Adam"), {}, [], "slots"),
    "dense_exchange": ({}, dict(dense_exchange_max_rows=1000), [], "slots"),
    "split_sorted": ({}, {}, [], "sorted"),
    "split_counted": ({}, {}, [], "counted"),
    "host_tables": ({}, {}, "all", "slots"),
    "host_cache": ({}, {}, "all", "slots"),
}
CACHE_SET_BITS = 3            # host_cache: 8 sets of 8 ways, far fewer than the rows of a step
SHARDED = {"shard_g2": (2, []), "shard_g3_mixed": (3, SUBSET)}
DIGESTS = {
    "adagrad_ftrl": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "adam": ["12e75d5edc4572597b1be235ff902fa117e14479a8748b93b85e881d3e087d9e"],
    "dense_exchange": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "host_cache": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "host_tables": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "rmsprop_dim64": ["b74569b00b3c2a15387bcd260c4bdf44a29928c6b96906857c151621be0461cf"],
    "split_counted": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "split_sorted": ["9f5fa30738599662e211f6f7e3ff5824a5e38b86acc63493d302d9a3a745c7c7"],
    "shard_g2": ["ce31a7e721a98ff41a5ba021567d02da7d69df51c6c2d7a522e47e57ebc40d81", "f72fda3b1c949b9f97d6c7344ad67df62bd439e3a81685722adb3acf1dfa913b"],
    "shard_g3_mixed": ["b2dfb1bc0bbc822d85a782cc5853d64fcd40b0fb621ffc603b691468318b4fea", "a83e14147c08fdf185a7522f08f69e931878fd73a1f8fd1067fd3c76c143365f", "66694f8edaf7c86f341ee370d6f281a295e97880baac8c5d096f8729047d9e8f"],
}


class _One(object):
    def __init__(self, pm):
        self.models = [pm]


def _digest(losses, pm):
    h = hashlib.sha256()
    h.update(np.float32(losses).tobytes())
    for name in sorted(pm.tensor_names()):
        for s in range(pm.n_slots(name) + 1):
            h.update(("%s/%d" % (name, s)).encode())
            h.update(np.ascontiguousarray(pm.get_tensor(name, slot=s), dtype=np.float32).tobytes())
    return h.hexdigest()


def run_single(name):
    """Digest of the trained model, and the facts the case must show."""
    conf, kw, host, how = SINGLE[name]
    fc, cross, model = small_conf(**conf)
    plan = _plan(fc, cross, model, B, "warp", host, **kw)
    if name == "host_cache":
        plan.host_cache_bytes = _bytes_for(plan, CACHE_SET_BITS)
    pm = WideDeepModel(plan).init(11)
    batches = _batches(plan, fc, B, STEPS, 5, "warp")
    losses = _train(pm, batches) if how == "slots" else split_train(pm, batches, how)
    out = [_digest(losses, pm)]
    facts = {"finite": bool(np.isfinite(losses).all()), "tables_where_planned": (pm.memory_usage()[1] > 0) == bool(host)}
    if kw.get("dense_exchange_max_rows"):            # small embedding tables and wide columns go through the dense block
        facts["dense_block"] = plan.wide_small_base < plan.wide_rows and any(t["rows"] <= kw["dense_exchange_max_rows"] for t in plan.tables)
    if name == "host_cache":
        c = pm.host_cache_stats()
        facts["cache_hits_and_overflows"] = c["hits"] > 0 and c["overflow"] > 0
    pm.forward(batches[-1])                          # (column_ids reads the ids of the last forward)
    facts["hot_h2"] = _max_occurrences(_One(pm), "h2_embedding") > K_CHUNK
    pm.close()
    return out, facts


def run_sharded(name):
    """Per-rank digests of a LocalShardGroup trained on multihot bags, and the facts the case must show."""
    G, host = SHARDED[name]
    fc, cross, model = small_conf()
    per = 512 // G
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(7 + G)
    grp = _group(_plans(fc, cross, model, "wide_deep", G, per, 64, host), om)
    assert all((m.memory_usage()[1] > 0) == bool(host) for m in grp.models)
    rng = np.random.default_rng(31 + G)
    plan0 = grp.models[0].plan
    losses, hot = [], []
    for _ in range(STEPS):
        raw = random_raw_batch(fc, per * G, rng)
        label = (rng.random(per * G) < 0.3).astype(np.float32)
        losses.append(grp.train_step([to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per])
                                      for r in range(G)]))
        hot.append(_max_occurrences(grp, "h2_embedding"))
    facts = {"finite": bool(np.isfinite(losses).all()), "hot_h2": max(hot) > K_CHUNK}
    return [_digest(losses, m) for m in grp.models], facts


def run(name):
    return run_single(name) if name in SINGLE else run_sharded(name)


@pytest.mark.parametrize("name", sorted(SINGLE) + sorted(SHARDED))
def test_trained_state_matches_recorded_digest(name):
    digests, facts = run(name)
    assert all(facts.values()), facts
    assert digests == DIGESTS[name]


if __name__ == "__main__":
    for name in sorted(SINGLE) + sorted(SHARDED):
        digests, facts = run(name)
        print("    %r: %r,    # %s" % (name, digests, facts), flush=True)
