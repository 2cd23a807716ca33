"""The deep input, the wide logit, the logits, the loss and the eval metrics against float64 (tests/input_ref.py), on every gather
path: both pooling kernels at every embedding width, host-placed tables with and without their HBM cache, and row-sharded tables
on a LocalShardGroup of 2 and 3 ranks.  Every reference is built from the batch's own ids (held to the oracle's transform) and
the fp32 tables the GPU read.  Run with -s to see the worst ratio of each check kind."""
from collections import OrderedDict, defaultdict

import numpy as np
import pytest

from oracle import hashing as OH
from oracle import model as OM
from tests import input_ref as IR
from tests.helpers import to_product_batch
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 200, 1000]
MAX_B = 128
WORST = defaultdict(float)
KERNELS = set()


def conf(n_cross=2):
    """Hashed columns of natural widths 2, 4, 8 and 16 (40, 1000, 5000 and 200 000 buckets), a long multihot column, a vocab and an
    identity column (indicators), the four normalisers (min_max and standard with bucketized twins in the wide part), a cross of
    identity and bucketized keys and n_cross hashed crosses with deep embeddings (cheap extra tables)."""
    fc = OrderedDict()
    for f, n in (("w2", 40), ("w4", 1000), ("w8", 5000), ("w16", 200000), ("h5", 300), ("h6", 700)):
        fc[f] = dict(type="category", transform="hash_bucket", parameter=n)
    fc["tags"] = dict(type="category", transform="hash_bucket", parameter=5000)
    fc["v"] = dict(type="category", transform="vocab", parameter=["a", "b", "c", "d", "e"])
    fc["idn"] = dict(type="category", transform="identity", parameter=15)
    fc["xn"] = dict(type="continuous", transform=None, parameter=dict(normalization=None, boundaries=None))
    fc["xm"] = dict(type="continuous", transform="min_max", parameter=dict(normalization=[10, 90], boundaries=[15, 30, 45, 60]))
    fc["xs"] = dict(type="continuous", transform="standard", parameter=dict(normalization=[40.0, 30.0], boundaries=[-1, 0, 1]))
    fc["xl"] = dict(type="continuous", transform="log", parameter=dict(normalization=[0, 1], boundaries=None))
    cross = [(["idn", "xm"], 100, 1)]
    pairs = [(a, b) for i, a in enumerate(["w2", "w4", "w8", "w16", "h5", "h6"]) for b in ["w2", "w4", "w8", "w16", "h5", "h6"][i + 1:]]
    cross += [([a, b], 1500 + 100 * k, 1) for k, (a, b) in enumerate(pairs[:n_cross])]
    model = dict(linear_optimizer="Ftrl", linear_initial_learning_rate=0.01, dnn_hidden_units=[64, 32], dnn_connected_mode="simple",
                 dnn_optimizer="Adagrad", dnn_initial_learning_rate=0.01, dnn_activation_function="relu", dnn_dropout=None,
                 dnn_batch_normalization=0)
    return fc, cross, model


def raw_batch(fc, B, rng, long_bags=True, log_edges=False):
    """Raw batch (oracle format).  tags: bag lengths cycling through LENGTHS (capped at 65 without long_bags), Zipf-hot tokens with
    duplicates; other string fields 0-3 tokens; vocab with OOV tokens; identity values -2 .. buckets + 2; xl > 0 unless log_edges
    (then every third value is 0 or negative)."""
    raw = {}
    for f, c in fc.items():
        if c["type"] == "category" and c["transform"] != "identity":
            if f == "tags":
                lens = np.array([LENGTHS[(i * 5) % len(LENGTHS)] for i in range(B)])
                if B == 1:
                    lens[:] = 1000 if long_bags else 65
                if not long_bags:
                    lens = np.minimum(lens, 65)
                toks = ["t%d" % v for v in (rng.zipf(1.2, size=int(lens.sum())) - 1) % 3000]
            else:
                lens = rng.integers(0, 4, size=B)
                pool = c["parameter"] if c["transform"] == "vocab" else ["%s_%d" % (f, i) for i in range(60)]
                toks = [str(pool[int(rng.integers(len(pool)))]) if rng.random() > 0.2 else "oov%d" % rng.integers(9)
                        for _ in range(int(lens.sum()))]
            offs = np.zeros(B + 1, dtype=np.int64)
            offs[1:] = np.cumsum(lens)
            raw[f] = (offs, OH.fingerprint64_tokens(toks))
        elif c["type"] == "category":
            raw[f] = rng.integers(-2, c["parameter"] + 3, size=B).astype(np.int64)
        elif f == "xl":
            x = np.exp(rng.uniform(-3, 5, size=B))
            if log_edges:
                x[::3] = 0.0
                x[1::3] = -x[1::3]
            raw[f] = x.astype(np.float32)
        else:
            raw[f] = (rng.standard_normal(B) * 30 + 40).astype(np.float32)
    return raw


def pool_kernel(plan, dim):
    """The pooling kernel sparse_forward_emb picks for a physical width: 'rows' or 'warp' (the profile marks cannot tell)."""
    n_cat = max(len(plan.cat_fields), 1)
    keys_cap = plan.max_keys if plan.max_keys > 0 else plan.max_batch * n_cat * 4
    widebag = keys_cap // (plan.max_batch * n_cat) >= 8
    return "rows" if dim == 4 else "warp" if dim == 128 else ("warp" if widebag else "rows")


def make_plan(fc, cross, model, model_type, kernel, emb_dim=None, **kw):
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    keys = MAX_B * n_cat * (6 if kernel == "rows" else 32)
    plan = Plan(fc, cross, model, model_type, max_batch=kw.pop("max_batch", MAX_B), embedding_dim_override=emb_dim,
                max_nnz=MAX_B * 400, max_keys=keys, gemm_engine="ffma", **kw)
    for t in plan.tables:
        want = "rows" if (t["dim"] + 3) // 4 * 4 == 4 else "warp" if t["dim"] == 128 else kernel
        got = pool_kernel(plan, (t["dim"] + 3) // 4 * 4)
        assert got == want, (t["name"], t["dim"], got, want)
        KERNELS.add((t["dim"], got))
    return plan


def set_values(target, plan, rng, scale=1.0):
    """Random fp32 embedding tables (N(0, 0.3) * scale) and wide weights (N(0, 0.1) * scale, bias 0.2)."""
    for name, (_, _, _, shape) in plan.tensor_names.items():
        if "embedding_weights" in name or name.startswith("linear/"):
            sd = 0.3 if "embedding_weights" in name else 0.1
            v = rng.standard_normal(shape) * sd * scale if not name.endswith("bias_weights") else np.full(shape, 0.2)
            target.set_tensor(name, v.astype(np.float32))


def record(kind, res):
    WORST[kind] = max(WORST[kind], res.worst)
    assert res.worst <= 1.0, res


def tables_of(src, plan):
    emb = {t["name"]: src.get_tensor("dnn/input_from_feature_columns/input_layer/%s/embedding_weights" % t["name"]) for t in plan.tables}
    wide = {c.name: src.get_tensor("linear/linear_model/%s/weights" % c.name) for c in plan.wide_columns}
    bias = src.get_tensor("linear/linear_model/bias_weights")[0] if plan.use_wide else 0.0
    return emb, wide, bias


def check_inputs(pm, plan, om, raw, B, emb, G=1, tag=""):
    """X0 of the model's last batch against the reference (every physical column)."""
    offs, ids = pm.column_ids()
    IR.check_transform(om, plan, offs, ids, raw, B)
    if plan.use_deep:
        dense = np.stack([raw[f] for f in plan.dense_fields], axis=1)
        ref, bound, kind = IR.x0_reference(plan, offs, ids, B, emb, dense, G)
        for kd, res in IR.check_x0("X0 %s B=%d" % (tag, B), pm.deep_input(B), ref, bound, kind).items():
            record("x0 " + kd, res)
    return offs, ids


def check_head(pm, plan, batch, logits, offs, ids, wide, bias, G=1):
    B = batch.batch_size
    if plan.model_type == "wide":
        ref, bound = IR.wide_reference(plan, offs, ids, B, wide, bias, G)
        record("wide logit", IR.judge("wide logit", logits, ref, bound))
    elif G == 1:
        params = {n: pm.get_tensor(n) for n in pm.tensor_names()}
        ref, bound = IR.logit_reference(pm, batch, params, "ffma")
        record("logit", IR.judge("logits", logits, ref, bound))


def check_loss(loss, logits, batch):
    ref, bound = IR.loss_reference(logits, batch.label, batch.weight)
    record("loss", IR.judge("loss", np.array([loss]), np.array([ref]), np.array([bound])))


def single_case(model_type, kernel, emb_dim=None, n_cross=2, tf_compat_pad=False, graphs=True, host=None, cache_sets=None,
                monkeypatch=None, seed=0):
    if not graphs:
        monkeypatch.setenv("WD_NO_GRAPH", "1")
    fc, cross, model = conf(n_cross)
    plan = make_plan(fc, cross, model, model_type, kernel, emb_dim, tf_compat_pad=tf_compat_pad, host_tables=host)
    if cache_sets is not None:
        nslots = 1                                                       # Adagrad: one slot per weight
        stride = max((t["dim"] + 3) // 4 * 4 for t in plan.tables) * (1 + nslots)
        plan.host_cache_bytes = 8 * (1 << cache_sets) * stride * 4      # 8 ways: a step both hits and overflows
    om = OM.OracleModel(fc, cross, model, model_type, embedding_dim_override=emb_dim, tf_compat_pad=tf_compat_pad)
    pm = WideDeepModel(plan).init(seed)
    rng = np.random.default_rng(seed + 1)
    long_bags = kernel == "warp" and not tf_compat_pad
    for step, (B, scale) in enumerate([(MAX_B, 1e3), (1, 1.0), (65, 1.0), (MAX_B, 1.0)]):
        set_values(pm, plan, rng, scale)                              # (the first batch's large values would show in a stale row)
        raw = raw_batch(fc, B, rng, long_bags)
        label = (rng.random(B) < 0.3).astype(np.float32)
        weight = (rng.random(B) * 2).astype(np.float32) if step % 2 else None
        batch = to_product_batch(plan, raw, label, weight, tf_compat_pad=tf_compat_pad)
        emb, wide, bias = tables_of(pm, plan)
        logits, loss = pm.forward(batch)
        offs, ids = check_inputs(pm, plan, om, raw, B, emb, tag="forward")
        check_head(pm, plan, batch, logits, offs, ids, wide, bias)
        check_loss(loss, logits, batch)
        if step == 2:                                                  # train_step_slot on a prefetched slot
            pm.prefetch_slot(1, batch)
            loss = pm.train_step_slot(1)
        else:
            loss = pm.train_step(batch)
        check_inputs(pm, plan, om, raw, B, emb, tag="train")
        check_loss(loss, logits, batch)
    # eval over two batches: the metrics of the GPU's own logits
    pm.eval_reset()
    xs, ys, ws = [], [], []
    for B in (65, MAX_B):
        raw = raw_batch(fc, B, rng, long_bags)
        label = (rng.random(B) < 0.4).astype(np.float32)
        weight = (rng.random(B) * 2).astype(np.float32)
        batch = to_product_batch(plan, raw, label, weight, tf_compat_pad=tf_compat_pad)
        logits, _ = pm.forward(batch)
        pm.eval_accumulate(batch)
        xs.append(logits), ys.append(label), ws.append(weight)
    got = pm.eval_finish()
    record("metrics", IR.check_metrics(got, IR.metrics_reference(np.concatenate(xs), np.concatenate(ys), np.concatenate(ws), 2)))
    return pm


@pytest.mark.parametrize("kernel", ["rows", "warp"])
@pytest.mark.parametrize("model_type", ["wide_deep", "deep", "wide"])
def test_natural_widths(model_type, kernel):
    """Widths 2, 4, 8 and 16 in one plan, on both pooling kernels."""
    single_case(model_type, kernel)


@pytest.mark.parametrize("kernel", ["rows", "warp"])
@pytest.mark.parametrize("emb_dim,n_cross", [(32, 15), (64, 8), (128, 2)])
def test_override_widths(emb_dim, n_cross, kernel):
    """Widths 32 (17 tables: a second round of tables in the rows kernel), 64 (9 tables: also a second round) and 128."""
    single_case("wide_deep", kernel, emb_dim, n_cross)


@pytest.mark.parametrize("kernel,tf_compat_pad", [("rows", False), ("warp", True)])
def test_without_graphs(kernel, tf_compat_pad, monkeypatch):
    """WD_NO_GRAPH=1 on both kernels; tf_compat_pad pads every string field to its longest row (on the full-warp kernel only: the
    padded long bags need more keys than a rows-kernel plan holds)."""
    single_case("wide_deep", kernel, tf_compat_pad=tf_compat_pad, graphs=False, monkeypatch=monkeypatch)


@pytest.mark.parametrize("cache_sets", [None, 0])
def test_host_tables(cache_sets):
    """Every table in host memory, without a cache and behind a cache of 8 slots (one step both hits and overflows)."""
    pm = single_case("wide_deep", "rows", host="all", cache_sets=cache_sets)
    if cache_sets is not None:
        st = pm.host_cache_stats()
        assert st["hits"] > 0 and st["overflow"] > 0, st


def test_log_at_zero_and_below():
    """log of 0 is -inf and of a negative value NaN in the deep input, exactly."""
    fc, cross, model = conf()
    plan = make_plan(fc, cross, model, "deep", "rows")
    om = OM.OracleModel(fc, cross, model, "deep")
    pm = WideDeepModel(plan).init(3)
    rng = np.random.default_rng(4)
    raw = raw_batch(fc, 65, rng, long_bags=False, log_edges=True)
    pm.forward(to_product_batch(plan, raw, np.zeros(65, dtype=np.float32)))
    emb, _, _ = tables_of(pm, plan)
    check_inputs(pm, plan, om, raw, 65, emb, tag="log edges")
    X = pm.deep_input(65)[:, plan.deep_layout["xl"][1]]
    assert np.all(np.isneginf(X[::3])) and np.all(np.isnan(X[1::3]))


HOST = ["w8_embedding", "tags_embedding"]


@pytest.mark.parametrize("model_type,G,host,cache", [("wide_deep", 2, None, False), ("wide_deep", 3, None, False), ("wide", 2, None, False),
                                                    ("wide", 3, None, False), ("wide_deep", 2, HOST, False), ("wide_deep", 3, HOST, True)])
def test_sharded_group(model_type, G, host, cache):
    """Row-sharded large tables and wide columns next to replicated small ones (<= 400 rows); host-placed shards with and without
    the owner's cache.  Each rank's X0 against the full tables; the group loss; evaluate with n_valid below the batch."""
    fc, cross, model = conf()
    per = 48
    plans = []
    for r in range(G):
        plans.append(Plan(fc, cross, model, model_type, max_batch=per, max_nnz=per * 400, max_keys=per * 9 * 32, gemm_engine="ffma",
                          dense_exchange_max_rows=400, shard_world=G, shard_rank=r, shard_slack=float(G),
                          host_tables=host, shard_cache_bytes=8 * 2 * 16 * 4 if cache else 0))   # 8 ways x 2 sets of 16 floats
    grp = LocalShardGroup([WideDeepModel(p).init(5) for p in plans])
    plan0 = plans[0]
    assert any(plan0.is_sharded_tensor(n) for n in plan0.tensor_names)
    om = OM.OracleModel(fc, cross, model, model_type)
    rng = np.random.default_rng(11 + G)
    for step in range(2):
        set_values(grp, plan0, rng, 1e3 if step == 0 else 1.0)
        raw = raw_batch(fc, per * G, rng)
        label = (rng.random(per * G) < 0.3).astype(np.float32)
        shards = [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
        emb, wide, bias = tables_of(grp, plan0)
        logits = grp.forward(shards)
        for r, m in enumerate(grp.models):
            m._rows_hint = per
            offs, ids = check_inputs(m, plans[r], om, slice_raw(raw, r * per, (r + 1) * per), per, emb, G=G, tag="rank %d" % r)
            check_head(m, plans[r], shards[r], logits[r], offs, ids, wide, bias, G)
        loss = grp.train_step(shards)
        refs = [IR.loss_reference(logits[r], shards[r].label, None) for r in range(G)]
        ref, bound = sum(v[0] for v in refs), sum(v[1] for v in refs) + 2.0 ** -44 * sum(abs(v[0]) for v in refs)
        record("loss", IR.judge("group loss", np.array([loss]), np.array([ref]), np.array([bound])))
    # evaluate: rank r keeps its first per - 5 r rows
    nv = [per - 5 * r for r in range(G)]
    raw = raw_batch(fc, per * G, rng)
    label = (rng.random(per * G) < 0.4).astype(np.float32)
    shards = [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
    logits = grp.forward(shards)
    got = grp.evaluate([[s] for s in shards], [[n] for n in nv])
    x = np.concatenate([logits[r][:nv[r]] for r in range(G)])
    y = np.concatenate([shards[r].label[:nv[r]] for r in range(G)])
    ref = IR.metrics_reference(x, y, None, 1)
    for g in got:
        record("metrics", IR.check_metrics(g, ref))


def test_zz_report():
    """Worst ratio per check kind over the file, and the pooling kernel of every physical width that ran."""
    print("\n" + "\n".join("%-14s worst ratio %.3g" % kv for kv in sorted(WORST.items())))
    print("pooling kernels (width, kernel): %s" % sorted(KERNELS))
