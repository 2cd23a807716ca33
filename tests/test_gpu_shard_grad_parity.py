"""Every gradient and every optimizer update of a row-sharded train step against float64 (tests/shard_ref.py), per rank, on a
LocalShardGroup of 2, 3 or 5 ranks on one GPU.

Gradient cases probe the group with SGD at a learning rate of 2^24 (kernel_ref.probe_step, on the group): the reference is
StepRef on the ranks' concatenated values, criterion 1 with the rank-order adds of the all-reduce, criterion 2 held to
test_gpu_kernel_parity.TAU unchanged.  Optimizer cases run an A / T twin as test_gpu_optimizer_parity does: T, an SGD-probe
group on the same batches, gives the exact gradient A's step applies, and every element of every shard and slot of A goes
through optimizer_ref.check.  Every replicated tensor must be byte-identical on every rank; sharded tensors are read through
LocalShardGroup.get_tensor, so the owner mapping is held by the global reference.

Per-rank batches differ in size (one rank has a single example whose multihot bag is empty: no ids of that column), a vocab column
drops its out-of-vocabulary ids, and Zipf-hot tags put rows with more than 16 occurrences, from several ranks, through the owners'
chunked combine.  The multi-process driver runs the same shard_step (test_gpu_shard_drivers holds it byte-identical to
LocalShardGroup).  Run with -s to see the worst ratios per engine and tensor kind."""
from collections import defaultdict

import numpy as np
import pytest

from oracle import hashing as OH
from tests import kernel_ref as KR
from tests import shard_ref as SR
from tests import test_gpu_optimizer_parity as OP
from tests.helpers import to_product_batch
from tests.test_gpu_kernel_parity import TAU
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu

MAX_B = 128
HIDDEN = (129, 33)
WORST1 = defaultdict(float)                   # (engine, kind) -> worst criterion-1 ratio
WORST2 = defaultdict(float)                   # (engine, kind) -> worst criterion-2 tile
WORST_OPT = defaultdict(float)                # (optimizer, tensor kind) -> worst optimizer_ref ratio


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print()
    for k in sorted(WORST1):
        print("%-7s %-10s worst criterion-1 ratio %.3g, worst criterion-2 tile %.3g" % (k[0], k[1], WORST1[k], WORST2[k]))
    for k, w in sorted(WORST_OPT.items()):
        print("%-12s %-15s worst optimizer ratio %.3g" % (k[0], k[1], w))


# ------------------------------------------------------------------------------------------------ groups and batches
def conf(opt_lin=KR.SGD_PROBE, opt_dnn=KR.SGD_PROBE, dropout=0.0, hidden=HIDDEN):
    """parity_conf (c1 3000 and tags 5000 buckets, c2 40, x2 bucketized) and a vocab column of 5 words with OOV tokens."""
    fc, cross, model = KR.parity_conf(hidden, dropout=dropout)
    fc["v"] = dict(type="category", transform="vocab", parameter=["a", "b", "c", "d", "e"])
    model = dict(model, linear_optimizer=opt_lin, dnn_optimizer=opt_dnn)
    return fc, cross, model


def make_group(G, model_type="wide_deep", engine="ffma", emb=8, dense_rows=400, max_batch=MAX_B, host=None, cache=0, **kw):
    fc, cross, model = conf(**kw)
    plans = [Plan(fc, cross, model, model_type, max_batch=max_batch, embedding_dim_override=emb, max_nnz=max_batch * 40,
                  max_keys=max_batch * 40, gemm_engine=engine, dense_exchange_max_rows=dense_rows, shard_world=G, shard_rank=r,
                  shard_slack=float(G), host_tables=host, shard_cache_bytes=cache) for r in range(G)]
    return LocalShardGroup([WideDeepModel(p) for p in plans])


def raw_batch(B, rng, empty_tags=False):
    raw = KR.raw_batch(B, rng)
    if empty_tags:
        raw["tags"] = (np.zeros(B + 1, dtype=np.int64), np.zeros(0, dtype=np.uint64))
    toks = [str(rng.choice(["a", "b", "c", "d", "e", "oov1", "oov2"])) for _ in range(B * 2)]
    raw["v"] = (np.arange(0, 2 * B + 1, 2, dtype=np.int64), OH.fingerprint64_tokens(toks))
    return raw


def batches_for(plan, Bs, rng):
    """One batch per rank; a rank of one example gets an empty tags bag."""
    out = []
    for b in Bs:
        raw = raw_batch(b, rng, empty_tags=b == 1)
        out.append(to_product_batch(plan, raw, (rng.random(b) < 0.3).astype(np.float32), (rng.random(b) + 0.5).astype(np.float32)))
    return out


def full_batches(plan, G, rng):
    """G full batches sliced from one concatenated batch (also returned, for a one-GPU model of max_batch G * MAX_B)."""
    B = G * MAX_B
    raw = raw_batch(B, rng)
    label, weight = (rng.random(B) < 0.3).astype(np.float32), (rng.random(B) + 0.5).astype(np.float32)
    shards = [to_product_batch(plan, slice_raw(raw, r * MAX_B, (r + 1) * MAX_B), label[r * MAX_B:(r + 1) * MAX_B],
                               weight[r * MAX_B:(r + 1) * MAX_B]) for r in range(G)]
    return shards, (raw, label, weight)


def space_facts(grp, Bs):
    """Premises from the ids: the most occurrences of one sharded tags row and on how many ranks they lie, the ranks without any
    tags id, and whether each table space has sharded tensors."""
    plan = grp.models[0].plan
    C = len(plan.columns)
    facts = dict(emb=any(plan.is_sharded_tensor(n) for n in plan.tensor_names if "embedding_weights" in n),
                 wide=any(plan.is_sharded_tensor(n) for n in plan.tensor_names if n.startswith("linear/") and "bias" not in n))
    ti = [i for i, c in enumerate(plan.columns) if c.name == "tags"][0]
    per_rank = []
    for m, b in zip(grp.models, Bs):
        m._rows_hint = b
        offs, ids = m.column_ids()
        col = np.repeat(np.tile(np.arange(C), b), np.diff(offs))
        per_rank.append(ids[col == ti])
    allids = np.concatenate(per_rank)
    hot = np.bincount(allids).argmax() if len(allids) else 0
    facts["hot"] = int((allids == hot).sum())
    facts["hot_ranks"] = sum(int((p == hot).any()) for p in per_rank)
    facts["ranks_without_tags"] = sum(int(len(p) == 0) for p in per_rank)
    return facts


def assert_replicas_identical(grp, slots=(0,)):
    m0 = grp.models[0]
    for name in m0.tensor_names():
        if m0.plan.is_sharded_tensor(name):
            continue
        for s in slots:
            if s > m0.n_slots(name):
                continue
            a = m0.get_tensor(name, s)
            for r, m in enumerate(grp.models[1:], 1):
                assert np.array_equal(a.view(np.uint32), m.get_tensor(name, s).view(np.uint32)), "%s slot %d: rank %d differs" % (name, s, r)


def kind_of(name, plan):
    if name.startswith("tower"):
        return "forward"
    return ("sharded" if plan.is_sharded_tensor(name) else "replicated") if not name.startswith("dnn/dnn_") else "dense"


# ------------------------------------------------------------------------------------------------ gradient cases
def probe(grp, batches, params, engine):
    """One SGD-probe step of the group: every replica identical, every layer output and gradient against GroupStepRef."""
    plan = grp.models[0].plan
    step = grp.models[0].global_step
    for n, v in params.items():
        grp.set_tensor(n, v)
    grp.train_step(batches)
    assert_replicas_identical(grp)
    grads = {n: (params[n].astype(np.float64) - grp.get_tensor(n)) / KR.LR_PROBE for n in params}
    ref = SR.GroupStepRef(grp.models, batches, params, engine, step=step)
    checks = (ref.forward_checks() if plan.use_deep else []) + ref.gradient_checks(grads, params)
    bad = []
    for c in checks:
        kind = kind_of(c.name, plan)
        WORST1[engine, kind] = max(WORST1[engine, kind], c.worst1)
        WORST2[engine, kind] = max(WORST2[engine, kind], c.worst2)
        tau = TAU["forward" if kind == "forward" else "gradient"][engine]
        if not (c.worst1 <= 1.0 and c.worst2 <= tau):
            bad.append(c)
    assert not bad, "\n".join(map(repr, bad))
    for m in grp.models:
        assert m.gemm_fallback_count() == 0
    return grads


def params_for(plan, rng):
    return KR.random_params([(n, s[3]) for n, s in plan.tensor_names.items()], rng, plan.activation)


GRAD_CASES = [
    # (G, per-rank batch sizes, model type, engine, embedding width, dense_exchange_max_rows)
    (2, (65, 128), "wide_deep", "ffma", 8, 400),
    (3, (65, 1, 128), "wide_deep", "bf16x3", 64, 400),
    (3, (128, 65, 1), "wide_deep", "ffma", 4, 3000),
    (5, (65, 1, 128, 17, 100), "deep", "bf16x3", 8, 400),
    (3, (1, 128, 65), "wide", "ffma", 8, 400),
]


@pytest.mark.parametrize("G,Bs,model_type,engine,emb,dense_rows", GRAD_CASES,
                         ids=["G%d-%s-%s-emb%d-rows%d" % (c[0], c[2], c[3], c[4], c[5]) for c in GRAD_CASES])
def test_gradients(G, Bs, model_type, engine, emb, dense_rows):
    """Both table spaces sharded (the wide space routed and served on the auxiliary stream), only the embedding space (deep) or
    only the wide space (wide); c2, v and the bucketized x2 (<= 400 rows) in the all-reduced small-table block, and with 3000
    rows c1 too; embedding widths 4, 8 and 64."""
    grp = make_group(G, model_type, engine, emb, dense_rows)
    plan = grp.models[0].plan
    rng = np.random.default_rng(G * 100 + emb)
    batches = batches_for(plan, Bs, rng)
    probe(grp, batches, params_for(plan, rng), engine)
    f = space_facts(grp, Bs)
    assert f["emb"] == (model_type != "wide") and f["wide"] == (model_type != "deep"), f
    assert f["hot"] > SR.K_CHUNK and f["hot_ranks"] >= 2 and f["ranks_without_tags"] == (1 in Bs), f
    assert model_type == "deep" or plan.is_sharded_tensor("linear/linear_model/c1/weights") == (dense_rows < 3000)
    assert any(not plan.is_sharded_tensor(n) for n in plan.tensor_names if "embedding_weights" in n or "linear/" in n)


@pytest.mark.parametrize("engine", ["ffma", "bf16x3"])
def test_dropout(engine):
    """dnn_dropout 0.25 over two steps.  Step 1: three full batches; the group's layer outputs equal those of one GPU on the
    concatenated batch (the same keep mask), and every rank's mask differs.  Step 2: batches of 65, 1 and 128 rows, against the
    reference's mask at global row r * max_batch + m."""
    G = 3
    grp = make_group(G, engine=engine, dropout=0.25)
    plan = grp.models[0].plan
    rng = np.random.default_rng(40)
    fc, cross, model = conf(dropout=0.25)
    one = WideDeepModel(Plan(fc, cross, model, "wide_deep", max_batch=G * MAX_B, embedding_dim_override=8, max_nnz=G * MAX_B * 40,
                             max_keys=G * MAX_B * 40, gemm_engine=engine))
    shards, (raw, label, weight) = full_batches(plan, G, rng)
    params = params_for(plan, rng)
    probe(grp, shards, params, engine)
    for n, v in params.items():
        one.set_tensor(n, v)
    one.train_step(to_product_batch(one.plan, raw, label, weight))
    for t, tw in enumerate(plan.towers):
        for l in range(len(tw["hidden"])):
            h1 = one.hidden_output(t, l, G * MAX_B)
            hg = np.concatenate([m.hidden_output(t, l, MAX_B) for m in grp.models])
            np.testing.assert_allclose(hg, h1, rtol=1e-4, atol=1e-5, err_msg="tower %d layer %d" % (t, l))
            dropped = [hg[r * MAX_B:(r + 1) * MAX_B] == 0 for r in range(G)]
            assert not np.array_equal(dropped[0], dropped[1]) and not np.array_equal(dropped[1], dropped[2])
    probe(grp, batches_for(plan, (65, 1, 128), rng), params_for(plan, rng), engine)


# ------------------------------------------------------------------------------------------------ optimizer cases
class GroupView(object):
    """The group as test_gpu_optimizer_parity's helpers read one model: global tensors and slots, the concatenated batch's ids."""

    def __init__(self, grp, Bs):
        self.grp, self.plan, self.Bs = grp, grp.models[0].plan, Bs

    def tensor_names(self):
        return self.grp.models[0].tensor_names()

    def n_slots(self, name):
        return self.grp.models[0].n_slots(name)

    def get_tensor(self, name, slot=0):
        return self.grp.get_tensor(name, slot)

    def column_ids(self):
        return SR.group_column_ids(self.grp.models, self.Bs)


def upload_group(grp, params, slots=None):
    for name, v in params.items():
        grp.set_tensor(name, v)
        for k, s in enumerate((slots or {}).get(name, [])):
            grp.set_tensor(name, s, slot=k + 1)


def zero_weight_batches(plan, Bs, rng):
    """batches_for, with the first example of every rank of weight 0 (some touched rows take a gradient of exactly 0)."""
    out = batches_for(plan, Bs, rng)
    for b in out:
        b.weight[:1] = 0
    return out


def run_optimizer(G, lin, dnn, steps, model_type="wide_deep", **kw):
    """steps: per-rank batch sizes of each step; the first uploads fresh parameters and slots (Adam: 5 steps done), the later
    ones continue from A's state.  -> facts"""
    A = make_group(G, model_type, opt_lin=OP.OPTS[lin], opt_dnn=OP.OPTS[dnn], **kw)
    kw.pop("host", None), kw.pop("cache", None)
    T = make_group(G, model_type, **kw)
    plan = A.models[0].plan
    rng = np.random.default_rng(G * 7 + len(lin) + len(dnn))
    adam = "adam" in (plan.lin_opt["kind"], plan.dnn_opt["kind"])
    facts, t, prev, bad = defaultdict(int), 5, None, []
    for i, Bs in enumerate(steps):
        batches = zero_weight_batches(plan, Bs, rng)
        view = GroupView(A, Bs)
        if i == 0:
            upload_group(A, params_for(plan, rng))
        before = OP.read_state(view)
        params = {n: v[0] for n, v in before.items()}
        grads = probe(T, batches, params, "ffma")
        if i == 0:
            upload_group(A, {}, OP.make_slots(plan, grads, params, rng))
            if adam:
                for m in A.models:
                    m.set_opt_step(t)
            before = OP.read_state(view)
        else:
            t += 1
        A.train_step(batches)
        assert_replicas_identical(A, slots=(0, 1, 2))
        after = OP.read_state(view)
        touched, _ = OP.touched_rows(view)
        if prev is not None:
            facts["touched_then_untouched"] += sum(int((prev[n] & ~m).sum()) for n, m in touched.items() if plan.is_sharded_tensor(n))
        prev = touched
        facts["untouched_sharded_rows"] += sum(int((~m).sum()) for n, m in touched.items() if plan.is_sharded_tensor(n))
        bad += OP.check_step("shard", view, (lin, dnn), before, after, grads, touched, t, "G=%d step %d" % (G, i))
    for (okey, route, kind), w in OP.WORST.items():
        if route == "shard":
            WORST_OPT[okey, kind] = max(WORST_OPT[okey, kind], w)
    assert not bad, "\n".join(bad[:20])
    facts["hot"] = space_facts(A, steps[-1])["hot"]
    return facts, A


OPT_CASES = [
    # (G, linear, dnn, per-rank batch sizes of each step)
    (3, "ftrl_l1l2", "adagrad", [(65, 1, 128)]),
    (2, "adagrad", "ftrl", [(128, 65)]),
    (3, "adam_b08", "rmsprop_mom", [(65, 1, 128), (17, 40, 1)]),
    (5, "rmsprop", "adam", [(65, 1, 128, 17, 100), (1, 30, 2, 9, 64)]),
]


@pytest.mark.parametrize("G,lin,dnn,steps", OPT_CASES, ids=["G%d-%s-%s" % c[:3] for c in OPT_CASES])
def test_optimizers(G, lin, dnn, steps):
    """Adagrad, FTRL, RMSProp and Adam on the shards of both table spaces and on the dense arena; Adam's second step runs on a
    smaller batch, so rows the first step touched take the untouched form."""
    facts, _ = run_optimizer(G, lin, dnn, steps)
    assert facts["untouched_sharded_rows"] > 0, facts
    if len(steps) > 1:
        assert facts["touched_then_untouched"] > 0, facts


def test_wide_only_ftrl():
    """A wide-only FTRL model of 3 ranks with every wide column sharded: the all-reduced arena is the wide bias alone, padded to
    4 floats, so ranks 1 and 2 reduce empty slices."""
    facts, A = run_optimizer(3, "ftrl_l1l2", "adagrad", [(65, 1, 128)], model_type="wide", dense_rows=1)
    plan = A.models[0].plan
    assert all(plan.is_sharded_tensor(n) for n in plan.tensor_names if "bias" not in n)
    G = 3
    for m in A.models:
        assert m.dense_grad()[1] == 4                       # the wide bias alone, padded to 4 floats
    n4 = 1                                                   # one float4
    slice4 = (n4 + G - 1) // G
    assert [max(0, min(n4, (r + 1) * slice4) - r * slice4) for r in range(G)] == [1, 0, 0]


@pytest.mark.parametrize("cache", [False, True])
def test_host_shards(cache):
    """Embedding shards of tags and c1 in page-locked host memory, without and behind the owner cache (8 ways x 2 sets)."""
    facts, A = run_optimizer(3, "ftrl", "adagrad", [(65, 1, 128)], host=["tags_embedding", "c1_embedding"],
                             cache=8 * 2 * 16 * 4 if cache else 0)
    if cache:
        st = A.host_cache_stats()
        assert sum(s["hits"] + s["loads"] + s["overflow"] for s in st) > 0, st


def test_host_shards_refuse_adam():
    with pytest.raises(Exception, match="Adam"):
        make_group(2, opt_dnn=OP.OPTS["adam"], host=["tags_embedding"])
