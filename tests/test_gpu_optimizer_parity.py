"""Every optimizer update against float64 from the step's own gradients, on every update route (tests/optimizer_ref.py).

Each case runs two models on one plan: A with the optimizers under test, and its twin T with the SGD probe (learning rate 2^24)
for both the linear and the dnn optimizer.  Forward and backward do not depend on the optimizer, so T's probe step
(tests/kernel_ref.py probe_step) gives the exact fp32 gradient A's step applies, to within dg = 2^-24 |g| + 2^-47 |w|.  A step:

1. the same parameters go to A and T; T's probe step gives every gradient;
2. chosen optimizer states go to A's slots (Adam: set_opt_step(t));
3. A's full state is read back, A runs its step along the route under test and its full state is read again;
4. every element of every tensor and slot is compared with ``optimizer_ref.check`` (the bound is derived, not calibrated).

Rows a step cannot touch (from column_ids, not from g != 0) come back bit-identical, except under Adam, whose untouched rows take
the decay and the step.  A continuing step starts from the state A's previous step left instead of an upload, so Adam rows
touched in the previous step and not in this one must take the untouched form (their bit was cleared).

Routes (each asserts what it depends on):
  fused      wd_train_step: emb_grad_sum<true> + chunk_combine<1> for direct and hot rows (some row occurs more than kChunk = 16
             times), wide_grad_sum<true> + chunk_combine<2>, the dense arena through dense_apply_kernel (ffma) or
             dense_vec_kernel<2> (bf16x3; one tower, no crelu: the dense update is split over the two streams); Adam: the
             unfused lists and the untouched passes.  Two steps on different batches, the second continuing.
  split      wd_step_backward + wd_step_apply: emb_apply, wide_apply, dense_vec<1> / dense_reduce + dense_apply; A's own sparse
             gradient lists must hold exactly the touched rows, with T's gradients.
  exchange   dense_exchange_max_rows 3000 (c1, c2 and their wide columns, the bucketized x2): small_scatter / small_apply and
             Adam's untouched pass over the small tables.
  host       every table in host memory behind an HBM cache that both hits and overflows (staged records); two steps on one
             batch, the second continuing, so the second hits.  Not for an Adam dnn optimizer, which host tables refuse.
  width4     embeddings 4 wide: chunk_combine_kernel's lane groups of one lane, 32 chunks per step.
  width128   embeddings 128 wide: lane groups of 32 lanes, one chunk per step.
             A plan and wd_model_create take any width that is a multiple of 4, but the embedding forward
             (sparse_forward_emb) runs only 4, 8, ..., 128 and refuses a train step on any other width, so the list width
             (the widest table) is always one of those and the embeddings' update always has its lane-group branch;
             test_train_step_refuses_other_widths holds that.  The combine's scalar branch is the wide rows' (width 1), in
             every case.
  crelu      crelu layers with a stateful dnn optimizer: after crelu_mirror the tied half must be minus the updated half (a
             forward of A equals, bit for bit, one of T after T takes A's parameters; the tied half's slots are never read).
  graph      the fused step as the 1st to 4th step of one handle (the 3rd is captured, the 4th replays: graph_stats shows
             both), states re-uploaded.

Every batch has examples of weight 0 whose c1 and tags ids no other example uses, so some rows are touched with g exactly 0
(FTRL still rebuilds w from (z, n), RMSProp still decays ms).  Hidden widths 129 and 33 and the scalar logits bias exercise the
arena's tail lanes.  The worst ratio per (optimizer, route, tensor kind) is printed at the end; every one must be <= 1.
"""
from collections import defaultdict

import numpy as np
import pytest

from oracle import hashing as OH
from tests import kernel_ref as KR
from tests import optimizer_ref as R
from tests.helpers import to_product_batch
from tests.test_gpu_host_cache import _bytes_for
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

B = 384
K_CHUNK = 16
HIDDEN = (129, 33)
N_ZERO = 24                                   # examples of weight 0 per batch, with ids of their own
OPTS = {
    "adagrad": "Adagrad",
    "ftrl_l1l2": "tf.train.FtrlOptimizer(learning_rate=0.1,l1_regularization_strength=0.5,l2_regularization_strength=1.0)",
    "ftrl": "tf.train.FtrlOptimizer(learning_rate=0.1)",
    "rmsprop": "tf.train.RMSPropOptimizer(learning_rate=0.05,decay=0.8)",
    "rmsprop_mom": "tf.train.RMSPropOptimizer(learning_rate=0.05,decay=0.8,momentum=0.5)",
    "adam": "Adam",
    "adam_b08": "tf.train.AdamOptimizer(learning_rate=0.01,beta1=0.8)",
    "sgd": "tf.train.GradientDescentOptimizer(learning_rate=0.01)",
}
# (linear optimizer, dnn optimizer): every optimizer runs on the wide records and on the embedding records and dense arena
PAIRS = [("ftrl_l1l2", "adagrad"), ("adagrad", "ftrl_l1l2"), ("ftrl", "rmsprop_mom"), ("rmsprop_mom", "ftrl"),
         ("rmsprop", "adam"), ("adam_b08", "rmsprop"), ("adam", "sgd"), ("sgd", "adam_b08")]
ADAM_T = (0, 1, 5000)
WORST = defaultdict(float)                    # (optimizer, route, tensor kind) -> worst ratio


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print()
    for (opt, route, kind), w in sorted(WORST.items()):
        print("%-12s %-9s %-15s worst ratio %.3g" % (opt, route, kind, w))


def _id(p):
    return "%s-%s" % p


# ------------------------------------------------------------------------------------------------ models and batches
def make_plan(lin, dnn, engine="ffma", act="relu", emb=8, **kw):
    fc, cross, model = KR.parity_conf(HIDDEN if act != "crelu" else (48, 33), act=act, bn=1)
    model = dict(model, linear_optimizer=OPTS[lin] if lin in OPTS else lin, dnn_optimizer=OPTS[dnn] if dnn in OPTS else dnn)
    return Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, max_nnz=B * 40, max_keys=B * 40,
                gemm_engine=engine, **kw)


def make_pair(lin, dnn, host_cache_sets=None, **kw):
    plan = make_plan(lin, dnn, **kw)
    if host_cache_sets is not None:
        plan.host_cache_bytes = _bytes_for(plan, host_cache_sets)
    kw.pop("host_tables", None)
    return WideDeepModel(plan), WideDeepModel(make_plan(KR.SGD_PROBE, KR.SGD_PROBE, **kw))


def make_batch(plan, rng):
    """parity_conf's batch (c2 and tags have hot rows) whose first N_ZERO examples have weight 0 and c1 / tags ids of their own."""
    raw = KR.raw_batch(B, rng)
    offs, fp = raw["c1"]
    fp = fp.copy()
    fp[:N_ZERO] = OH.fingerprint64_tokens(["c1_only_zero_weight_%d" % i for i in range(N_ZERO)])
    raw["c1"] = (offs, fp)
    offs, fp = raw["tags"]
    fp = fp.copy()
    n = int(offs[N_ZERO])
    fp[:n] = OH.fingerprint64_tokens(["t_only_zero_weight_%d" % i for i in range(n)])
    raw["tags"] = (offs, fp)
    weight = (rng.random(B) + 0.5).astype(np.float32)
    weight[:N_ZERO] = 0
    return to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32), weight)


def tensor_kind(plan, name):
    kind = plan.tensor_names[name][0]
    return {0: "wide", 1: "emb", 2: "dense", 3: "bias"}[kind]


def opt_of(plan, name):
    return plan.lin_opt if name.startswith("linear/") else plan.dnn_opt


def read_state(pm):
    """name -> (w, s1, s2) fp32 as the model holds them (zeros for slots the optimizer does not have)."""
    out = {}
    for name in pm.tensor_names():
        w = pm.get_tensor(name)
        s = [pm.get_tensor(name, slot=k) if k <= pm.n_slots(name) else np.zeros_like(w) for k in (1, 2)]
        out[name] = (w, s[0], s[1])
    return out


def touched_rows(pm):
    """name -> boolean mask of the rows the last batch touches (embedding tables and wide columns), and the most occurrences of
    one embedding row."""
    plan = pm.plan
    offs, ids = pm.column_ids()
    C = len(plan.columns)
    col = np.repeat(np.tile(np.arange(C), (len(offs) - 1) // C), np.diff(offs))
    out, hottest = {}, 0
    for c in plan.columns:
        v = ids[col == plan._col_index[id(c)]]
        if c.emb_table >= 0:
            tb = plan.tables[c.emb_table]
            v = v[(v >= 0) & (v < tb["rows"])]
            cnt = np.bincount(v, minlength=tb["rows"])
            out["dnn/input_from_feature_columns/input_layer/%s/embedding_weights" % tb["name"]] = cnt > 0
            hottest = max(hottest, int(cnt.max(initial=0)))
        if c in plan.wide_columns:
            v = ids[col == plan._col_index[id(c)]]
            v = v[(v >= 0) & (v < c.buckets)]
            out["linear/linear_model/%s/weights" % c.name] = np.bincount(v, minlength=c.buckets) > 0
    return out, hottest


# ------------------------------------------------------------------------------------------------ optimizer states
def make_slots(plan, grads, params, rng):
    """Slot values for A: Adagrad acc in [1e-6, 1e3]; FTRL n in [1e-6, 1e3] with z placing |z1| within 1% of l1 on both signs
    for about 10% of the elements (w stays the uploaded one, inconsistent with (z, n)); RMSProp ms in [1e-6, 1e2] and 0 on 10%,
    momentum up to 0.1; Adam m up to 0.1 and v in [1e-8, 1], v = 0 on 10% (m = 0 on half of those)."""
    out = {}
    for name, (_, _, _, shape) in plan.tensor_names.items():
        o = opt_of(plan, name)
        n = int(np.prod(shape))
        logu = lambda lo, hi: 10.0 ** rng.uniform(lo, hi, n)
        sel = rng.random(n) < 0.1
        k = o["kind"]
        if k == "adagrad":
            s = [logu(-6, 3)]
        elif k == "ftrl":
            acc, z = logu(-6, 3), rng.standard_normal(n) * logu(-3, 0)
            g, w = grads[name].reshape(-1), params[name].astype(np.float64).reshape(-1)
            lr, l1 = R.f32(o["lr"]), R.f32(o["l1"])
            target = np.where(rng.random(n) < 0.5, -1.0, 1.0) * l1 * (1 + rng.uniform(-0.01, 0.01, n))
            near = target - (g - (np.sqrt(acc + g * g) - np.sqrt(acc)) / lr * w)
            s = [acc, np.where(sel, near, z)]
        elif k == "rmsprop":
            s = [np.where(sel, 0.0, logu(-6, 2)), rng.standard_normal(n) * logu(-4, -1)]
        elif k == "adam":
            half = rng.random(n) < 0.5
            s = [np.where(sel & half, 0.0, rng.standard_normal(n) * logu(-4, -1)), np.where(sel, 0.0, logu(-8, 0))]
        else:
            s = []
        out[name] = [np.asarray(x, dtype=np.float32).reshape(shape) for x in s]
    return out


def upload(pm, params, slots=None):
    for name, v in params.items():
        pm.set_tensor(name, v)
        for k, s in enumerate((slots or {}).get(name, [])):
            pm.set_tensor(name, s, slot=k + 1)


# ------------------------------------------------------------------------------------------------ one checked step
def check_step(route, pm, keys, before, after, grads, touched, steps, label):
    """Compare every element of every tensor and slot of one step (keys: the OPTS names of the linear and the dnn optimizer);
    record the worst ratios; -> list of failures."""
    plan = pm.plan
    bad = []
    for name, (w, s1, s2) in before.items():
        o = opt_of(plan, name)
        kind = o["kind"]
        okey = keys[0] if name.startswith("linear/") else keys[1]
        tk = tensor_kind(plan, name)
        aw, as1, as2 = after[name]
        g = grads[name].reshape(w.shape)
        dg = 2.0 ** -24 * np.abs(g) + 2.0 ** -47 * np.abs(w.astype(np.float64))
        if tk in ("dense", "bias"):
            groups = [(tk, np.ones(w.shape[0], dtype=bool), True)]
        else:
            m = touched[name]
            groups = [(tk, m, True), (tk + " untouched", ~m, False)]
        for gk, rows, is_touched in groups:
            if not rows.any():
                continue
            sub = lambda a: a[rows]
            if not is_touched and kind != "adam":
                for a, b, s in ((w, aw, "w"), (s1, as1, "s1"), (s2, as2, "s2")):
                    if not np.array_equal(sub(a), sub(b)):
                        bad.append("%s %s %s: an untouched row changed" % (label, name, s))
                WORST[okey, route, gk] = max(WORST[okey, route, gk], 0.0)
                continue
            res = R.check(kind, o, (sub(w), sub(s1), sub(s2)), sub(g) if is_touched else np.zeros_like(sub(w)),
                          (sub(aw), sub(as1), sub(as2)), dg=sub(dg) if is_touched else 0.0, steps=steps, touched=is_touched,
                          dense=tk in ("dense", "bias"))
            for out, r in res.ratio.items():
                worst = float(r.max(initial=0.0))
                WORST[okey, route, gk] = max(WORST[okey, route, gk], worst)
                if not worst <= 1.0:
                    i = np.unravel_index(int(np.argmax(r)), r.shape)
                    gpu = (sub(aw), sub(as1), sub(as2))[R.OUTS.index(out)][i]
                    bad.append("%s %s [%s] %s: ratio %.3g at %s (gpu %r, ref %r, bound %.3g; in w %r s1 %r s2 %r g %r)" % (
                        label, name, gk, out, worst, i, float(gpu), float(res.ref[out][i]), float(res.bound[out][i]),
                        float(sub(w)[i]), float(sub(s1)[i]), float(sub(s2)[i]), float(sub(g)[i]) if is_touched else 0.0))
    return bad


class Case(object):
    """One handle pair and its batches; step() runs and checks one step of A along `how`."""

    def __init__(self, route, lin, dnn, seed, **plan_kw):
        self.route, self.lin, self.dnn = route, lin, dnn
        self.A, self.T = make_pair(lin, dnn, **plan_kw)
        self.plan = self.A.plan
        self.rng = np.random.default_rng(seed)
        self.adam = "adam" in (self.plan.lin_opt["kind"], self.plan.dnn_opt["kind"])
        self.t = None
        self.facts = defaultdict(int)
        self.prev_touched = None

    def close(self):
        self.A.close()
        self.T.close()

    def step(self, batch, fresh=True, t=0, how="train", premise=None):
        A, T, plan = self.A, self.T, self.plan
        if fresh:
            params = KR.random_params([(n, s[3]) for n, s in plan.tensor_names.items()], self.rng, plan.activation)
            upload(A, params)
        before = read_state(A)
        params = {n: v[0] for n, v in before.items()}
        grads, _ = KR.probe_step(T, batch, params)
        if fresh:
            upload(A, {}, make_slots(plan, grads, params, self.rng))
            if self.adam:
                A.set_opt_step(t)
            self.t = t
            before = read_state(A)
        else:
            self.t += 1
        if how == "train":
            A.train_step(batch)
        else:
            A.step_backward(batch)
            if premise:
                premise(self, grads, before)
            A.step_apply()
        after = read_state(A)
        touched, hottest = touched_rows(A)
        self.facts["hot"] = max(self.facts["hot"], hottest)
        if not fresh and self.prev_touched is not None:        # rows the previous step touched and this one does not
            self.facts["touched_then_untouched"] += sum(int((self.prev_touched[n] & ~m).sum()) for n, m in touched.items())
        self.prev_touched = touched
        for name, m in touched.items():
            g = grads[name].reshape(before[name][0].shape)
            self.facts["zero_g_rows"] += int((m & ~np.any(g.reshape(len(m), -1) != 0, axis=1)).sum())
            self.facts["untouched_rows"] += int((~m).sum())
        label = "%s %s/%s t=%d" % (self.route, self.lin, self.dnn, self.t)
        if plan.host_cache_bytes:
            self.facts["cache"] = A.host_cache_stats()
        return check_step(self.route, A, (self.lin, self.dnn), before, after, grads, touched, self.t, label)


def run(case, steps):
    """steps: list of (batch, fresh, t, how, premise)."""
    bad = []
    try:
        for args in steps:
            bad += case.step(*args)
    finally:
        case.close()
    assert not bad, "\n".join(bad[:20])
    assert case.facts["zero_g_rows"] > 0, "no row was touched with a zero gradient"
    return case.facts


# ------------------------------------------------------------------------------------------------ routes
@pytest.mark.parametrize("engine", ["ffma", "bf16x3"])
@pytest.mark.parametrize("pair", PAIRS, ids=_id)
def test_fused_train_step(pair, engine):
    i = PAIRS.index(pair)
    case = Case("fused", pair[0], pair[1], 10 + i, engine=engine)
    plan = case.plan
    assert len(plan.towers) == 1 and plan.activation != "crelu"
    b1, b2 = make_batch(plan, case.rng), make_batch(plan, case.rng)
    facts = run(case, [(b1, True, ADAM_T[(i + (engine == "bf16x3")) % 3], "train", None), (b2, False, 0, "train", None)])
    assert facts["hot"] > K_CHUNK and facts["touched_then_untouched"] > 0, facts


def _premise(case, grads, before):
    """After step_backward: A's own sparse gradient lists hold exactly the touched rows, with T's gradients."""
    import torch
    from wide_deep_b200.parallel import wrap_device
    A, plan = case.A, case.plan
    dev = torch.device("cuda", A.device)
    touched, _ = touched_rows(A)
    base, acc = {}, 0
    for tb in plan.tables:
        base[tb["name"]] = acc
        acc += tb["rows"]
    for which in (0, 1):
        rows_ptr, grads_ptr, n, width, cap = A.sparse_grads(which)
        torch.cuda.synchronize(dev)
        rows = wrap_device(rows_ptr, (cap,), torch.int32, dev)[:n].cpu().numpy().astype(np.int64)
        lg = wrap_device(grads_ptr, (cap, width), torch.float32, dev)[:n].cpu().numpy().astype(np.float64)
        expect_rows, expect_g, expect_dg = [], [], []
        for name, m in touched.items():
            if (which == 0) != name.startswith("dnn/"):
                continue
            ids = np.nonzero(m)[0]
            if which == 0:
                tb = next(t for t in plan.tables if name.endswith("/%s/embedding_weights" % t["name"]))
                r0, dim = base[tb["name"]], tb["dim"]
            else:
                col = next(c for c in plan.wide_columns if name == "linear/linear_model/%s/weights" % c.name)
                r0, dim = col.wide_base, 1
            g = grads[name].reshape(len(m), -1)[ids]
            w = before[name][0].astype(np.float64).reshape(len(m), -1)[ids]
            expect_rows.append(r0 + ids)
            expect_g.append(np.pad(g, ((0, 0), (0, width - dim)), constant_values=np.nan))
            expect_dg.append(np.pad(2.0 ** -24 * np.abs(g) + 2.0 ** -47 * np.abs(w), ((0, 0), (0, width - dim))))
        er = np.concatenate(expect_rows)
        order = np.argsort(er)
        assert np.array_equal(np.sort(rows), er[order]), "list %d: rows differ from the touched rows" % which
        eg, edg = np.concatenate(expect_g)[order], np.concatenate(expect_dg)[order]
        got = lg[np.argsort(rows)]
        live = ~np.isnan(eg)
        assert np.all(np.abs(got[live] - eg[live]) <= edg[live]), "list %d: gradients differ from the twin's" % which
        case.facts["premise_rows"] += len(rows)


@pytest.mark.parametrize("pair", PAIRS, ids=_id)
def test_split_step(pair):
    i = PAIRS.index(pair)
    case = Case("split", pair[0], pair[1], 30 + i, engine=("ffma", "bf16x3")[i % 2])
    b = make_batch(case.plan, case.rng)
    facts = run(case, [(b, True, ADAM_T[i % 3], "split", _premise)])
    assert facts["premise_rows"] > 0


@pytest.mark.parametrize("pair", PAIRS, ids=_id)
def test_dense_exchange_small_tables(pair):
    i = PAIRS.index(pair)
    case = Case("exchange", pair[0], pair[1], 50 + i, engine=("bf16x3", "ffma")[i % 2], dense_exchange_max_rows=3000)
    plan = case.plan
    small = [t for t in plan.tables if t["rows"] <= 3000]
    assert small and plan.wide_small_base < plan.wide_rows
    b1, b2 = make_batch(plan, case.rng), make_batch(plan, case.rng)
    facts = run(case, [(b1, True, ADAM_T[(i + 2) % 3], "train", None), (b2, False, 0, "train", None)])
    assert facts["hot"] > K_CHUNK and facts["untouched_rows"] > 0 and facts["touched_then_untouched"] > 0, facts


HOST_PAIRS = [p for p in PAIRS if not p[1].startswith("adam")]


@pytest.mark.parametrize("pair", HOST_PAIRS, ids=_id)
def test_host_tables_behind_a_small_cache(pair):
    i = PAIRS.index(pair)
    case = Case("host", pair[0], pair[1], 70 + i, host_tables="all", host_cache_sets=2)
    b = make_batch(case.plan, case.rng)
    facts = run(case, [(b, True, ADAM_T[i % 3], "train", None), (b, False, 0, "train", None)])
    c = facts["cache"]
    assert facts["hot"] > K_CHUNK and c["hits"] > 0 and c["overflow"] > 0, facts


@pytest.mark.parametrize("emb", [4, 128])
@pytest.mark.parametrize("pair", PAIRS, ids=_id)
def test_embedding_widths(pair, emb):
    i = PAIRS.index(pair)
    case = Case("width%d" % emb, pair[0], pair[1], 90 + i + emb, engine=("bf16x3", "ffma")[i % 2], emb=emb)
    assert case.plan.tables[0]["dim"] == emb
    b = make_batch(case.plan, case.rng)
    facts = run(case, [(b, True, ADAM_T[i % 3], "train", None)])
    assert facts["hot"] > K_CHUNK


@pytest.mark.parametrize("engine", ["ffma", "bf16x3"])
@pytest.mark.parametrize("dnn", ["ftrl_l1l2", "rmsprop_mom", "adam"])
def test_crelu_tied_half(dnn, engine):
    case = Case("crelu", "adagrad", dnn, 110 + len(dnn), engine=engine, act="crelu")
    A, T, plan = case.A, case.T, case.plan
    b = make_batch(plan, case.rng)
    bad = case.step(b, True, 1)
    # the tied half after crelu_mirror: A's forward equals that of T holding A's parameters (an upload derives the tied half)
    now = read_state(A)
    for name, (w, _, _) in now.items():
        T.set_tensor(name, w)
    A.forward(b)
    T.forward(b)
    for l in range(len(plan.towers[0]["hidden"])):
        ha, ht = A.hidden_output(0, l, B), T.hidden_output(0, l, B)
        if ha.tobytes() != ht.tobytes():
            bad.append("crelu layer %d: the tied half is not minus the updated half" % l)
    case.close()
    assert not bad, "\n".join(bad[:20])


@pytest.mark.parametrize("pair", [("ftrl_l1l2", "rmsprop_mom"), ("adam_b08", "adagrad")], ids=_id)
def test_graph_replay(pair):
    """Steps 1 to 4 of one handle with states re-uploaded before each: the 3rd step is captured into the step graph and the 4th
    replays it; every one is checked."""
    case = Case("graph", pair[0], pair[1], 130, engine="bf16x3")
    b = make_batch(case.plan, case.rng)
    stats = []
    case.A.train_step = _recording(case.A, case.A.train_step, stats)
    run(case, [(b, True, t, "train", None) for t in (0, 1, 5000, 1)])
    # (a capture that fails leaves the model eager without an error)
    assert [s["captures"] for s in stats] == [0, 0, 1, 1] and [s["replays"] for s in stats] == [0, 0, 0, 1], stats


def _recording(pm, train_step, stats):
    def step(batch):
        loss = train_step(batch)
        stats.append(pm.graph_stats())
        return loss
    return step


def test_train_step_refuses_other_widths():
    """Embeddings 12 wide: the plan and the model are built, the train step is refused by the embedding forward."""
    from wide_deep_b200._native import NativeError
    plan = make_plan("adagrad", "adagrad", emb=12)
    pm = WideDeepModel(plan)
    try:
        with pytest.raises(NativeError, match="unsupported embedding width 12"):
            pm.train_step(make_batch(plan, np.random.default_rng(0)))
    finally:
        pm.close()
