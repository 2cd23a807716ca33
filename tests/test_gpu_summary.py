"""Layer summaries on the GPU (csrc/summary.cu): the statistics of an armed train step against numpy on the values the step produced,
armed steps leaving training untouched, row-sharded ranks merging to one GPU's statistics, and the event files of the entry
points."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from tests.test_gpu_sharded import make_group
from tests.test_parallel_gloo import slice_raw
from tests.test_summary_host import read_events
from wide_deep_b200 import summary as S
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def expect(values):
    """(counts, num, zeros, min, max, sum, sum of squares) of float32 values, as the library defines them."""
    d = np.asarray(values, dtype=np.float32).astype(np.float64).ravel()
    counts = np.zeros(1551, dtype=np.int64)
    np.add.at(counts, np.searchsorted(S.bucket_limits(), d, side="right"), 1)
    return counts, d.size, int(np.count_nonzero(d == 0.0)), d.min(), d.max(), d.sum(), (d * d).sum(), np.abs(d).sum()


def check_segment(stats, key, values, what):
    i = stats.index(key)
    counts, num, zeros, mn, mx, sm, sq, asum = expect(values)
    assert tuple(stats.ints[i]) == (num, zeros, 0), what
    assert np.array_equal(stats.counts[i], counts), what
    assert stats.reals[i, 0] == mn and stats.reals[i, 1] == mx, what
    assert abs(stats.reals[i, 2] - sm) <= 1e-12 * max(asum, 1e-300), what
    assert abs(stats.reals[i, 3] - sq) <= 1e-12 * max(sq, 1e-300), what


def build(hidden=(48, 32), mode="simple", act="relu", bn=1, dropout=None, engine="ffma", B=200, model_type="wide_deep", seed=0):
    fc, cross, model = small_conf(hidden=hidden, mode=mode, act=act, bn=bn)
    model["dnn_dropout"] = dropout
    plan = Plan(fc, cross, model, model_type, max_batch=max(B, 8), max_nnz=max(B, 8) * 64, max_keys=max(B, 8) * 64, gemm_engine=engine)
    pm = WideDeepModel(plan).init(seed)
    rng = np.random.default_rng(seed)
    if bn:                                               # gamma / beta away from 1 / 0, so the affine matters
        for t, tw in enumerate(plan.towers):
            for l in range(len(tw["hidden"])):
                pre = "dnn/dnn_%d/hiddenlayer_%d/batch_normalization/" % (t + 1, l)
                shape = plan.tensor_names[pre + "gamma"][3]        # (crelu: 2u features)
                pm.set_tensor(pre + "gamma", 1 + 0.3 * rng.standard_normal(shape).astype(np.float32))
                pm.set_tensor(pre + "beta", 0.2 * rng.standard_normal(shape).astype(np.float32))
    return fc, plan, pm, rng


def batch(fc, plan, B, rng):
    return to_product_batch(plan, random_raw_batch(fc, B, rng), (rng.random(B) < 0.3).astype(np.float32))


CASES = [dict(), dict(bn=0), dict(dropout=0.3), dict(dropout=0.25, bn=0), dict(act="crelu"), dict(mode="first_dense"),
         dict(mode="last_dense"), dict(mode="dense", dropout=0.2), dict(mode="resnet"), dict(B=1), dict(B=257, hidden=(40, 24))]


@pytest.mark.parametrize("engine", ["ffma", "tc3x"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_statistics_equal_numpy_on_step_values(engine, case):
    kw = dict(CASES[case])
    B = kw.pop("B", 200)
    fc, plan, pm, rng = build(engine=engine, B=B, **kw)
    pm.train_step(batch(fc, plan, B, rng))                   # a plain step first: the armed one is the second of the model
    pm.arm_summary()
    pm.train_step(batch(fc, plan, B, rng))
    stats = pm.layer_statistics()
    assert stats.keys == plan.summary_segments()
    keys = stats.keys
    check_segment(stats, (S.SEG_DEEP_INPUT, -1, -1), pm.deep_input(B)[:, real_columns(plan)], "deep input")
    for t, tw in enumerate(plan.towers):
        for l, u in enumerate(tw["hidden"]):
            n = plan.out_width(u)
            h = pm.hidden_output(t, l, B)
            check_segment(stats, (S.SEG_HIDDEN, t, l), h[:, :n], "layer %d %s" % (l, kw))
        i = keys.index((S.SEG_TOWER_LOGITS, t, -1))
        assert stats.ints[i, 0] == B and stats.counts[i].sum() == B
    i = keys.index((S.SEG_WIDE_LOGIT, -1, -1))
    assert stats.ints[i, 0] == B and stats.counts[i].sum() == B
    with pytest.raises(Exception):                           # read once per armed step
        pm.layer_statistics()


def real_columns(plan):
    """The deep input's logical columns (Plan.deep_layout: name -> (logical offset, physical offset, width))."""
    mask = np.zeros(plan.d0_phys, dtype=bool)
    for _, po, width in plan.deep_layout.values():
        mask[po:po + width] = True
    assert mask.sum() == plan.d0
    return mask


def test_bf16x3_last_layer_bit_exact():
    """bf16x3 keeps fp32 H only for the layer the logits read: the rebuilt value equals it bit for bit."""
    for kw in (dict(), dict(dropout=0.3), dict(bn=0, act="crelu")):
        fc, plan, pm, rng = build(engine="bf16x3", B=300, hidden=(64, 40), **kw)
        pm.arm_summary()
        pm.train_step(batch(fc, plan, 300, rng))
        stats = pm.layer_statistics()
        n = plan.out_width(40)
        check_segment(stats, (S.SEG_HIDDEN, 0, 1), pm.hidden_output(0, 1, 300)[:, :n], "bf16x3 last layer %s" % kw)
        i = stats.index((S.SEG_HIDDEN, 0, 0))
        assert stats.ints[i, 0] == 300 * plan.out_width(64)


def snapshot(models):
    out = []
    for m in models:
        for name in m.tensor_names():
            for s in range(m.n_slots(name) + 1):
                out.append(m.get_tensor(name, s).tobytes())
    return out


@pytest.mark.parametrize("no_graph", [False, True])
def test_armed_steps_change_nothing(no_graph, monkeypatch):
    if no_graph:
        monkeypatch.setenv("WD_NO_GRAPH", "1")
    runs = []
    for arm in (False, True):
        fc, plan, pm, rng = build(engine="bf16x3", B=256, dropout=0.1, hidden=(64, 32))
        data = [batch(fc, plan, 256, np.random.default_rng(s)) for s in range(4)]
        losses, launches = [], []
        for step in range(20):
            pm.upload_slot(step % 2, data[step % 4])
            if arm and step % 5 == 0:
                pm.arm_summary()
            l0 = pm.launch_count()
            losses.append(pm.train_step_slot(step % 2))
            launches.append(pm.launch_count() - l0)
            if arm and step % 5 == 0:
                pm.layer_statistics()
        runs.append((losses, snapshot([pm]), launches))
    assert runs[0][0] == runs[1][0]
    assert runs[0][1] == runs[1][1]
    for step in range(20):                               # unarmed steps launch what they launched before
        if step % 5:
            assert runs[1][2][step] == runs[0][2][step], step
        else:
            assert runs[1][2][step] == runs[0][2][step] + 1, step


def group_run(G, arm_every, B=120, seed=3, dropout=None):
    from oracle import model as OM
    fc, cross, model = small_conf(hidden=(48, 32))
    model["dnn_dropout"] = dropout                       # (the keep mask is drawn per rank row: sharded and one GPU differ under it)
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(seed)
    grp = make_group(fc, cross, model, "wide_deep", G, B // G, om, dense_rows=400)
    plan0 = grp.models[0].plan
    rng = np.random.default_rng(seed)
    losses, stats = [], []
    per = B // G
    for step in range(20 if arm_every else 1):
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        shards = [to_product_batch(plan0, slice_raw(raw, r * per, (r + 1) * per), label[r * per:(r + 1) * per]) for r in range(G)]
        armed = arm_every is not None and (arm_every == 0 or step % arm_every == 0)
        if armed:
            grp.arm_summary()
        losses.append(grp.train_step(shards))
        if armed:
            stats.append(grp.layer_statistics())
    return grp, losses, stats, (fc, cross, model, om, raw, label)


def test_sharded_armed_steps_change_nothing():
    a, la, _, _ = group_run(2, 10 ** 9, dropout=0.2)
    b, lb, sb, _ = group_run(2, 5, dropout=0.2)
    assert la == lb and len(sb) == 4
    assert snapshot(a.models) == snapshot(b.models)


@pytest.mark.parametrize("G", [2, 3])
def test_sharded_statistics_equal_one_gpu(G):
    grp, _, stats, (fc, cross, model, om, raw, label) = group_run(G, 0, B=120)
    from oracle import model as OM
    from tests.helpers import copy_params_to_product
    om1 = OM.OracleModel(fc, cross, model, "wide_deep").init(3)           # the group's initial parameters
    plan = Plan(fc, cross, model, "wide_deep", max_batch=120, max_nnz=120 * 64, max_keys=120 * 64, gemm_engine="ffma",
                dense_exchange_max_rows=400)
    pm = WideDeepModel(plan)
    copy_params_to_product(om1, pm)
    pm.arm_summary()
    pm.train_step(to_product_batch(plan, raw, label))
    s1, sg = pm.layer_statistics(), stats[0]
    assert sg.keys == s1.keys
    assert np.array_equal(sg.counts, s1.counts) and np.array_equal(sg.ints, s1.ints)
    assert np.array_equal(sg.reals[:, :2], s1.reals[:, :2])
    # the ranks' layer values may differ from one GPU's in the last bit (pooling and GEMM order), never across a bucket limit here
    np.testing.assert_allclose(sg.reals[:, 2:], s1.reals[:, 2:], rtol=1e-6)


def test_non_finite_layer_value_raises_with_tag():
    fc, plan, pm, rng = build(B=64)
    beta = pm.get_tensor("dnn/dnn_1/hiddenlayer_1/batch_normalization/beta")
    beta[3] = np.nan
    pm.set_tensor("dnn/dnn_1/hiddenlayer_1/batch_normalization/beta", beta)
    pm.arm_summary()
    pm.train_step(batch(fc, plan, 64, rng))
    ts = S.TrainSummaries(None, 10, 100, plan.summary_layout(), write=False)
    with pytest.raises(ValueError, match="dnn/dnn/dnn_1/hiddenlayer_1/activation"):
        ts.write_step(1, pm.layer_statistics(), 1.0, 64.0)


def test_entry_points_write_event_files(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    mdir = str(tmp_path / "model")
    r = subprocess.run([sys.executable, "train.py", "--model_dir", mdir, "--train_epochs", "1", "--batch_size", "64"],
                       cwd=os.path.join(ROOT, "python"), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    d = os.path.join(mdir, "wide_deep")
    assert glob.glob(os.path.join(d, "events.out.tfevents.*"))
    acc = read_events(d)
    from wide_deep_b200.config import Config
    from wide_deep_b200.plan import compile_plan
    layout = compile_plan(Config(), "wide_deep", 64).summary_layout()
    tags = acc.Tags()
    assert {t + "/activation" for t, _ in layout} <= set(tags["histograms"])
    assert {t + "/fraction_of_zero_values" for t, _ in layout} | {"loss", "average_loss"} <= set(tags["scalars"])
    ev = read_events(os.path.join(d, "eval"))
    assert {"auc", "accuracy", "loss", "average_loss"} <= set(ev.Tags()["scalars"])
    assert "global_step" not in ev.Tags()["scalars"]


def test_torchrun_writes_from_rank_zero_only(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, WD_SHARD_SAME_GPU="1")
    mdir = str(tmp_path / "model")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29691", "train.py", "--model_dir", mdir, "--train_epochs", "1", "--batch_size", "32"],
                       cwd=os.path.join(ROOT, "python"), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    files = glob.glob(os.path.join(mdir, "wide_deep", "events.out.tfevents.*"))
    assert files and all(os.path.getsize(f) > 0 for f in files)
    acc = read_events(os.path.join(mdir, "wide_deep"))
    steps = [e.step for e in acc.Scalars("loss")]
    assert steps and len(steps) == len(set(steps))     # one writer: each summary step once
