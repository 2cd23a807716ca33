"""Evaluation and prediction of row-sharded models: every rank adds the metrics of its own rows on the device, one collective sums
the accumulators of all ranks in rank order (wd_shard_eval_finish), and the file's lines are split r, r + G, ... with the tail kept,
so the last steps leave some ranks short and some without rows (n_valid = 0, a one-row placeholder batch).

The G ranks are G handles in one process (LocalShardGroup); the multi-process driver runs under torchrun through python/eval.py and
python/pred.py (test_entry_points_under_torchrun)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import model as OM
from oracle.metrics import EvalAccumulator, thresholds
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from wide_deep_b200.dataset import interleave_ranks, shard_steps
from wide_deep_b200.model import METRIC_KEYS, WideDeepModel
from wide_deep_b200.plan import Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DENSE_ROWS = 400                   # larger tables and wide columns are row-sharded (h1, h3 and three crosses)
COUNT_KEYS = ["accuracy", "accuracy_baseline", "label/mean", "precision", "recall"]   # ratios of sums of 0 / 1 terms


def take_raw(raw, idx):
    """Rows `idx` of an oracle raw batch."""
    out = {}
    for f, v in raw.items():
        if isinstance(v, tuple):
            offs, fp = v
            lens = np.diff(offs)[idx]
            o = np.zeros(len(idx) + 1, dtype=np.int64)
            o[1:] = np.cumsum(lens)
            out[f] = (o, np.concatenate([fp[offs[i]:offs[i + 1]] for i in idx]) if len(idx) else fp[:0])
        else:
            out[f] = v[idx]
    return out


def _load(models, om):
    for pm in models:
        for name in pm.tensor_names():
            pm.set_tensor(name, om.params[name])
            slots = om.slots[name]
            if "acc" in slots:
                pm.set_tensor(name, slots["acc"], slot=1)
            if "n" in slots:
                pm.set_tensor(name, slots["n"], slot=1)
                pm.set_tensor(name, slots["z"], slot=2)


def _rank_batches(plan, raw, label, G, per):
    """Lines r, r + G, ... of rank r in batches of `per`, with a one-row placeholder where the rank has run out."""
    N = len(label)
    steps, n_valid = shard_steps(N, G, per)
    batches = []
    for r in range(G):
        idx = np.arange(r, N, G)
        bs = []
        for s in range(steps):
            sub = idx[s * per:(s + 1) * per]
            assert len(sub) == n_valid[r][s]
            sub = sub if len(sub) else np.array([0])
            bs.append(to_product_batch(plan, take_raw(raw, sub), label[sub]))
        batches.append(bs)
    return steps, n_valid, batches


@pytest.mark.parametrize("placement", ["hbm", "host"])
@pytest.mark.parametrize("model_type", ["wide_deep", "deep"])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_collective_eval_and_predict_order(G, model_type, placement):
    fc, cross, model = small_conf(hidden=(64, 32))
    per = 48
    N = 2 * G * per + G - 1                            # last step: ranks 0 .. G-2 hold one line, rank G-1 none
    om = OM.OracleModel(fc, cross, model, model_type).init(41 + G)
    rng = np.random.default_rng(43 + G)
    if om.use_wide:
        for c in om.wide_cols:
            om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1

    def plan(r, host_tables):
        return Plan(fc, cross, model, model_type, max_batch=per, gemm_engine="ffma", max_nnz=per * 64, max_keys=per * 64,
                    dense_exchange_max_rows=DENSE_ROWS, shard_world=G, shard_rank=r, shard_slack=float(G), host_tables=host_tables)

    plan0 = plan(0, [])
    host = [t["name"] for t in plan0.tables if t["sharded"]] if placement == "host" else []
    assert any(t["sharded"] for t in plan0.tables)
    grp = LocalShardGroup([WideDeepModel(plan(r, host)) for r in range(G)])
    _load(grp.models, om)
    assert all((m.memory_usage()[1] > 0) == (placement == "host") for m in grp.models)
    raw = random_raw_batch(fc, N, rng)
    label = (rng.random(N) < 0.3).astype(np.float32)
    steps, n_valid, batches = _rank_batches(plan0, raw, label, G, per)
    assert steps == 3 and n_valid[:, -1].min() == 0 and n_valid[:, -1].max() == 1

    res = grp.evaluate(batches, n_valid)
    vals = [np.array([d[k] for k in METRIC_KEYS]) for d in res]
    for v in vals[1:]:
        assert v.tobytes() == vals[0].tobytes()
    got = res[0]

    # the same group's forward logits, step by step (rank order inside a step), through the oracle's metrics
    acc = EvalAccumulator()
    per_rank = [[] for _ in range(G)]
    margin = np.inf
    for s in range(steps):
        out = grp.forward([batches[r][s] for r in range(G)])
        lg = [out[r][:n_valid[r][s]] for r in range(G)]
        for r in range(G):
            per_rank[r].append(lg[r])
        x = np.concatenate(lg)
        y = np.concatenate([batches[r][s].label[:n_valid[r][s]] for r in range(G)])
        acc.update(x, y)
        p = (1.0 / (1.0 + np.exp(-x.astype(np.float64)))).astype(np.float32).astype(np.float64)
        margin = min(margin, float(np.abs(p[:, None] - thresholds()[None, :]).min()))
    exp = acc.result()
    for k in COUNT_KEYS:
        assert abs(got[k] - exp[k]) <= 1e-12 * max(abs(exp[k]), 1e-300), (k, got[k], exp[k])
    # every threshold count exact, so the trapezoids match to rounding -- unless a prediction lies within a few fp32 ulps of a
    # threshold, where the kernel's fp32 sigmoid and the oracle's rounded float64 one may fall on either side
    tol = 1e-12 if margin > 3e-7 else 1e-4
    for k in ("auc", "auc_precision_recall"):
        assert abs(got[k] - exp[k]) <= tol * abs(exp[k]), (k, got[k], exp[k], margin)
    # sums of per-row fp32 terms (the kernel's loss and sigmoid)
    for k in ("average_loss", "prediction/mean", "loss"):
        assert abs(got[k] - exp[k]) <= 1e-6 * abs(exp[k]), (k, got[k], exp[k])

    # one GPU holding the same parameters, on the same global steps
    one = WideDeepModel(Plan(fc, cross, model, model_type, max_batch=G * per, gemm_engine="ffma", max_nnz=G * per * 64,
                             max_keys=G * per * 64))
    _load([one], om)
    one.eval_reset()
    for s in range(steps):
        idx = np.concatenate([np.arange(r, N, G)[s * per:(s + 1) * per] for r in range(G)])
        one.eval_accumulate(to_product_batch(plan0, take_raw(raw, idx), label[idx]))
    single = one.eval_finish()
    for k in ("loss", "auc", "average_loss"):
        assert abs(got[k] - single[k]) <= 1e-5 * max(abs(single[k]), 1.0), (k, got[k], single[k])

    # predictions back in file order: line i is line i // G of rank i % G
    mine = interleave_ranks([np.concatenate(p) for p in per_rank])
    ref = np.concatenate([one.forward(to_product_batch(plan0, take_raw(raw, np.arange(lo, min(lo + G * per, N))),
                                                       label[lo:lo + G * per]))[0] for lo in range(0, N, G * per)])
    np.testing.assert_allclose(mine, ref, rtol=1e-5, atol=1e-5)


def test_eval_accumulator_is_per_rank_and_rows_are_masked():
    """wd_eval_finish keeps meaning this rank's accumulator; rows past n_valid count for nothing, whatever their labels."""
    G, per = 2, 32
    fc, cross, model = small_conf()
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(9)
    grp = LocalShardGroup([WideDeepModel(Plan(fc, cross, model, "wide_deep", max_batch=per, gemm_engine="ffma", max_nnz=per * 64,
                                              max_keys=per * 64, dense_exchange_max_rows=DENSE_ROWS, shard_world=G, shard_rank=r,
                                              shard_slack=float(G))) for r in range(G)])
    _load(grp.models, om)
    rng = np.random.default_rng(5)
    raw = random_raw_batch(fc, G * per, rng)
    label = np.ones(G * per, dtype=np.float32)
    plan0 = grp.models[0].plan
    batches = [[to_product_batch(plan0, take_raw(raw, np.arange(r * per, (r + 1) * per)), label[r * per:(r + 1) * per])] for r in range(G)]
    res = grp.evaluate(batches, [[per], [0]])
    assert res[0] == res[1] and res[0]["label/mean"] == 1.0
    assert grp.models[0].eval_finish()["label/mean"] == 1.0
    assert grp.models[1].eval_finish() == dict.fromkeys(METRIC_KEYS, 0.0) | {"accuracy_baseline": 1.0, "auc": 0.0}
    logits = grp.forward([b[0] for b in batches])[0]
    acc = EvalAccumulator()
    acc.update(logits, label[:per])
    assert abs(res[0]["average_loss"] - acc.result()["average_loss"]) <= 1e-6 * acc.result()["average_loss"]


def _run(cmd, env, cwd):
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=cwd, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _metrics(out):
    vals = {}
    for line in out.split("-" * 80)[-1].strip().splitlines():
        k, v = line.split(": ")
        vals[k] = float(v)
    return vals


def _preds(out):
    rows = [l for l in out.splitlines() if l.startswith("Prediction is")]
    return [(int(l.split('"')[1]), float(l.split("(")[1].rstrip("%)"))) for l in rows]


@pytest.mark.parametrize("same_gpu", [True, False])
def test_entry_points_under_torchrun(tmp_path, same_gpu):
    """python/eval.py and python/pred.py under torchrun (one process per rank, CUDA IPC, flag barriers, graph capture and replay,
    a last step in which rank 1 only serves) against the single-process run on the same checkpoint.  --batch_size is per rank, so
    the single process runs a batch of 2 x 64 lines.  The bundled conf with tf_compat_pad off: the reference's '' padding of
    multi-valued fields depends on which lines share a batch, and a rank's batch holds other lines than the single process's."""
    import torch
    n = torch.cuda.device_count()
    if not same_gpu and n < 2:
        pytest.skip("needs 2 GPUs")
    import re
    import shutil
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import input_fn
    from wide_deep_b200.estimator import build_custom_estimator
    conf = tmp_path / "conf"
    shutil.copytree(os.path.join(ROOT, "conf"), conf)
    txt = (conf / "train.yaml").read_text()
    (conf / "train.yaml").write_text(re.sub(r"^train:[ \t]*$", "train:\n  tf_compat_pad: false", txt, count=1, flags=re.M))
    cfg = Config(conf_dir=str(conf))
    assert cfg.train["tf_compat_pad"] is False
    mdir = tmp_path / "model"
    est = build_custom_estimator(str(mdir / "wide_deep"), "wide_deep", config=cfg, max_batch=64)
    train = os.path.join(ROOT, "data", "train", "train1")
    est.train(input_fn=lambda: input_fn(train, None, "train", 64, config=cfg, plan=est.plan))
    est._model.close()                                 # (its HBM goes back before the workers start)
    N = 8 * 128 + 1                                    # 9 steps of 2 x 64 lines; the last one holds one line, on rank 0
    for src, name in (("eval/eval1", "eval.tsv"), ("pred/pred1", "pred.tsv")):
        lines = open(os.path.join(ROOT, "data", src)).read().split("\n")
        (tmp_path / name).write_text("\n".join([l for l in lines if l][:N]) + "\n")
    env = dict(os.environ, PYTHONPATH=ROOT, WD_CONF_DIR=str(conf))
    if same_gpu:
        env["WD_SHARD_SAME_GPU"] = "1"
    py = os.path.join(ROOT, "python")
    tr = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
          "--master-port", "29671" if same_gpu else "29672"]
    ev = ["--model_dir", str(mdir), "--test_data", str(tmp_path / "eval.tsv")]
    one = _metrics(_run([sys.executable, "eval.py"] + ev + ["--batch_size", "128"], env, py))
    two = _metrics(_run(tr + ["eval.py"] + ev + ["--batch_size", "64"], env, py))
    assert sorted(one) == sorted(two) and len(one) == 11, (one, two)
    for k in one:
        assert abs(one[k] - two[k]) <= 1e-5 * max(abs(one[k]), 1.0), (k, one[k], two[k])
    pr = ["--model_dir", str(mdir), "--data_dir", str(tmp_path / "pred.tsv")]
    p1 = _preds(_run([sys.executable, "pred.py"] + pr + ["--batch_size", "128"], env, py))
    p2 = _preds(_run(tr + ["pred.py"] + pr + ["--batch_size", "64"], env, py))
    assert len(p1) == len(p2) == N
    for (c1, v1), (c2, v2) in zip(p1, p2):
        assert c1 == c2 and abs(v1 - v2) <= 0.1 + 1e-9
