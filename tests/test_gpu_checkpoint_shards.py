"""Sharded-layout checkpoints of real models (wide_deep_b200/checkpoint.py over wd_tensor_io_rows).

A checkpoint written by G ranks restores into G' ranks byte for byte, and training on from it computes what training on from the
same state restored through whole-tensor IO (the .npz path) computes.  Host placement, its HBM cache and deferred Adam do not
show in the files.  A save and a restore hold about one chunk of rows in host memory, where the .npz layout holds the model.  The
G ranks are G handles in one process (`LocalShardGroup`); the entry points run the torchrun driver.
"""
import os
import re
import shutil
import subprocess
import sys
import tracemalloc
from collections import OrderedDict

import numpy as np
import pytest

from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_parity import small_conf
from tests.test_gpu_sharded_eval import _metrics
from tests.test_parallel_gloo import slice_raw
from wide_deep_b200 import checkpoint
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import T_DENSE, T_EMB_TABLE, Plan
from wide_deep_b200.sharded import LocalShardGroup

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DENSE_ROWS = 40                    # tables of more rows are row-sharded when G > 1; h2_embedding (37 rows) stays replicated
B = 96                             # global batch: G' in 1..4 ranks split it evenly
H3_ROWS = 3000                     # h3 shrunk from small_conf's 200000 rows so that chunks of a few rows stay quick
SMALL_CHUNK = 4 * 16 * 3           # 3 rows of the 16-wide h3 table, 12 of a 4-wide table, 24 of h2 (37 rows), 48 of a wide column:
                                   # every call but a table's first starts at row0 > 0 and covers a part of the table and its cache


def small_conf_h3(dnn_opt):
    fc, cross, model = small_conf(dnn_opt=dnn_opt)
    fc["h3"] = dict(fc["h3"], parameter=H3_ROWS)
    return fc, cross, model


class Ranks(object):
    """The ranks of one model: a LocalShardGroup for G > 1, one handle for G = 1."""

    def __init__(self, G, dnn_opt, seed=None, **kw):
        fc, cross, model = small_conf_h3(dnn_opt)
        self.fc, self.G, self.per = fc, G, B // G
        self.plans = [Plan(fc, cross, model, "wide_deep", max_batch=self.per, gemm_engine="ffma", max_nnz=self.per * 64,
                           max_keys=self.per * 64, dense_exchange_max_rows=DENSE_ROWS if G > 1 else 0, shard_world=G, shard_rank=r,
                           shard_slack=float(max(G, 2)), **kw) for r in range(G)]
        self.models = [WideDeepModel(p) for p in self.plans]
        if seed is not None:
            for m in self.models:
                m.init(seed)
        self.grp = LocalShardGroup(self.models) if G > 1 else None

    def step(self, raw, label):
        shards = [to_product_batch(self.plans[0], slice_raw(raw, r * self.per, (r + 1) * self.per), label[r * self.per:(r + 1) * self.per])
                  for r in range(self.G)]
        if self.grp is not None:
            return self.grp.train_step(shards)
        return self.models[0].train_step(shards[0])

    def get(self, name, slot=0):
        return self.grp.get_tensor(name, slot) if self.grp is not None else self.models[0].get_tensor(name, slot)

    def state(self):
        m0 = self.models[0]
        return OrderedDict(("%s/slot%d" % (n, s), self.get(n, s)) for n in m0.tensor_names() for s in range(m0.n_slots(n) + 1))

    def load_whole(self, state, step):
        """What restoring an .npz does: every global tensor through set_tensor, after the step count."""
        for m in self.models:
            m.global_step = step
            m.set_opt_step(step)
            for key, v in state.items():
                name, s = key.rsplit("/slot", 1)
                m.set_tensor(name, v, int(s))

    def close(self):
        for m in self.models:
            m.close()


def _assert_same(a, b, what):
    assert list(a) == list(b)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), (what, k)


def _batches(fc, n, seed):
    rng = np.random.default_rng(seed)
    return [(random_raw_batch(fc, B, rng), (rng.random(B) < 0.3).astype(np.float32)) for _ in range(n)]


@pytest.mark.parametrize("dnn_opt", ["Adagrad", "Adam"])
@pytest.mark.parametrize("G", [2, 3, 4])
def test_resharding_round_trip(tmp_path, monkeypatch, G, dnn_opt):
    monkeypatch.setattr(checkpoint, "CHUNK_BYTES", SMALL_CHUNK)
    src = Ranks(G, dnn_opt, seed=11)
    assert any(src.plans[0].is_sharded_tensor(n) for n in src.plans[0].tensor_names)
    assert any(not t["sharded"] for t in src.plans[0].tables)
    assert src.plans[0].lin_opt["kind"] == "ftrl"
    for raw, label in _batches(src.fc, 3, G):
        src.step(raw, label)
    state = src.state()
    path = src.grp.save(str(tmp_path))
    src.close()
    assert checkpoint.read_manifest(path)["world"] == G
    more = _batches(src.fc, 2, 100 + G)
    for G2 in (1, 2, 3, 4):
        dst, ref = Ranks(G2, dnn_opt), Ranks(G2, dnn_opt)
        if dst.grp is not None:
            assert dst.grp.restore(path) == 3
        else:
            assert checkpoint.restore(path, dst.models) == 3
        assert all(m.global_step == 3 for m in dst.models)
        _assert_same(dst.state(), state, "restored at G'=%d" % G2)
        ref.load_whole(state, 3)
        for raw, label in more:
            la, lb = dst.step(raw, label), ref.step(raw, label)
            assert np.float32(la).tobytes() == np.float32(lb).tobytes() and np.isfinite(la)
        _assert_same(dst.state(), ref.state(), "two steps at G'=%d" % G2)
        dst.close()
        ref.close()


def _files(path):
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


@pytest.mark.parametrize("G", [1, 2])
def test_host_placement_does_not_show_in_the_files(tmp_path, monkeypatch, G):
    """Host-placed tables behind an HBM cache with deferred Adam write the files their HBM twin writes, and read them back.  In
    chunks of a few rows: every range starts inside the table and leaves other rows of it dirty, stale or unsettled in the cache."""
    monkeypatch.setattr(checkpoint, "CHUNK_BYTES", SMALL_CHUNK)
    fc = small_conf_h3("Adam")[0]
    hbm = Ranks(G, "Adam", seed=5, host_tables=[])
    host = [t["name"] for t in hbm.plans[0].tables if (t["sharded"] if G > 1 else t["rows"] > DENSE_ROWS)]
    cache = dict(shard_cache_bytes=1 << 20) if G > 1 else dict(host_cache_bytes=1 << 20)
    hst = Ranks(G, "Adam", seed=5, host_tables=host, defer_adam=True, **cache)
    assert all(m.memory_usage()[1] > 0 for m in hst.models)
    for raw, label in _batches(fc, 5, 3):
        hbm.step(raw, label)
        hst.step(raw, label)
    a = checkpoint.save(str(tmp_path / "hbm"), hbm.models)
    b = checkpoint.save(str(tmp_path / "host"), hst.models)
    assert _files(a) == _files(b)
    assert sum(m.deferred_adam_stats()["rows"] for m in hst.models) > 0
    assert sum(m.host_cache_stats()["capacity"] for m in hst.models) > 0
    # a restore into the cached, deferred model (its cached copies of the rows go, the rows are stamped) trains on like the twin
    more = _batches(fc, 2, 4)
    hbm.step(*more[0])
    hst.step(*more[0])
    checkpoint.restore(a, hst.models)
    checkpoint.restore(a, hbm.models)
    for raw, label in more:
        assert np.float32(hst.step(raw, label)).tobytes() == np.float32(hbm.step(raw, label)).tobytes()
    _assert_same(hst.state(), hbm.state(), "trained on after a restore")
    hbm.close()
    hst.close()


def test_memory_bound_of_a_save_and_a_restore(tmp_path):
    """One 2^21 x 32 Adagrad table (256 MB of values, 256 MB of accumulators): a sharded-layout save and restore hold less than two
    chunks beside the dense tensors in traced host memory; the .npz save holds more than the table."""
    fc = OrderedDict(h=dict(type="category", transform="hash_bucket", parameter=1 << 21),
                     x=dict(type="continuous", transform=None, parameter=dict(normalization=None, boundaries=None)))
    model = dict(small_conf(hidden=(16,))[2], dnn_optimizer="Adagrad")
    plan = Plan(fc, [], model, "deep", max_batch=64, embedding_dim_override=32, gemm_engine="ffma", max_nnz=64 * 8, max_keys=64 * 8)
    m = WideDeepModel(plan).init(3)
    rows = [n for n in m.tensor_names() if plan.tensor_names[n][0] == T_EMB_TABLE]
    assert [plan.tensor_names[n][3] for n in rows] == [(1 << 21, 32)]
    table = (1 << 21) * 32 * 4
    dense = sum(m.get_tensor(n, s).nbytes for n in m.tensor_names() if n not in rows for s in range(m.n_slots(n) + 1))
    bound = 2 * checkpoint.CHUNK_BYTES + dense
    assert bound < table

    def peak(fn):
        tracemalloc.start()
        try:
            tracemalloc.reset_peak()
            out = fn()
            return out, tracemalloc.get_traced_memory()[1]
        finally:
            tracemalloc.stop()

    path, p_save = peak(lambda: checkpoint.save(str(tmp_path / "s"), [m]))
    want = {n: m.get_tensor(n, 1) for n in rows}
    m2 = WideDeepModel(plan)
    _, p_restore = peak(lambda: checkpoint.restore(path, [m2]))
    assert p_save < bound and p_restore < bound, (p_save, p_restore, bound)
    assert m2.get_tensor(rows[0], 1).tobytes() == want[rows[0]].tobytes()
    m2.close()
    # the .npz layout (WideAndDeepClassifier.save's)
    _, p_npz = peak(lambda: checkpoint.save_npz(str(tmp_path / "n"), m))
    assert p_npz > table, (p_npz, table)
    m.close()


def test_row_ranges_are_checked():
    """wd_tensor_io_rows reads the rows asked for and refuses ranges outside the tensor and tensors without rows."""
    from wide_deep_b200._native import NativeError
    r = Ranks(1, "Adagrad", seed=1)
    m = r.models[0]
    emb = "dnn/input_from_feature_columns/input_layer/h3_embedding/embedding_weights"
    wide = "linear/linear_model/h3/weights"
    full = m.get_tensor(emb, 1)
    assert m.get_rows(emb, H3_ROWS - 5, 5, slot=1).tobytes() == full[-5:].tobytes()
    assert m.get_rows(wide, 7, 3).tobytes() == m.get_tensor(wide)[7:10].tobytes()
    for name, row0, n in ((emb, H3_ROWS - 4, 5), (emb, -1, 2), (wide, H3_ROWS, 1)):
        with pytest.raises(NativeError):
            m.get_rows(name, row0, n)
    with pytest.raises(NativeError):
        m.set_rows(emb, H3_ROWS - 1, np.zeros((2, full.shape[1]), dtype=np.float32))
    kind, index, sub, _ = next(v for v in m.plan.tensor_names.values() if v[0] == T_DENSE)       # no rows: refused
    out = np.zeros(4, dtype=np.float32)
    assert m._lib.wd_tensor_io_rows(m._h, kind, index, sub, 0, 0, 1, out.ctypes.data, 0) == -1
    assert m.get_tensor(emb, 1).tobytes() == full.tobytes()
    r.close()


def _run(cmd, env, cwd):
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=cwd, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_entry_points_in_both_layouts(tmp_path):
    """torchrun train.py on two ranks (one GPU) in each layout, then eval.py single-process and under torchrun: the sharded layout
    is restored at G' = 1 and 2, and every metric equals the .npz flow's."""
    env = dict(os.environ, PYTHONPATH=ROOT, WD_SHARD_SAME_GPU="1")
    py = os.path.join(ROOT, "python")
    tr = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
          "--master-port", "29683"]
    lines = [l for l in open(os.path.join(ROOT, "data", "eval", "eval1")).read().split("\n") if l]
    (tmp_path / "train.tsv").write_text("\n".join(lines[:1024]) + "\n")
    (tmp_path / "eval.tsv").write_text("\n".join(lines[1024:1024 + 513]) + "\n")
    out = {}
    for layout in ("npz", "sharded"):
        conf = tmp_path / ("conf_" + layout)
        shutil.copytree(os.path.join(ROOT, "conf"), conf)
        txt = (conf / "train.yaml").read_text()
        txt = re.sub(r"^train:[ \t]*$", "train:\n  tf_compat_pad: false", txt, count=1, flags=re.M)
        if layout == "sharded":
            txt = re.sub(r"^runconfig:[ \t]*$", "runconfig:\n  checkpoint_layout: sharded", txt, count=1, flags=re.M)
        (conf / "train.yaml").write_text(txt)
        e = dict(env, WD_CONF_DIR=str(conf))
        mdir = tmp_path / ("model_" + layout)
        _run(tr + ["train.py", "--model_dir", str(mdir), "--train_data", str(tmp_path / "train.tsv"), "--train_epochs", "1",
                   "--batch_size", "64", "--keep_train", "0"], e, py)
        found = checkpoint.list_checkpoints(str(mdir / "wide_deep"))
        assert len(found) == 1 and os.path.isdir(found[0][1]) == (layout == "sharded"), found
        ev = ["--model_dir", str(mdir), "--test_data", str(tmp_path / "eval.tsv")]
        out[layout] = (_metrics(_run([sys.executable, "eval.py"] + ev + ["--batch_size", "128"], e, py)),
                       _metrics(_run(tr + ["eval.py"] + ev + ["--batch_size", "64"], e, py)))
    assert out["npz"] == out["sharded"], out
    assert out["npz"][0]["global_step"] == 8
