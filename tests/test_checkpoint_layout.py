"""The sharded checkpoint layout (wide_deep_b200/checkpoint.py) on numpy stand-ins for the model's tensor IO: re-sharding from any
writer count G to any reader count G', chunked reads and writes, manifest checks, and listing / rotation beside .npz checkpoints."""
import json
import os
import threading
from collections import OrderedDict

import numpy as np
import pytest

from wide_deep_b200 import checkpoint
from wide_deep_b200.plan import T_DENSE, T_EMB_TABLE, T_WIDE_BIAS, T_WIDE_COL

# name -> (kind, global shape, sharded at world G): as in the model, whether a table is sharded depends on G
SPECS = OrderedDict([
    ("linear/linear_model/C1/weights", (T_WIDE_COL, (13,), lambda G: G > 1)),
    ("linear/linear_model/bias_weights", (T_WIDE_BIAS, (1,), lambda G: False)),
    ("dnn/input_from_feature_columns/input_layer/big/embedding_weights", (T_EMB_TABLE, (23, 3), lambda G: G > 1)),
    ("dnn/input_from_feature_columns/input_layer/tiny/embedding_weights", (T_EMB_TABLE, (3, 4), lambda G: G > 1)),
    ("dnn/input_from_feature_columns/input_layer/mid/embedding_weights", (T_EMB_TABLE, (10, 2), lambda G: G in (2, 3))),
    ("dnn/input_from_feature_columns/input_layer/rep/embedding_weights", (T_EMB_TABLE, (6, 5), lambda G: False)),
    ("dnn/hiddenlayer_0/kernel", (T_DENSE, (4, 3), lambda G: False)),
])


class FakePlan(object):
    def __init__(self, world, rank, specs=SPECS):
        self.shard_world, self.shard_rank = world, rank
        self.tensor_names = OrderedDict((n, (k, i, 0, shape)) for i, (n, (k, shape, _)) in enumerate(specs.items()))
        self._sharded = {n: bool(f(world)) for n, (_, _, f) in specs.items()}

    def is_sharded_tensor(self, name):
        return self.shard_world > 1 and self._sharded[name]

    def local_shape(self, name):
        shape = tuple(self.tensor_names[name][3])
        if not self.is_sharded_tensor(name):
            return shape
        return ((shape[0] - self.shard_rank + self.shard_world - 1) // self.shard_world,) + shape[1:]


class FakeRank(object):
    """One rank's tensors in numpy, with WideDeepModel's tensor IO calls; counts the row calls and their sizes."""

    def __init__(self, world, rank, full=None, slots=None, specs=SPECS):
        self.plan = FakePlan(world, rank, specs)
        self.global_step, self.opt_step = 0, None
        self.slots = slots or (lambda name: 2 if name.startswith("linear/") else 1)
        self.t = {}
        self.row_calls = []
        for name in self.plan.tensor_names:
            for s in range(1 + self.n_slots(name)):
                self.t[name, s] = np.zeros(self.plan.local_shape(name), dtype=np.float32)
                if full is not None:
                    self.set_tensor(name, full[name, s], s)

    def n_slots(self, name):
        return self.slots(name)

    def tensor_names(self):
        return list(self.plan.tensor_names)

    def set_opt_step(self, step):
        self.opt_step = step

    def get_tensor(self, name, slot=0):
        return self.t[name, slot].copy()

    def set_tensor(self, name, value, slot=0):
        v = np.asarray(value, dtype=np.float32)
        if self.plan.is_sharded_tensor(name):
            v = v[self.plan.shard_rank::self.plan.shard_world]
        self.t[name, slot][...] = v

    def _rows(self, name, row0, n):
        assert self.plan.tensor_names[name][0] in (T_EMB_TABLE, T_WIDE_COL), name
        assert 0 <= row0 and n > 0 and row0 + n <= self.t[name, 0].shape[0], (name, row0, n)
        self.row_calls.append((name, n))

    def get_rows(self, name, row0, nrows, slot=0):
        self._rows(name, row0, nrows)
        return self.t[name, slot][row0:row0 + nrows].copy()

    def set_rows(self, name, row0, value, slot=0):
        self._rows(name, row0, len(value))
        self.t[name, slot][row0:row0 + len(value)] = value


def full_state(seed=0):
    rng = np.random.default_rng(seed)
    fake = FakeRank(1, 0)
    return {k: rng.standard_normal(v.shape).astype(np.float32) for k, v in fake.t.items()}


def save_threads(tmp_path, ranks):
    """Every rank saves from its own thread, meeting at one barrier, as the ranks of a torchrun job do."""
    bar = threading.Barrier(len(ranks))
    out, errs = [None] * len(ranks), []

    def run(i):
        try:
            out[i] = checkpoint.save(str(tmp_path), [ranks[i]], barrier=bar.wait)
        except BaseException as e:                # pragma: no cover (reported below)
            errs.append(e)
            bar.abort()
    th = [threading.Thread(target=run, args=(i,)) for i in range(len(ranks))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    assert all(p is None for p in out[1:])
    return out[0]


def check_ranks(ranks, full):
    for m in ranks:
        G, r = m.plan.shard_world, m.plan.shard_rank
        for (name, s), want in full.items():
            exp = want[r::G] if m.plan.is_sharded_tensor(name) else want
            np.testing.assert_array_equal(m.t[name, s], exp, err_msg="%s slot %d rank %d of %d" % (name, s, r, G))


@pytest.mark.parametrize("G", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("G2", [1, 2, 3, 4, 5])
def test_round_trip_any_world(tmp_path, monkeypatch, G, G2):
    monkeypatch.setattr(checkpoint, "CHUNK_BYTES", 3 * 4 * 2)        # two rows of the widest table per chunk
    full = full_state(G * 10 + G2)
    src = [FakeRank(G, r, full) for r in range(G)]
    for m in src:
        m.global_step = 37
    path = save_threads(tmp_path, src)
    assert path == str(tmp_path / "model.ckpt-37")
    man = checkpoint.read_manifest(path)
    assert man["world"] == G and man["global_step"] == 37
    dst = [FakeRank(G2, r) for r in range(G2)]
    assert checkpoint.restore(path, dst) == 37
    assert all(m.global_step == 37 and m.opt_step == 37 for m in dst)
    check_ranks(dst, full)


def test_one_process_holds_every_rank(tmp_path):
    """LocalShardGroup's call: all G ranks in one save, no barrier."""
    full = full_state(7)
    src = [FakeRank(3, r, full) for r in range(3)]
    path = checkpoint.save(str(tmp_path), src)
    files = sorted(os.listdir(path))
    name = "dnn/input_from_feature_columns/input_layer/big/embedding_weights"
    parts = [f for f in files if ".big." in f]
    assert len(parts) == 3 * 2 and all("-of-3" in f for f in parts)       # value and Adagrad slot, one part per rank
    assert len([f for f in files if ".rep." in f]) == 2                    # replicated: written once
    np.testing.assert_array_equal(np.load(os.path.join(path, parts[0])), full[name, 0][0::3])
    dst = [FakeRank(2, r) for r in range(2)]
    checkpoint.restore(path, dst)
    check_ranks(dst, full)


def test_chunks_bound_every_row_call(tmp_path, monkeypatch):
    monkeypatch.setattr(checkpoint, "CHUNK_BYTES", 4 * 4 * 3)          # 3 rows of 4 floats, 4 of 3, 12 of a wide column
    full = full_state(3)
    src = [FakeRank(2, r, full) for r in range(2)]
    path = checkpoint.save(str(tmp_path), src)
    dst = [FakeRank(1, 0)]
    checkpoint.restore(path, dst)
    check_ranks(dst, full)
    for m in src + dst:
        for name, n in m.row_calls:
            width = int(np.prod(SPECS[name][1][1:], dtype=np.int64))
            assert n * width * 4 <= checkpoint.CHUNK_BYTES, (name, n)
    big = "dnn/input_from_feature_columns/input_layer/big/embedding_weights"
    assert sum(1 for name, _ in dst[0].row_calls if name == big) == 2 * 6            # 23 rows in chunks of 4, two slots
    assert sum(1 for name, _ in src[0].row_calls if name == big) == 2 * 3            # 12 local rows


def _saved(tmp_path, G=2, step=5):
    src = [FakeRank(G, r, full_state(1)) for r in range(G)]
    for m in src:
        m.global_step = step
    return checkpoint.save(str(tmp_path), src)


def _edit_manifest(path, fn):
    p = os.path.join(path, checkpoint.MANIFEST)
    man = json.load(open(p))
    fn(man)
    json.dump(man, open(p, "w"))


def test_manifest_errors_raise_value_error(tmp_path):
    path = _saved(tmp_path)
    big = "dnn/input_from_feature_columns/input_layer/big/embedding_weights"
    # tensors the model needs: missing, wrong shape, too few optimizer slots
    specs = OrderedDict(SPECS)
    specs["dnn/hiddenlayer_1/kernel"] = (T_DENSE, (3, 1), lambda G: False)
    with pytest.raises(ValueError, match="missing 2 of"):
        checkpoint.restore(path, [FakeRank(1, 0, specs=specs)])
    specs = OrderedDict(SPECS)
    specs[big] = (T_EMB_TABLE, (24, 3), lambda G: G > 1)
    with pytest.raises(ValueError, match="has shape"):
        checkpoint.restore(path, [FakeRank(1, 0, specs=specs)])
    with pytest.raises(ValueError, match="missing .* e.g. .*slot2"):
        checkpoint.restore(path, [FakeRank(1, 0, slots=lambda name: 2)])
    # a part that does not hold the rows the manifest says
    part = os.path.join(path, checkpoint.read_manifest(path)["tensors"][big]["files"][0][1])
    good = np.load(part)
    np.save(part, good[:-1])
    with pytest.raises(ValueError, match="part"):
        checkpoint.restore(path, [FakeRank(1, 0)])
    np.save(part, good)
    checkpoint.restore(path, [FakeRank(1, 0)])
    # malformed manifests
    for edit in (lambda m: m.update(format="other"), lambda m: m.update(world=0), lambda m: m.pop("global_step"),
                 lambda m: m["tensors"][big].update(files=m["tensors"][big]["files"][:1]),
                 lambda m: m["tensors"][big]["files"][0].pop(),
                 lambda m: m["tensors"][big]["files"][0].__setitem__(0, "../x.npy"),
                 lambda m: m["tensors"]["dnn/hiddenlayer_0/kernel"].update(sharded=True,
                                                                          files=[["a.npy", "b.npy"], ["c.npy", "d.npy"]])):
        path = _saved(tmp_path / str(id(edit)))
        _edit_manifest(path, edit)
        with pytest.raises(ValueError):
            checkpoint.restore(path, [FakeRank(1, 0)])
    with open(os.path.join(path, checkpoint.MANIFEST), "w") as fh:
        fh.write("{")
    with pytest.raises(ValueError, match="manifest"):
        checkpoint.restore(path, [FakeRank(1, 0)])
    os.remove(os.path.join(path, checkpoint.MANIFEST))
    with pytest.raises(ValueError, match="manifest"):
        checkpoint.restore(path, [FakeRank(1, 0)])


def test_incomplete_directories_are_ignored(tmp_path):
    d = str(tmp_path)
    _saved(tmp_path, step=5)
    os.makedirs(os.path.join(d, "model.ckpt-9.tmp"))                       # a save in progress (or crashed)
    open(os.path.join(d, "model.ckpt-9.tmp", checkpoint.MANIFEST), "w").write("{}")
    os.makedirs(os.path.join(d, "model.ckpt-8"))                           # no manifest
    open(os.path.join(d, "model.ckpt-7.npz.tmp.123"), "wb").close()
    assert checkpoint.list_checkpoints(d) == [(5, os.path.join(d, "model.ckpt-5"))]
    assert checkpoint.list_checkpoints(os.path.join(d, "absent")) == []


def test_a_crashed_save_of_the_same_step_leaves_no_stray_part(tmp_path):
    tmp = tmp_path / "model.ckpt-5.tmp"
    tmp.mkdir()
    (tmp / "0002.stale.slot0.part3-of-4.npy").write_bytes(b"x")
    path = _saved(tmp_path, step=5)
    assert not os.path.exists(str(tmp)) and "0002.stale.slot0.part3-of-4.npy" not in os.listdir(path)
    path = _saved(tmp_path, G=3, step=5)                                   # the same step saved again replaces it
    assert checkpoint.read_manifest(path)["world"] == 3


def test_rotation_over_both_layouts_keeps_the_newest_steps(tmp_path):
    d = str(tmp_path)
    for step in (3, 10, 30):
        np.savez(os.path.join(d, "model.ckpt-%d.npz" % step), global_step=np.asarray(step))
    for step in (7, 20, 40):
        _saved(tmp_path, step=step)
    os.makedirs(os.path.join(d, "model.ckpt-1"))                           # incomplete: not a checkpoint, left alone
    assert [s for s, _ in checkpoint.list_checkpoints(d)] == [3, 7, 10, 20, 30, 40]
    checkpoint.rotate(d, 3)
    assert checkpoint.list_checkpoints(d) == [(20, os.path.join(d, "model.ckpt-20")), (30, os.path.join(d, "model.ckpt-30.npz")),
                                              (40, os.path.join(d, "model.ckpt-40"))]
    assert sorted(os.listdir(d)) == ["model.ckpt-1", "model.ckpt-20", "model.ckpt-30.npz", "model.ckpt-40"]


def test_npz_layout_round_trip(tmp_path):
    full = full_state(9)
    src = FakeRank(1, 0, full)
    src.global_step = 12
    path = checkpoint.save_npz(str(tmp_path), src)
    assert path == str(tmp_path / "model.ckpt-12.npz") and checkpoint.list_checkpoints(str(tmp_path)) == [(12, path)]
    assert checkpoint.save_npz(str(tmp_path / "other"), src, write=False) is None and not os.path.exists(str(tmp_path / "other"))
    dst = [FakeRank(2, r) for r in range(2)]
    for m in dst:
        checkpoint.restore_npz(path, m)
    assert all(m.global_step == 12 and m.opt_step == 12 for m in dst)
    check_ranks(dst, full)
    with pytest.raises(ValueError, match="missing"):
        checkpoint.restore_npz(path, FakeRank(1, 0, slots=lambda name: 2))


def test_estimator_does_not_repeat_a_sharded_save_at_the_same_step(tmp_path, monkeypatch):
    """A second save() with no step in between (train() on input without a batch) writes nothing; a restore forgets the save."""
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import WideAndDeepClassifier
    est = WideAndDeepClassifier(str(tmp_path), "wide_deep", config=Config(), max_batch=64, checkpoint_layout="sharded")
    est._model = FakeRank(1, 0, full_state(2))
    calls = []
    real = checkpoint.save
    monkeypatch.setattr(checkpoint, "save", lambda *a, **k: calls.append(a) or real(*a, **k))
    est._model.global_step = 4
    path = est.save()
    assert est.save() == path and len(calls) == 1
    est._model.global_step = 5
    est.save()
    est.restore(path)
    assert est._model.global_step == 4
    est.save()
    assert len(calls) == 3 and [s for s, _ in checkpoint.list_checkpoints(str(tmp_path))] == [4, 5]
    with pytest.raises(ValueError, match="checkpoint_layout"):
        WideAndDeepClassifier(str(tmp_path), "wide_deep", config=Config(), max_batch=64, checkpoint_layout="zip")
