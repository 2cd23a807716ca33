"""TensorBoard summaries without a GPU: TensorFlow's histogram limits and encoding, the tag layout of every connected mode, the event
file read back through TensorBoard, and the SummarySaverHook cadence of WideAndDeepClassifier.train."""
import bisect
import glob
import struct
import sys

import numpy as np
import pytest

from tests.test_gpu_parity import small_conf
from wide_deep_b200 import summary as S
from wide_deep_b200.plan import Plan

DBL_MAX = sys.float_info.max


def tf_limits():
    """histogram.cc InitDefaultBucketsInner, transcribed."""
    buckets, neg = [], []
    v = 1.0e-12
    while v < 1.0e20:
        buckets.append(v)
        neg.append(-v)
        v *= 1.1
    buckets.append(DBL_MAX)
    neg.append(-DBL_MAX)
    return list(reversed(neg)) + [0.0] + buckets


class TfHistogram(object):
    """histogram::Histogram: Add and EncodeToProto(preserve_zero_buckets = false), transcribed value by value."""

    def __init__(self):
        self.limits = tf_limits()
        self.buckets = [0.0] * len(self.limits)
        self.min, self.max, self.num, self.sum, self.sum_squares = self.limits[-1], -DBL_MAX, 0.0, 0.0, 0.0

    def add(self, value):
        b = bisect.bisect_right(self.limits, value)
        self.buckets[b] += 1.0
        self.min = min(self.min, value)
        self.max = max(self.max, value)
        self.num += 1
        self.sum += value
        self.sum_squares += value * value

    def encode(self):
        lim, cnt = [], []
        i = 0
        while i < len(self.buckets):
            end, count = self.limits[i], self.buckets[i]
            j = i + 1
            while count == 0.0 and j < len(self.buckets) and self.buckets[j] == 0.0:
                end = self.limits[j]
                j += 1
            lim.append(end)
            cnt.append(count)
            i = j
        return lim, cnt


def test_bucket_limits_equal_tensorflow_bytes(native_lib):
    got = S.bucket_limits()
    exp = np.array(tf_limits(), dtype=np.float64)
    assert got.shape == (1551,) and got.tobytes() == exp.tobytes()
    assert got[0] == -DBL_MAX and got[-1] == DBL_MAX and got[775] == 0.0
    assert np.array_equal(got, -got[::-1])
    assert np.all(np.diff(got) > 0)


def stats_of(values_per_segment, keys):
    """LayerStats as the library defines them, computed in numpy (value v -> bucket searchsorted(limits, v, 'right'))."""
    lim = S.bucket_limits()
    n = len(keys)
    counts, ints, reals = np.zeros((n, 1551), np.int64), np.zeros((n, 3), np.int64), np.zeros((n, 4))
    for i, v in enumerate(values_per_segment):
        d = np.asarray(v, dtype=np.float32).astype(np.float64)
        fin = d[np.isfinite(d)]
        np.add.at(counts[i], np.searchsorted(lim, fin, side="right"), 1)
        ints[i] = (d.size, int(np.count_nonzero(fin == 0.0)), d.size - fin.size)
        reals[i] = (fin.min() if fin.size else DBL_MAX, fin.max() if fin.size else -DBL_MAX, fin.sum(), (fin * fin).sum())
    return S.LayerStats(keys, counts, ints, reals)


def test_histogram_encoding_matches_tensorflow_transcription(native_lib):
    lim = tf_limits()
    rng = np.random.default_rng(5)
    seg_a = np.concatenate([np.zeros(7), -np.zeros(5), np.array(lim[776:790]), -np.array(lim[770:775]),      # zeros, exact limits
                            rng.standard_normal(300) * 3, -rng.random(50) * 1e-9, [1e30, -1e25]]).astype(np.float32)
    seg_b = np.concatenate([np.full(4, 0.25), [1e-3, 7.0]]).astype(np.float32)                     # long empty runs between
    keys = [(S.SEG_HIDDEN, 0, 0), (S.SEG_DEEP_INPUT, -1, -1)]
    stats = stats_of([seg_a, seg_b], keys)
    ts = S.combine(stats, keys)
    h = TfHistogram()
    for v in np.concatenate([seg_a, seg_b]).astype(np.float64):
        h.add(float(v))
    lim_got, cnt_got = S.encode_histogram(ts.counts, S.bucket_limits())
    lim_exp, cnt_exp = h.encode()
    assert lim_got == lim_exp and cnt_got == cnt_exp
    assert (ts.min, ts.max, ts.num) == (h.min, h.max, h.num)
    assert ts.sum == pytest.approx(h.sum, rel=1e-12) and ts.sum_squares == pytest.approx(h.sum_squares, rel=1e-12)
    assert ts.zeros == 12 and ts.zero_fraction() == float(np.float32(12 / h.num))
    # a zero-valued float lands in the bucket of the first limit above 0
    assert bisect.bisect_right(lim, -0.0) == 776 == bisect.bisect_right(lim, 0.0)


def expected_tags(plan):
    """The issue-table reading of dnn.py for every tower, written out independently of Plan.summary_layout."""
    x = (S.SEG_DEEP_INPUT, -1, -1)
    out = {}
    for t, tw in enumerate(plan.towers):
        L, mode = len(tw["hidden"]), tw["mode"]
        for l in range(L):
            h = [(S.SEG_HIDDEN, t, j) for j in range(L)]
            out["dnn/dnn/dnn_%d/hiddenlayer_%d" % (t + 1, l)] = {
                "simple": [h[l]], "last_dense": [h[l]], "first_dense": [h[l], x], "dense": [x] + h[:l + 1],
                "resnet": h[:l + 1][::-1] + [x]}[mode]
        out["dnn/dnn/dnn_%d/logits" % (t + 1)] = [(S.SEG_TOWER_LOGITS, t, -1)]
    if plan.use_wide:
        out["linear/linear"] = [(S.SEG_WIDE_LOGIT, -1, -1)]
    return out


@pytest.mark.parametrize("mode", ["simple", "first_dense", "last_dense", "dense", "resnet"])
@pytest.mark.parametrize("model_type", ["wide_deep", "deep", "wide"])
def test_tag_layout(mode, model_type):
    fc, cross, model = small_conf(hidden=(48, 32, 16), mode=mode)
    plan = Plan(fc, cross, model, model_type, max_batch=64)
    layout = plan.summary_layout()
    assert dict(layout) == expected_tags(plan) and len(layout) == len(expected_tags(plan))
    segs = plan.summary_segments()
    assert all(k in segs for _, ks in layout for k in ks)
    if model_type == "wide":
        assert layout == [("linear/linear", [(S.SEG_WIDE_LOGIT, -1, -1)])]


def test_tag_layout_multi_tower_crelu():
    fc, cross, model = small_conf(hidden=(32, 16), act="crelu")
    model["dnn_hidden_units"] = [[32, 16], [24]]
    model["dnn_connected_mode"] = ["resnet", "dense"]
    plan = Plan(fc, cross, model, "wide_deep", max_batch=64)
    assert plan.out_width(32) == 64                       # crelu hands on 2u features; the segment is the whole layer
    assert dict(plan.summary_layout()) == expected_tags(plan)
    assert "dnn/dnn/dnn_2/hiddenlayer_0" in dict(plan.summary_layout())
    assert plan.summary_segments() == [(0, -1, -1), (1, 0, 0), (1, 0, 1), (2, 0, -1), (1, 1, 0), (2, 1, -1), (3, -1, -1)]


def read_events(d):
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(d, size_guidance={"scalars": 0, "histograms": 0})
    acc.Reload()
    return acc


def test_event_file_round_trip(tmp_path, native_lib):
    fc, cross, model = small_conf(hidden=(8,), mode="first_dense")
    plan = Plan(fc, cross, model, "wide_deep", max_batch=64)
    keys = plan.summary_segments()
    rng = np.random.default_rng(0)
    vals = [np.maximum(rng.standard_normal(40), 0) for _ in keys]
    stats = stats_of(vals, keys)
    ts = S.TrainSummaries.open(str(tmp_path), 10, 100, plan.summary_layout())
    ts.write_step(7, stats, 12.5, 5.0)
    ts.close()
    assert glob.glob(str(tmp_path / "events.out.tfevents.*"))
    acc = read_events(str(tmp_path))
    tags = acc.Tags()
    layout = dict(plan.summary_layout())
    assert set(tags["histograms"]) == {t + "/activation" for t in layout}
    assert set(tags["scalars"]) == {t + "/fraction_of_zero_values" for t in layout} | {"loss", "average_loss"}
    assert [(e.step, e.value) for e in acc.Scalars("loss")] == [(7, 12.5)]
    assert acc.Scalars("average_loss")[0].value == 2.5
    tag = "dnn/dnn/dnn_1/hiddenlayer_0"
    h = TfHistogram()
    for k in layout[tag]:
        for v in vals[keys.index(k)].astype(np.float32).astype(np.float64):
            h.add(float(v))
    hv = acc.Histograms(tag + "/activation")[0]
    assert hv.step == 7
    lim, cnt = h.encode()
    assert list(hv.histogram_value.bucket_limit) == lim and list(hv.histogram_value.bucket) == cnt
    assert hv.histogram_value.num == h.num and hv.histogram_value.min == h.min and hv.histogram_value.max == h.max
    frac = acc.Scalars(tag + "/fraction_of_zero_values")[0].value
    assert frac == struct.unpack("f", struct.pack("f", sum(1 for k in layout[tag] for v in vals[keys.index(k)] if v == 0) / h.num))[0]


def test_non_finite_value_raises_with_tag(tmp_path, native_lib):
    fc, cross, model = small_conf(hidden=(8,))
    plan = Plan(fc, cross, model, "deep", max_batch=64)
    keys = plan.summary_segments()
    vals = [np.ones(4) for _ in keys]
    vals[keys.index((S.SEG_HIDDEN, 0, 0))][2] = np.nan
    ts = S.TrainSummaries.open(str(tmp_path), 10, 100, plan.summary_layout(), write=False)
    with pytest.raises(ValueError, match="Nan in summary histogram for: dnn/dnn/dnn_1/hiddenlayer_0/activation"):
        ts.write_step(1, stats_of(vals, keys), 1.0, 1.0)


class FakeModel(object):
    """What WideAndDeepClassifier.train drives, with no device: records which steps were armed."""

    def __init__(self, plan):
        self.plan, self.global_step, self.armed_steps, self._armed = plan, 0, [], False

    def feed_slot(self, slot, item):
        pass

    def arm_summary(self):
        self._armed = True

    def train_step_slot(self, slot, want_loss=True):
        self.global_step += 1
        if self._armed:
            self.armed_steps.append(self.global_step)
        self._armed = False

    def last_loss(self):
        return 0.5

    def slot_weight_sum(self, slot):
        return 4.0

    def layer_statistics(self):
        keys = self.plan.summary_segments()
        return stats_of([np.ones(4) for _ in keys], keys)


@pytest.mark.parametrize("every", [1, 3, 4, None])
def test_cadence_matches_summary_saver_hook(tmp_path, every, native_lib):
    from wide_deep_b200.config import Config
    from wide_deep_b200.estimator import WideAndDeepClassifier
    class Cfg(Config):
        @property
        def runconfig(self):
            return dict(Config.runconfig.fget(self) or {}, save_summary_steps=every, log_step_count_steps=2)
    cfg = Cfg()
    est = WideAndDeepClassifier(str(tmp_path), "wide_deep", config=cfg, max_batch=16)
    fake = FakeModel(est.plan)
    est._model = fake
    est.save = lambda: None
    for n_steps in (10, 5, 1):                           # three train() calls, as dynamic_train makes one per file and epoch
        est.train(lambda n=n_steps: iter(range(n)))
    # SummarySaverHook: the first step of each call, then every `every` global steps after the last summary
    exp, step = [], 0
    for n_steps in (10, 5, 1):
        last = None
        for _ in range(n_steps):
            step += 1
            if every and (last is None or step >= last + every):
                exp.append(step)
                last = step
    assert fake.armed_steps == exp
    files = glob.glob(str(tmp_path / "events.out.tfevents.*"))
    if not every:
        assert not files                                 # no summaries: no writer opened
        return
    acc = read_events(str(tmp_path))
    assert [e.step for e in acc.Scalars("loss")] == exp
    assert [e.step for e in acc.Histograms("linear/linear/activation")] == exp
    rate, step = [], 0                                   # StepCounterHook, every 2 steps: from each call's first step on
    for n_steps in (10, 5, 1):
        last = step + 1
        rate += list(range(last + 2, step + n_steps + 1, 2))
        step += n_steps
    assert [e.step for e in acc.Scalars("global_step/sec")] == rate
