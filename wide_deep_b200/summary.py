"""TensorBoard summaries of training and evaluation, as the reference's Estimator writes them.

Training (``WideAndDeepClassifier.train``) writes an event file into ``model_dir``:
  - per hidden layer, tower logits and wide logit (``add_layer_summary``, reference python/lib/utils/model_util.py:15-17):
    ``<tag>/fraction_of_zero_values`` and the histogram ``<tag>/activation``, taken from the statistics the library computes on
    the GPU in the step's forward (``WideDeepModel.arm_summary`` / ``layer_statistics``, wide_deep_b200/csrc/summary.cu);
  - the head's ``loss`` and ``average_loss`` at the same steps;
  - ``global_step/sec`` every ``log_step_count_steps`` steps (StepCounterHook).
Summaries follow SummarySaverHook: the first step of every ``train()`` call, then whenever ``save_summary_steps`` steps have
passed since the last one, at the global step after the step.  ``evaluate()`` writes its metrics into ``model_dir/eval``.

The histogram is TensorFlow's ``histogram::Histogram`` with its default bucket limits, encoded as ``EncodeToProto`` with
``preserve_zero_buckets = false``.
"""
from __future__ import annotations

import os
import time

import numpy as np

from . import _native

SEG_DEEP_INPUT, SEG_HIDDEN, SEG_TOWER_LOGITS, SEG_WIDE_LOGIT = 0, 1, 2, 3     # WD_SEG_*


def bucket_limits():
    """The 1551 ascending histogram limits of TensorFlow's default buckets (computed by the library, no GPU needed)."""
    out = np.empty(1551, dtype=np.float64)
    n = _native.lib().wd_summary_limits(out.ctypes.data, out.size)
    if n != out.size:
        _native.check(n if n < 0 else _native.EINVAL)
    return out


def tower_tag(tower, layer=None):
    """Tag prefix of a tower's hidden layer (``layer`` >= 0) or of its logits (``layer`` None).  TF 1.x summary_scope: the name
    scope of joint.py's variable_scope('dnn') plus the scope add_layer_summary is given, which starts with 'dnn' again; towers
    count from 1 (dnn.py:258-269)."""
    if layer is None:
        return "dnn/dnn/dnn_%d/logits" % (tower + 1)
    return "dnn/dnn/dnn_%d/hiddenlayer_%d" % (tower + 1, layer)


LINEAR_TAG = "linear/linear"      # joint.py:195, inside variable_scope('linear')


class LayerStats(object):
    """Statistics of segments (library order, keys (kind, tower, layer)): counts [n, 1551] int64, ints [n, 3] = values, zeros,
    non-finite values, reals [n, 4] = min, max, sum, sum of squares."""

    def __init__(self, keys, counts, ints, reals):
        self.keys = [tuple(int(v) for v in k) for k in keys]
        self.counts, self.ints, self.reals = counts, ints, reals

    def index(self, key):
        return self.keys.index(tuple(key))

    @staticmethod
    def merge_ranks(parts):
        """Statistics of the global batch from each rank's: counts and ints summed, min and max combined, sums added in rank
        order."""
        first = parts[0]
        counts, ints, reals = first.counts.copy(), first.ints.copy(), first.reals.copy()
        for p in parts[1:]:
            if p.keys != first.keys:
                raise ValueError("ranks disagree on the summary segments")
            counts += p.counts
            ints += p.ints
            reals[:, 0] = np.minimum(reals[:, 0], p.reals[:, 0])
            reals[:, 1] = np.maximum(reals[:, 1], p.reals[:, 1])
            reals[:, 2:] += p.reals[:, 2:]
        return LayerStats(first.keys, counts, ints, reals)


class TagStats(object):
    """Histogram state of one tag: what Histogram holds after adding every value of its segments."""

    def __init__(self, counts, num, zeros, nonfinite, vmin, vmax, vsum, vsum_squares):
        self.counts, self.num, self.zeros, self.nonfinite = counts, int(num), int(zeros), int(nonfinite)
        self.min, self.max, self.sum, self.sum_squares = float(vmin), float(vmax), float(vsum), float(vsum_squares)

    def zero_fraction(self):
        """tf.nn.zero_fraction: zeros over values, as float32."""
        return float(np.float32(self.zeros / self.num)) if self.num else 0.0


def combine(stats: LayerStats, segments):
    """One tag's statistics from its segments (the concatenation the reference summarises): counts and counts of values add, min
    and max combine, sums add in segment order."""
    idx = [stats.index(k) for k in segments]
    counts = np.zeros(stats.counts.shape[1], dtype=np.int64)
    num = zeros = nonfinite = 0
    vmin, vmax, vsum, vsq = np.finfo(np.float64).max, -np.finfo(np.float64).max, 0.0, 0.0
    for i in idx:
        counts += stats.counts[i]
        num += int(stats.ints[i, 0]); zeros += int(stats.ints[i, 1]); nonfinite += int(stats.ints[i, 2])
        vmin, vmax = min(vmin, float(stats.reals[i, 0])), max(vmax, float(stats.reals[i, 1]))
        vsum += float(stats.reals[i, 2]); vsq += float(stats.reals[i, 3])
    return TagStats(counts, num, zeros, nonfinite, vmin, vmax, vsum, vsq)


def encode_histogram(counts, limits):
    """Histogram::EncodeToProto(preserve_zero_buckets = false): (bucket_limit, bucket) lists; a run of empty buckets becomes one
    bucket whose limit is the run's last limit."""
    out_lim, out_cnt = [], []
    n = len(counts)
    i = 0
    while i < n:
        end, c = float(limits[i]), float(counts[i])
        j = i + 1
        while c == 0.0 and j < n and counts[j] == 0:
            end = float(limits[j])
            j += 1
        out_lim.append(end)
        out_cnt.append(c)
        i = j
    return out_lim, out_cnt


class StepTimer(object):
    """SecondOrStepTimer(every_steps): triggers for the first step it sees, then once `every` steps have passed."""

    def __init__(self, every):
        self.every, self.last_step, self.last_time = int(every), None, None

    def should_trigger(self, step):
        return self.last_step is None or step >= self.last_step + self.every

    def update(self, step):
        """-> (seconds, steps) since the last trigger (None, None the first time)."""
        now = time.time()
        out = (None, None) if self.last_step is None else (now - self.last_time, step - self.last_step)
        self.last_step, self.last_time = step, now
        return out


class SummaryCadence(object):
    """SummarySaverHook's schedule over one ``train()`` call: ``arm(next_step)`` before a step (``next_step``: the global step
    after it) says whether that step takes summaries."""

    def __init__(self, save_summary_steps):
        self.timer = StepTimer(save_summary_steps)

    def arm(self, next_step):
        if self.timer.should_trigger(next_step):
            self.timer.update(next_step)
            return True
        return False


class TrainSummaries(object):
    """The event file of one ``train()`` call (None from ``open`` when summaries are off).  Only the writing rank writes."""

    def __init__(self, model_dir, save_summary_steps, log_step_count_steps, layout, write=True):
        self.model_dir, self.layout = model_dir, layout
        self.cadence = SummaryCadence(save_summary_steps)
        self.rate = StepTimer(log_step_count_steps)
        self.limits = bucket_limits()
        self.writer = None
        if write:
            from torch.utils.tensorboard import SummaryWriter
            self.writer = SummaryWriter(log_dir=model_dir)

    @staticmethod
    def open(model_dir, save_summary_steps, log_step_count_steps, layout, write=True):
        """None when save_summary_steps is empty (RunConfig(save_summary_steps=None): no summaries, no writer)."""
        if not save_summary_steps:
            return None
        return TrainSummaries(model_dir, int(save_summary_steps), int(log_step_count_steps), layout, write)

    def step_done(self, global_step):
        """StepCounterHook: global_step/sec once log_step_count_steps steps have passed."""
        if self.rate.should_trigger(global_step):
            secs, steps = self.rate.update(global_step)
            if secs is not None and secs > 0 and self.writer is not None:
                self.writer.add_scalar("global_step/sec", steps / secs, global_step)

    def write_step(self, global_step, stats: LayerStats, loss, weight_sum):
        """Layer summaries of an armed step plus the head's loss scalars.  Raises ValueError on a non-finite value, as
        SummaryHistoOp fails the step ("Nan in summary histogram for: <tag>")."""
        tags = [(tag, combine(stats, segs)) for tag, segs in self.layout]
        for tag, ts in tags:
            if ts.nonfinite:
                raise ValueError("Nan in summary histogram for: %s/activation" % tag)
        if self.writer is None:
            return
        w = self.writer
        w.add_scalar("loss", loss, global_step)
        w.add_scalar("average_loss", loss / weight_sum if weight_sum else float("nan"), global_step)
        for tag, ts in tags:
            w.add_scalar(tag + "/fraction_of_zero_values", ts.zero_fraction(), global_step)
            lim, cnt = encode_histogram(ts.counts, self.limits)
            w.add_histogram_raw(tag + "/activation", ts.min, ts.max, ts.num, ts.sum, ts.sum_squares, lim, cnt, global_step)

    def close(self):
        if self.writer is not None:
            self.writer.close()
            self.writer = None


def write_eval(model_dir, results):
    """Estimator.evaluate: every metric but global_step, as a scalar at global_step, into model_dir/eval."""
    from torch.utils.tensorboard import SummaryWriter
    step = int(results["global_step"])
    w = SummaryWriter(log_dir=os.path.join(model_dir, "eval"))
    for k, v in results.items():
        if k != "global_step":
            w.add_scalar(k, float(v), step)
    w.close()
