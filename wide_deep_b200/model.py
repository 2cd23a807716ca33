"""Python handle on a ``WdModel`` (libwd_b200) plus the host-side batch container.

``WideDeepModel`` is the thin object the estimator shim drives: it owns the native handle created from a
compiled ``Plan`` and exposes one call per C-ABI step (train_step / forward / eval), tensor IO by the
TensorFlow variable names of the reference's checkpoints, and the split backward/apply used for
data-parallel training.  All arithmetic happens in the CUDA library; numpy is only the container for host
buffers.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import _native
from ._native import BatchC, check
from .plan import Plan

METRIC_KEYS = ["accuracy", "accuracy_baseline", "auc", "auc_precision_recall", "average_loss", "label/mean", "loss",
               "precision", "prediction/mean", "recall"]


class Batch(object):
    """One batch in host memory: CSR of uint64 keys over (row, cat field) + dense matrix + labels.
    ``offsets`` may be None when every (row, field) holds exactly one key (Criteo-style)."""

    def __init__(self, batch_size, keys, offsets=None, dense=None, label=None, weight=None):
        self.batch_size = int(batch_size)
        self.keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self.offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int32)
        self.dense = None if dense is None else np.ascontiguousarray(dense, dtype=np.float32)
        self.label = None if label is None else np.ascontiguousarray(label, dtype=np.float32)
        self.weight = None if weight is None else np.ascontiguousarray(weight, dtype=np.float32)

    def h2d_bytes(self):
        n = self.keys.nbytes
        for a in (self.offsets, self.dense, self.label, self.weight):
            if a is not None:
                n += a.nbytes
        return n

    def to_c(self):
        c = BatchC()
        c.batch_size = self.batch_size
        c.cat_offsets = self.offsets.ctypes.data if self.offsets is not None else None
        c.cat_keys = self.keys.ctypes.data
        c.nnz = int(self.keys.shape[0])
        c.dense = self.dense.ctypes.data if self.dense is not None else None
        c.label = self.label.ctypes.data if self.label is not None else None
        c.weight = self.weight.ctypes.data if self.weight is not None else None
        return c

    def rows(self, lo, hi, n_fields):
        """Row slice [lo, hi) as a new Batch (used to shard a global batch over ranks)."""
        if self.offsets is None:
            keys, offs = self.keys[lo * n_fields:hi * n_fields], None
        else:
            s, e = int(self.offsets[lo * n_fields]), int(self.offsets[hi * n_fields])
            keys = self.keys[s:e]
            offs = self.offsets[lo * n_fields:hi * n_fields + 1] - s
        nd = 0 if self.dense is None else self.dense.size // max(self.batch_size, 1)
        return Batch(hi - lo, keys, offs,
                     None if self.dense is None else self.dense.reshape(self.batch_size, nd)[lo:hi],
                     None if self.label is None else self.label[lo:hi],
                     None if self.weight is None else self.weight[lo:hi])


class WideDeepModel(object):
    def __init__(self, plan: Plan, device=0):
        self.plan = plan
        self._lib = _native.lib()
        desc, self._keep = plan.to_c()
        h = ctypes.c_void_p()
        check(self._lib.wd_model_create(ctypes.byref(desc), int(device), ctypes.byref(h)))
        self._h = h
        self.device = int(device)
        self.global_step = 0
        if getattr(plan, "host_cache_bytes", 0) > 0:
            check(self._lib.wd_host_cache_enable(self._h, int(plan.host_cache_bytes)))
        if getattr(plan, "shard_cache_bytes", 0) > 0:
            check(self._lib.wd_shard_cache_enable(self._h, int(plan.shard_cache_bytes)))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.wd_model_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ parameters
    def init(self, seed=0):
        check(self._lib.wd_model_init(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF))
        return self

    def set_opt_step(self, steps):
        """Restore the optimizers' step count (Adam's beta powers) after loading a checkpoint."""
        check(self._lib.wd_set_opt_step(self._h, int(steps)))

    def tensor_names(self):
        return list(self.plan.tensor_names.keys())

    def memory_usage(self):
        """(device bytes, host bytes): HBM the model allocated, page-locked host memory of its host-placed embedding tables."""
        dev, host = ctypes.c_int64(), ctypes.c_int64()
        check(self._lib.wd_memory_usage(self._h, ctypes.byref(dev), ctypes.byref(host)))
        return dev.value, host.value

    def host_cache_stats(self, reset=False):
        """Cumulative counters of the HBM cache of host-table records (one GPU) or of this rank's host shard records (a rank of a
        row-sharded model): dict(capacity (slots), hits, loads (misses loaded into a slot), overflow (rows staged without a slot),
        evictions (dirty records written home)).  All 0 without a cache."""
        out = (ctypes.c_int64 * 5)()
        check(self._lib.wd_host_cache_stats(self._h, out, 5, 1 if reset else 0))
        return dict(zip(("capacity", "hits", "loads", "overflow", "evictions"), (int(v) for v in out)))

    def deferred_adam_stats(self, reset=False):
        """Cumulative counters of the catch-up of deferred Adam tables (Plan(defer_adam=True)): dict(rows (rows caught up),
        replayed (steps replayed), skipped (steps skipped once a row's values had stopped changing), max_gap (most steps one row
        had missed)).  All 0 without deferred tables."""
        out = (ctypes.c_int64 * 4)()
        check(self._lib.wd_deferred_adam_stats(self._h, out, 4, 1 if reset else 0))
        return dict(zip(("rows", "replayed", "skipped", "max_gap"), (int(v) for v in out)))

    def n_slots(self, name):
        o = self.plan.lin_opt if name.startswith("linear/") else self.plan.dnn_opt
        return {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[o["kind"]]

    def get_tensor(self, name, slot=0):
        """Parameter (slot 0) or optimizer slot by TensorFlow variable name.  Row-sharded tensors: this rank's rows
        (global rows rank, rank + G, ...; Plan.local_shape)."""
        kind, index, sub, _ = self.plan.tensor_names[name]
        shape = self.plan.local_shape(name)
        out = np.empty(shape, dtype=np.float32)
        check(self._lib.wd_tensor_io(self._h, kind, index, sub, slot, out.ctypes.data, out.size, 0))
        return out

    def set_tensor(self, name, value, slot=0):
        """``value`` has the GLOBAL shape; of a row-sharded tensor only this rank's rows are uploaded."""
        kind, index, sub, shape = self.plan.tensor_names[name]
        v = np.ascontiguousarray(value, dtype=np.float32).reshape(shape)
        if self.plan.is_sharded_tensor(name):
            v = np.ascontiguousarray(v[self.plan.shard_rank::self.plan.shard_world])
        check(self._lib.wd_tensor_io(self._h, kind, index, sub, slot, v.ctypes.data, v.size, 1))

    def get_rows(self, name, row0, nrows, slot=0):
        """Rows row0 .. row0 + nrows - 1 of an embedding table or wide column (this rank's local rows of a row-sharded one)."""
        kind, index, sub, shape = self.plan.tensor_names[name]
        out = np.empty((int(nrows),) + tuple(shape[1:]), dtype=np.float32)
        check(self._lib.wd_tensor_io_rows(self._h, kind, index, sub, slot, int(row0), int(nrows), out.ctypes.data, 0))
        return out

    def set_rows(self, name, row0, value, slot=0):
        """Writes ``value`` (nrows x the tensor's row shape) to local rows row0 .. row0 + nrows - 1 (get_rows' rows)."""
        kind, index, sub, shape = self.plan.tensor_names[name]
        v = np.ascontiguousarray(value, dtype=np.float32)
        if v.shape[1:] != tuple(shape[1:]):
            raise ValueError("%s: rows of shape %s, the tensor's rows have shape %s" % (name, v.shape[1:], tuple(shape[1:])))
        check(self._lib.wd_tensor_io_rows(self._h, kind, index, sub, slot, int(row0), int(v.shape[0]), v.ctypes.data, 1))

    # ------------------------------------------------------------------ steps
    def train_step(self, batch: Batch):
        """One optimizer step on a host batch; returns the sum-reduced loss (reference joint.py:404-406)."""
        c = batch.to_c()
        self._rows_hint = batch.batch_size
        loss = ctypes.c_float()
        check(self._lib.wd_train_step(self._h, ctypes.byref(c), ctypes.byref(loss)))
        self.global_step += 1
        return loss.value

    def upload(self, batch: Batch):
        c = batch.to_c()
        check(self._lib.wd_batch_upload(self._h, ctypes.byref(c)))
        self._rows_hint = batch.batch_size

    def train_step_resident(self, want_loss=True):
        loss = ctypes.c_float()
        check(self._lib.wd_train_step_resident(self._h, ctypes.byref(loss) if want_loss else None))
        self.global_step += 1
        return loss.value

    def forward(self, batch: Batch):
        """-> (logits float32[B], loss or None)"""
        c = batch.to_c()
        self._rows_hint = batch.batch_size
        logits = np.empty(batch.batch_size, dtype=np.float32)
        loss = ctypes.c_float()
        check(self._lib.wd_forward(self._h, ctypes.byref(c), logits.ctypes.data, ctypes.byref(loss)))
        return logits, (loss.value if batch.label is not None else None)

    def step_backward(self, batch: Batch | None, want_loss=True):
        loss = ctypes.c_float()
        c = batch.to_c() if batch is not None else None
        if batch is not None:
            self._rows_hint = batch.batch_size
        check(self._lib.wd_step_backward(self._h, ctypes.byref(c) if c is not None else None,
                                         ctypes.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def step_backward_slot(self, slot, want_loss=True):
        loss = ctypes.c_float()
        check(self._lib.wd_step_backward_slot(self._h, int(slot), ctypes.byref(loss) if want_loss else None))
        return loss.value if want_loss else None

    def step_apply(self):
        check(self._lib.wd_step_apply(self._h))
        self.global_step += 1

    def dense_grad(self):
        """(device pointer, float count) of the dense gradient arena after step_backward."""
        return int(self._lib.wd_dense_grad_ptr(self._h) or 0), int(self._lib.wd_dense_grad_count(self._h))

    def sparse_grads(self, which, want_count=True):
        """(rows ptr, grads ptr, n or None, width, capacity).  want_count=False does not synchronise."""
        rows, grads = ctypes.c_void_p(), ctypes.c_void_p()
        n, cap, width = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int32()
        check(self._lib.wd_sparse_grads(self._h, which, ctypes.byref(rows), ctypes.byref(grads),
                                        ctypes.byref(n) if want_count else None, ctypes.byref(width), ctypes.byref(cap)))
        return rows.value, grads.value, (n.value if want_count else None), width.value, cap.value

    def sparse_set(self, which, rows_ptr, grads_ptr, n):
        check(self._lib.wd_sparse_set(self._h, which, ctypes.c_void_p(rows_ptr), ctypes.c_void_p(grads_ptr), int(n)))

    def sparse_set_sorted(self, which, rows_ptr, grads_ptr, n_lists, list_len):
        """Merge n_lists sorted, duplicate-free, INVALID_ROW-padded lists of list_len rows (all-gathered wd_sparse_grads buffers)."""
        check(self._lib.wd_sparse_set_sorted(self._h, which, ctypes.c_void_p(rows_ptr), ctypes.c_void_p(grads_ptr), int(n_lists), int(list_len)))

    # ------------------------------------------------------------------ eval
    def eval_reset(self):
        check(self._lib.wd_eval_reset(self._h))

    def eval_accumulate(self, batch: Batch):
        c = batch.to_c()
        check(self._lib.wd_eval_accumulate(self._h, ctypes.byref(c)))

    def eval_accumulate_slot(self, slot):
        """Metrics of the batch a slot already holds (``prefetch_slot`` / ``parse_slot``)."""
        check(self._lib.wd_eval_accumulate_slot(self._h, int(slot)))

    def eval_finish(self):
        out = np.zeros(10, dtype=np.float64)
        check(self._lib.wd_eval_finish(self._h, out.ctypes.data))
        return dict(zip(METRIC_KEYS, (float(v) for v in out)))

    # ------------------------------------------------------------------ introspection
    def column_ids(self):
        """CSR (offsets int32[B*C+1], ids int64[nnz]) of the last batch, for parity tests."""
        nnz = ctypes.c_int64()
        check(self._lib.wd_debug_column_ids(self._h, None, 0, None, 0, ctypes.byref(nnz)))
        B = self._rows_hint
        offs = np.empty(B * len(self.plan.columns) + 1, dtype=np.int32)
        ids = np.empty(max(nnz.value, 1), dtype=np.int64)
        check(self._lib.wd_debug_column_ids(self._h, offs.ctypes.data, offs.size, ids.ctypes.data, ids.size, ctypes.byref(nnz)))
        return offs, ids[:nnz.value]

    def deep_input(self, batch_size):
        out = np.empty((batch_size, self.plan.d0_phys), dtype=np.float32)
        check(self._lib.wd_debug_deep_input(self._h, out.ctypes.data, out.size))
        return out

    def hidden_output(self, tower, layer, batch_size):
        """[batch_size, N_phys] output of a hidden layer after the last forward (bf16x3 layers without an fp32 copy: hi + lo)."""
        n_phys = (self.plan.out_width(self.plan.towers[tower]["hidden"][layer]) + 31) // 32 * 32
        out = np.empty(batch_size * n_phys, dtype=np.float32)
        n = self._lib.wd_debug_hidden(self._h, tower, layer, out.ctypes.data, out.size)
        if n < 0:
            check(n)
        return out[:batch_size * n].reshape(batch_size, n)

    # ------------------------------------------------------------------ layer summaries
    def summary_segments(self):
        """Keys (kind, tower, layer) of the segments layer_statistics returns (Plan.summary_segments)."""
        n = self._lib.wd_summary_segments(self._h, None, None, None, 0)
        if n < 0:
            check(n)
        k, t, l = (np.zeros(max(n, 1), dtype=np.int32) for _ in range(3))
        check(min(0, self._lib.wd_summary_segments(self._h, k.ctypes.data, t.ctypes.data, l.ctypes.data, n)))
        return [(int(k[i]), int(t[i]), int(l[i])) for i in range(n)]

    def arm_summary(self):
        """The next train step also takes the layer statistics (read them with layer_statistics after it)."""
        check(self._lib.wd_summary_arm(self._h))

    def layer_statistics(self):
        """Statistics of the last armed train step, per segment of this model's rows (summary.LayerStats)."""
        from .summary import LayerStats
        keys = self.summary_segments()
        n = len(keys)
        counts = np.zeros((n, 1551), dtype=np.int64)
        ints = np.zeros((n, 3), dtype=np.int64)
        reals = np.zeros((n, 4), dtype=np.float64)
        check(self._lib.wd_summary_read(self._h, counts.ctypes.data, ints.ctypes.data, reals.ctypes.data, n))
        return LayerStats(keys, counts, ints, reals)

    def slot_weight_sum(self, slot):
        """Sum of the example weights of the batch a slot holds (its rows when it has no weights)."""
        B, nnz, parts = ctypes.c_int32(), ctypes.c_int64(), ctypes.c_int32()
        check(self._lib.wd_debug_slot(self._h, int(slot), ctypes.byref(B), ctypes.byref(nnz), ctypes.byref(parts), None, None, None, None, None))
        if not parts.value & 4:
            return float(B.value)
        w = np.zeros(max(B.value, 1), dtype=np.float32)
        check(self._lib.wd_debug_slot(self._h, int(slot), ctypes.byref(B), ctypes.byref(nnz), ctypes.byref(parts), None, None, None, None,
                                      w.ctypes.data))
        return float(w[:B.value].astype(np.float64).sum())

    def launch_count(self):
        return int(self._lib.wd_launch_count(self._h))

    def gemm_fallback_count(self):
        """Tensor-core-engine GEMMs that ran on the FFMA kernel instead (must stay 0)."""
        return int(self._lib.wd_gemm_fallback_count(self._h))

    def graph_stats(self):
        """dict(captures, replays) of the model's step graphs since creation (a failed capture leaves the model eager, silently)."""
        out = (ctypes.c_int64 * 2)()
        check(self._lib.wd_graph_stats(self._h, out, 2))
        return dict(captures=int(out[0]), replays=int(out[1]))

    def set_profile(self, on=True):
        check(self._lib.wd_set_profile(self._h, 1 if on else 0))

    def last_timings(self):
        """OrderedDict phase -> ms of the last synchronised step ('total' first); needs set_profile(True)."""
        from collections import OrderedDict
        out = np.zeros(160, dtype=np.float32)                # PhaseTimer::kMax marks
        n = self._lib.wd_last_timings(self._h, out.ctypes.data, out.size)
        res = OrderedDict()
        for i in range(max(min(n, out.size), 0)):
            name = self._lib.wd_timing_name(self._h, i).decode()
            res[name] = res.get(name, 0.0) + float(out[i])
        return res

    def upload_slot(self, slot, batch: Batch):
        c = batch.to_c()
        check(self._lib.wd_batch_upload_slot(self._h, int(slot), ctypes.byref(c)))
        self._rows_hint = batch.batch_size

    def prefetch_slot(self, slot, batch: Batch):
        """Asynchronous refill of a batch slot on the upload stream (overlaps the step running on another slot).  The batch's
        host arrays (pinned for a truly asynchronous copy) are kept alive here until the slot is refilled again."""
        c = batch.to_c()
        check(self._lib.wd_batch_prefetch_slot(self._h, int(slot), ctypes.byref(c)))
        if not hasattr(self, "_prefetched"):
            self._prefetched = {}
        self._prefetched[int(slot)] = (batch, c)
        self._rows_hint = batch.batch_size

    def parse_slot(self, slot, tb):
        """Parse a ``TsvTextBatch`` on the GPU straight into a batch slot (wd_tsv_parse_slot): the slot then holds what
        ``prefetch_slot`` of the host-parsed batch would.  Returns when the parse is done; ``tb``'s buffers may then be reused."""
        r = tb.reader
        check(self._lib.wd_tsv_parse_slot(self._h, int(slot), ctypes.byref(r._spec), tb.text.ctypes.data, int(tb.starts[tb.n]),
                                          tb.starts.ctypes.data, tb.n))
        self._rows_hint = tb.n

    def feed_slot(self, slot, item):
        """Fill a batch slot from an input_fn item: ``parse_slot`` for a ``TsvTextBatch``, ``prefetch_slot`` for a ``Batch``."""
        from .dataset import TsvTextBatch
        if isinstance(item, TsvTextBatch):
            self.parse_slot(slot, item)
        else:
            self.prefetch_slot(slot, item)

    def tsv_parse_stats(self, reset=False):
        """dict(device = batches parse_slot parsed on the GPU, host = batches it handed to the host parser)."""
        out = (ctypes.c_int64 * 2)()
        check(self._lib.wd_tsv_parse_stats(self._h, out, 2, 1 if reset else 0))
        return dict(device=int(out[0]), host=int(out[1]))

    def slot_batch(self, slot):
        """The batch a slot holds, read back from the device (wd_debug_slot), as a ``Batch``."""
        B, nnz, parts = ctypes.c_int32(), ctypes.c_int64(), ctypes.c_int32()
        check(self._lib.wd_debug_slot(self._h, int(slot), ctypes.byref(B), ctypes.byref(nnz), ctypes.byref(parts), None, None, None, None, None))
        n, F, Nd = B.value, len(self.plan.cat_fields), len(self.plan.dense_fields)
        offs = np.zeros(n * F + 1, dtype=np.int32)
        keys = np.zeros(max(nnz.value, 1), dtype=np.uint64)
        dense = np.zeros(max(n * Nd, 1), dtype=np.float32)
        label, weight = np.zeros(n, dtype=np.float32), np.zeros(n, dtype=np.float32)
        check(self._lib.wd_debug_slot(self._h, int(slot), ctypes.byref(B), ctypes.byref(nnz), ctypes.byref(parts), offs.ctypes.data,
                                      keys.ctypes.data, dense.ctypes.data, label.ctypes.data, weight.ctypes.data))
        p = parts.value
        return Batch(n, keys[:nnz.value], offs if p & 1 else None, dense[:n * Nd].reshape(n, Nd) if Nd else None,
                     label if p & 2 else None, weight if p & 4 else None)

    def last_loss(self):
        loss = ctypes.c_float()
        check(self._lib.wd_last_loss(self._h, ctypes.byref(loss)))
        return loss.value

    def train_step_slot(self, slot, want_loss=True):
        loss = ctypes.c_float()
        check(self._lib.wd_train_step_slot(self._h, int(slot), ctypes.byref(loss) if want_loss else None))
        self.global_step += 1
        return loss.value if want_loss else None

    def stream(self):
        return int(self._lib.wd_stream(self._h) or 0)

    def stream_sparse(self, which):
        return int(self._lib.wd_stream_sparse(self._h, int(which)) or 0)

    def sync(self):
        check(self._lib.wd_sync(self._h))
