"""Training with ROW-SHARDED tables over the GPUs of one box.

The reference's distributed mode partitions large variables over parameter-server tasks (``min_max_variable_partitioner``,
reference python/lib/joint.py:141-143) and trains asynchronously (python/train.py:197-217, per-worker input shard
python/lib/dataset.py:173-174).  Here every embedding table / wide column larger than ``dense_exchange_max_rows`` is split by
row over the G ranks (row r lives on rank r mod G); the batch is split by example; one synchronous step computes EXACTLY what a
single GPU computes on the concatenated batch.  All traffic moves through peer memory inside the library's own kernels
(wide_deep_b200/csrc/shard.cu) — torch.distributed is used once, to all-gather the 64-byte CUDA IPC handles.

  ``ShardedTrainer``    one process per GPU (torchrun): ``step_slot`` is a collective call.
  ``LocalShardGroup``   G model handles in ONE process (any number of GPUs, also one): the phases of a step are ordered with
                        events instead of flag barriers.  This is what the single-GPU parity tests drive.

Evaluation: every rank adds the metrics of its own rows to its accumulator on the device, and one collective sums the
accumulators of all ranks in rank order (``eval_finish`` / ``evaluate``): the same ten values on every rank.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import _native, checkpoint
from ._native import check
from .model import METRIC_KEYS

N_PHASES = 5


class LocalShardGroup(object):
    def __init__(self, models):
        self.models = list(models)
        self.G = len(self.models)
        self._lib = _native.lib()
        self._arr = (ctypes.c_void_p * self.G)(*[m._h for m in self.models])
        check(self._lib.wd_shard_connect_local(self._arr, self.G))

    def _sync(self):
        check(self._lib.wd_shard_local_sync(self._arr, self.G))

    def _run(self, slot, train):
        for phase in range(N_PHASES if train else 3):
            for m in self.models:
                check(self._lib.wd_shard_phase(m._h, int(slot), phase, 1 if train else 0))
            self._sync()

    def train_step(self, batches=None, slot=0):
        """One synchronous step; ``batches[r]`` (optional) is uploaded to rank r's slot first.  Returns the global loss
        (sum over ranks: the loss is a sum over examples, reference joint.py:404-406)."""
        if batches is not None:
            for m, b in zip(self.models, batches):
                m.upload_slot(slot, b)
        self._run(slot, True)
        total = 0.0
        for m in self.models:
            loss = ctypes.c_float()
            check(self._lib.wd_shard_finish(m._h, ctypes.byref(loss), None))
            m.global_step += 1
            total += loss.value
        return total

    def forward(self, batches, slot=0):
        """-> list of logits arrays, one per rank."""
        for m, b in zip(self.models, batches):
            m.upload_slot(slot, b)
        self._run(slot, False)
        out = []
        for m, b in zip(self.models, batches):
            logits = np.empty(b.batch_size, dtype=np.float32)
            loss = ctypes.c_float()
            check(self._lib.wd_shard_finish(m._h, ctypes.byref(loss), logits.ctypes.data))
            out.append(logits)
        return out

    def evaluate(self, batches_per_rank, n_valid_per_rank, slot=0):
        """Metrics of the first ``n_valid_per_rank[r][s]`` rows of ``batches_per_rank[r][s]`` over every rank r and step s, from
        one collective reduction -> list of one metric dict per rank (identical).  Every rank runs every step: a rank without
        rows left passes any one-row batch with n_valid 0."""
        steps = len(batches_per_rank[0])
        for m in self.models:
            m.eval_reset()
        for s in range(steps):
            for m, bs in zip(self.models, batches_per_rank):
                m.upload_slot(slot, bs[s])
            self._run(slot, False)
            for m, nv in zip(self.models, n_valid_per_rank):
                check(self._lib.wd_shard_eval_accumulate_phase(m._h, int(nv[s])))
        self._sync()
        out = []
        for m in self.models:
            v = np.zeros(10, dtype=np.float64)
            check(self._lib.wd_shard_eval_finish(m._h, v.ctypes.data))
            out.append(dict(zip(METRIC_KEYS, (float(x) for x in v))))
        return out

    def arm_summary(self):
        """The next step takes the layer statistics on every rank."""
        for m in self.models:
            m.arm_summary()

    def layer_statistics(self):
        """Layer statistics of the last armed step over the global batch (every rank's rows)."""
        from .summary import LayerStats
        return LayerStats.merge_ranks([m.layer_statistics() for m in self.models])

    def host_cache_stats(self, reset=False):
        """Per rank, the counters of its cache of host shard records (WideDeepModel.host_cache_stats)."""
        return [m.host_cache_stats(reset) for m in self.models]

    def deferred_adam_stats(self, reset=False):
        """Per rank, the catch-up counters of its deferred Adam shards (WideDeepModel.deferred_adam_stats)."""
        return [m.deferred_adam_stats(reset) for m in self.models]

    def get_tensor(self, name, slot=0):
        """Global tensor: row-sharded tensors are interleaved back from the ranks' shards."""
        plan = self.models[0].plan
        if not plan.is_sharded_tensor(name):
            return self.models[0].get_tensor(name, slot)
        shape = tuple(plan.tensor_names[name][3])
        full = np.empty(shape, dtype=np.float32)
        for r, m in enumerate(self.models):
            full[r::self.G] = m.get_tensor(name, slot)
        return full

    def set_tensor(self, name, value, slot=0):
        for m in self.models:
            m.set_tensor(name, value, slot)

    def save(self, model_dir):
        """Sharded-layout checkpoint of every rank (wide_deep_b200/checkpoint.py) -> its directory."""
        return checkpoint.save(model_dir, self.models)

    def restore(self, path):
        """Every rank's rows from a sharded-layout checkpoint written at any GPU count -> global step."""
        return checkpoint.restore(path, self.models)


class ShardedTrainer(object):
    """One rank of a torchrun job.  ``group``: a torch.distributed process group (default: WORLD)."""

    def __init__(self, model, group=None):
        import torch
        import torch.distributed as dist
        self.model, self.group = model, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        if model.plan.shard_world != self.world or model.plan.shard_rank != self.rank:
            raise ValueError("plan was compiled for rank %d of %d, this process is rank %d of %d" % (
                model.plan.shard_rank, model.plan.shard_world, self.rank, self.world))
        self._lib = _native.lib()
        mine = np.zeros(64, dtype=np.uint8)
        check(self._lib.wd_shard_ipc_handle(model._h, mine.ctypes.data))
        dev = torch.device("cuda", model.device) if dist.get_backend(group) == "nccl" else torch.device("cpu")
        t = torch.from_numpy(mine).to(dev)
        parts = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(parts, t, group=group)
        self._handles = np.ascontiguousarray(torch.stack(parts).cpu().numpy())
        check(self._lib.wd_shard_connect_ipc(model._h, self._handles.ctypes.data, self.world))
        dist.barrier(group=group)                              # every rank has mapped every segment before anyone steps

    def step_slot(self, slot, want_loss=True):
        loss = ctypes.c_float()
        check(self._lib.wd_shard_train_step_slot(self.model._h, int(slot), ctypes.byref(loss) if want_loss else None))
        self.model.global_step += 1
        return loss.value if want_loss else None

    def step(self, batch, want_loss=True, slot=0):
        self.model.upload_slot(slot, batch)
        return self.step_slot(slot, want_loss)

    def forward(self, batch, slot=0):
        self.model.upload_slot(slot, batch)
        return self.forward_slot(slot, batch.batch_size)

    def forward_slot(self, slot, batch_size):
        """Collective forward of the batch of ``batch_size`` rows a slot holds -> (logits, loss)."""
        logits = np.empty(batch_size, dtype=np.float32)
        loss = ctypes.c_float()
        check(self._lib.wd_shard_forward_slot(self.model._h, int(slot), logits.ctypes.data, ctypes.byref(loss)))
        return logits, loss.value

    def eval_reset(self):
        self.model.eval_reset()

    def eval_accumulate_slot(self, slot, n_valid):
        """Collective: sharded forward of the slot's batch, metrics of its first ``n_valid`` rows into this rank's accumulator."""
        check(self._lib.wd_shard_eval_accumulate_slot(self.model._h, int(slot), int(n_valid)))

    def eval_finish(self):
        """Collective: metric dict of every rank's rows (the same on every rank)."""
        v = np.zeros(10, dtype=np.float64)
        check(self._lib.wd_shard_eval_finish(self.model._h, v.ctypes.data))
        return dict(zip(METRIC_KEYS, (float(x) for x in v)))

    def arm_summary(self):
        """The next step takes the layer statistics.  Every rank must arm the same steps (the cadence depends only on the global
        step)."""
        self.model.arm_summary()

    def layer_statistics(self):
        """Collective: layer statistics of the last armed step over the global batch, on every rank."""
        from .summary import LayerStats
        return LayerStats.merge_ranks(self.gather(self.model.layer_statistics()))

    def host_cache_stats(self, reset=False):
        """Collective: every rank's counters of its cache of host shard records, in rank order."""
        return self.gather(self.model.host_cache_stats(reset))

    def deferred_adam_stats(self, reset=False):
        """Collective: every rank's catch-up counters of its deferred Adam shards, in rank order."""
        return self.gather(self.model.deferred_adam_stats(reset))

    def gather(self, obj):
        """Collective: every rank's `obj`, in rank order."""
        import torch.distributed as dist
        parts = [None] * self.world
        dist.all_gather_object(parts, obj, group=self.group)
        return parts

    def save(self, model_dir):
        """Collective: sharded-layout checkpoint (wide_deep_b200/checkpoint.py), this rank's rows written by this rank; one barrier
        on the group, then rank 0 commits it.  -> its directory on rank 0, None elsewhere."""
        import torch.distributed as dist
        return checkpoint.save(model_dir, [self.model], barrier=lambda: dist.barrier(group=self.group))

    def restore(self, path):
        """This rank's rows from a sharded-layout checkpoint written at any GPU count (no collective) -> global step."""
        return checkpoint.restore(path, [self.model])

    def get_tensor(self, name, slot=0):
        """Global tensor on every rank (row-sharded tensors are all-gathered through the host and interleaved)."""
        import torch.distributed as dist
        plan = self.model.plan
        local = self.model.get_tensor(name, slot)
        if not plan.is_sharded_tensor(name):
            return local
        parts = [None] * self.world
        dist.all_gather_object(parts, local, group=self.group)
        full = np.empty(tuple(plan.tensor_names[name][3]), dtype=np.float32)
        for r in range(self.world):
            full[r::self.world] = parts[r]
        return full
