"""Estimator-shaped shim: the object ``python/train.py`` / ``eval.py`` / ``pred.py`` drive.

Mirrors ``build_custom_estimator(model_dir, model_type)`` -> ``WideAndDeepClassifier`` (reference
python/lib/build_estimator.py:264-294, python/lib/joint.py:272-432): ``.train(input_fn)``, ``.evaluate(input_fn)
-> dict of the head's metric keys``, ``.predict(input_fn) -> iterator of dicts``; state lives under ``model_dir``
and every ``train`` call resumes from the latest checkpoint there (hence train.py's keep_train / rmtree logic).
The reference's eval.py / pred.py build the *canned* TF estimator whose variable names do not match what
train.py wrote (quirk Q9, pred.py:5-6); here all three entry points share this one class, so eval evaluates what
train trained.
"""
from __future__ import annotations

import json
import os
import time

import numpy as np

from . import checkpoint
from .config import Config
from .model import Batch, WideDeepModel
from .plan import compile_plan


class WideAndDeepClassifier(object):
    def __init__(self, model_dir, model_type, config=None, device=0, max_batch=None, seed=None, tf_compat_pad=None,
                 gemm_engine="auto", shard_world=1, shard_rank=0, group=None, host_tables=None,
                 host_cache_bytes=0, shard_cache_bytes=0, defer_adam=False, checkpoint_layout=None):
        if model_type not in ("wide", "deep", "wide_deep"):
            raise ValueError("Invalid model type: {}, must be one of `wide`, `deep`, `wide_deep`".format(model_type))
        self.config = config or Config()
        self.model_dir, self.model_type = model_dir, model_type
        run = self.config.runconfig or {}
        self.seed = run.get("tf_random_seed", 123) if seed is None else seed
        self.keep_checkpoint_max = run.get("keep_checkpoint_max") or 5
        # checkpoints save() writes: "npz" = one flat .npz of the whole model, written by rank 0 (the default); "sharded" = every
        # rank writes its own rows in bounded chunks (wide_deep_b200/checkpoint.py), restorable at any GPU count.  restore() reads
        # either, whichever the newest checkpoint is.
        self.checkpoint_layout = checkpoint_layout or run.get("checkpoint_layout") or "npz"
        if self.checkpoint_layout not in ("npz", "sharded"):
            raise ValueError("checkpoint_layout must be `npz` or `sharded`, got {!r}".format(self.checkpoint_layout))
        mb = max_batch or self.config.train["batch_size"]
        # quirk Q2 (SURVEY Appendix A): the reference pads multi-valued string fields with '' per batch and the padding takes
        # part in SparseCross.  The file-based entry points reproduce that by default (train.yaml key `tf_compat_pad`, default
        # true), so train.py / eval.py / pred.py produce the ids the reference produces on the same file.
        if tf_compat_pad is None:
            tf_compat_pad = bool(self.config.train.get("tf_compat_pad", True))
        self.tf_compat_pad = bool(tf_compat_pad)
        slack = 8 if self.config.train.get("multivalue") else 1
        if self.tf_compat_pad and self.config.train.get("multivalue"):
            slack *= 4                                   # '' padding multiplies the ids of crosses over multi-valued fields
        # multi-GPU (python/train.py under torchrun): rank `shard_rank` of `shard_world`; large tables are row-sharded over the
        # ranks, every rank trains on its shard of the input (wide_deep_b200/sharded.py)
        self.shard_world, self.shard_rank, self.group = int(shard_world), int(shard_rank), group
        self._trainer = None
        # embedding tables in page-locked host memory (the reference's tables live in host RAM: it trains on the CPU or on
        # parameter servers, build_estimator.py:211-214): None = only the tables that do not fit in HBM, "all" or a list of table
        # names = exactly those.  Checkpoints do not depend on the placement.  With shard_world > 1 only row-sharded tables can go
        # there (each rank keeps its own shard).  host_cache_bytes > 0 (one GPU only): HBM budget of a write-back cache of the host
        # tables' most recently used records (results do not change, PCIe traffic does).  shard_cache_bytes > 0 (shard_world > 1):
        # the same cache per rank, in front of the rank's own host-placed shards.  defer_adam: host / auto tables also with the
        # Adam dnn optimizer, whose untouched rows then catch up when they are next read (Plan(defer_adam=...)).
        self.plan = compile_plan(self.config, model_type, mb, tf_compat_pad=tf_compat_pad, gemm_engine=gemm_engine, host_tables=host_tables,
                                 host_cache_bytes=host_cache_bytes, shard_cache_bytes=shard_cache_bytes, defer_adam=defer_adam,
                                 shard_world=self.shard_world, shard_rank=self.shard_rank, shard_slack=float(max(2, self.shard_world)),
                                 max_nnz=mb * len(self.config.read_feature_conf()) * 4 * slack + mb * 64,
                                 max_keys=mb * max(1, len(self.config.read_feature_conf())) * slack)
        self._model = None
        self._saved = None                               # (global step, path) of this process's last sharded-layout save
        self.device = device

    # ------------------------------------------------------------------ checkpoints
    def latest_checkpoint(self):
        found = checkpoint.list_checkpoints(self.model_dir)
        return found[-1][1] if found else None

    def _ensure_model(self, checkpoint_path=None, need_trained=False):
        if self._model is None:
            path = checkpoint_path or self.latest_checkpoint()
            if need_trained and not path:
                # tf.estimator raises the same way: "Could not find trained model in model_dir"
                raise ValueError("Could not find trained model in model_dir: {}.".format(self.model_dir))
            self._model = WideDeepModel(self.plan, device=self.device)
            if path:
                self.restore(path)
            else:
                self._model.init(self.seed)
            if self.shard_world > 1:
                from .sharded import ShardedTrainer
                self._trainer = ShardedTrainer(self._model, self.group)
        elif checkpoint_path:
            self.restore(checkpoint_path)
        return self._model

    def save(self):
        """Checkpoint of every variable (TensorFlow variable names) + optimizer slots in self.checkpoint_layout; keeps the newest
        keep_checkpoint_max checkpoints of either layout (reference conf/train.yaml runconfig).  Multi-GPU: a collective."""
        m = self._model
        if self.checkpoint_layout == "sharded":
            # Nothing has changed since this process's last save at this step (train() on input that yields no batch still ends in
            # save()): skipping it keeps a fast rank from writing the same .tmp directory that rank 0 is still committing.
            if self._saved is not None and self._saved[0] == m.global_step:
                return self._saved[1]
            if self._trainer is not None:
                path = self._trainer.save(self.model_dir)
            else:
                path = checkpoint.save(self.model_dir, [m])
            self._saved = (m.global_step, path)
        else:
            # multi-GPU: a collective — row-sharded tensors are gathered from all ranks; rank 0 alone writes
            get = self._trainer.get_tensor if self._trainer is not None else m.get_tensor
            path = checkpoint.save_npz(self.model_dir, m, get, write=self.shard_rank == 0)
        if self.shard_rank == 0:
            checkpoint.rotate(self.model_dir, self.keep_checkpoint_max)
        return path

    def restore(self, path):
        """Either layout: a sharded-layout directory (this rank's rows only) or an .npz file."""
        self._saved = None
        if os.path.isdir(path):
            checkpoint.restore(path, [self._model])
        else:
            checkpoint.restore_npz(path, self._model)

    # ------------------------------------------------------------------ estimator API
    def train(self, input_fn, hooks=None, steps=None, max_steps=None, saving_listeners=None):
        """Runs ``input_fn()`` to exhaustion (one pass = one epoch, like Estimator.train on a one-shot iterator),
        restoring the latest checkpoint first and saving one at the end."""
        m = self._ensure_model()
        run = self.config.runconfig or {}
        log_every = run.get("log_step_count_steps") or 1000
        # checkpoint cadence of tf.estimator.RunConfig (reference conf/train.yaml:80-98): every `save_checkpoints_steps` global
        # steps, else every `save_checkpoints_secs` seconds (600 when neither is set); the step-count test is deterministic, so
        # in a multi-GPU job every rank takes the collective save() at the same step; the timer of rank 0 decides for all ranks
        ck_steps, ck_secs = run.get("save_checkpoints_steps"), run.get("save_checkpoints_secs")
        if ck_steps and ck_secs:
            raise ValueError("Can not provide both save_checkpoints_steps and save_checkpoints_secs.")      # RunConfig's message
        if not ck_steps and not ck_secs:
            ck_secs = 600
        from .summary import TrainSummaries
        # TensorBoard event file of this call (wide_deep_b200/summary.py); in a multi-GPU job every rank takes the statistics of the
        # same steps and rank 0 writes those of the global batch
        summ = TrainSummaries.open(self.model_dir, run.get("save_summary_steps"), log_every, self.plan.summary_layout(),
                                   write=self.shard_rank == 0)
        try:
            return self._train_loop(m, input_fn, steps, max_steps, log_every, ck_steps, ck_secs, summ)
        finally:
            if summ is not None:
                summ.close()

    def _train_loop(self, m, input_fn, steps, max_steps, log_every, ck_steps, ck_secs, summ):
        from .dataset import Prefetcher
        n, t0, loss = 0, time.time(), float("nan")
        last_save = time.time()
        # one batch of look-ahead, as the reference's input_fn prefetches (python/lib/dataset.py:181-184): while step i runs on the
        # GPU, batch i+1 is parsed and its host->device copy issued (wd_batch_prefetch_slot, two alternating slots); a TsvTextBatch
        # (input_fn(device_parse=True)) is parsed on the GPU into the slot instead (wd_tsv_parse_slot, beside step i)
        it = Prefetcher(input_fn(), depth=2)             # batches are parsed on a background thread, two ahead of the step
        cur = next(it, None)
        slot = 0
        if cur is not None:
            m.feed_slot(slot, cur)
        stats_of = self._trainer if self._trainer is not None else m
        while cur is not None:
            armed = summ is not None and summ.cadence.arm(m.global_step + 1)
            if armed:
                stats_of.arm_summary()
            if self._trainer is not None:
                self._trainer.step_slot(slot, want_loss=False)   # collective: every rank steps on its shard of the batch
            else:
                m.train_step_slot(slot, want_loss=False)     # enqueue step i ...
            nxt = next(it, None)                             # ... parse batch i+1 on the host while it runs ...
            if nxt is not None:
                m.feed_slot(1 - slot, nxt)                   # ... start its copy (or parse) on the upload stream ...
            loss = m.last_loss()                             # ... and only then wait for step i's loss
            n += 1
            if armed:
                self._write_summary(summ, m, stats_of, slot, loss)
            if summ is not None:
                summ.step_done(m.global_step)
            if n % log_every == 0:
                print("INFO: global_step %d: loss = %.6g (%.1f steps/sec)" % (m.global_step, loss, n / (time.time() - t0)))
            if (steps and n >= steps) or (max_steps and m.global_step >= max_steps):
                break
            if nxt is not None and self._checkpoint_due(m.global_step, ck_steps, ck_secs, last_save):
                self.save()
                last_save = time.time()
            cur, slot = nxt, 1 - slot
        print("INFO: Loss for final step: %s." % loss)
        self.save()
        return self

    def _write_summary(self, summ, m, stats_of, slot, loss):
        """Layer statistics, loss and average loss of the armed step just run (global batch in a multi-GPU job)."""
        stats = stats_of.layer_statistics()
        wsum = m.slot_weight_sum(slot)
        if self._trainer is not None:
            parts = self._trainer.gather((loss, wsum))
            loss, wsum = sum(p[0] for p in parts), sum(p[1] for p in parts)
        summ.write_step(m.global_step, stats, loss, wsum)

    def _checkpoint_due(self, global_step, ck_steps, ck_secs, last_save):
        if ck_steps:
            return global_step % int(ck_steps) == 0
        due = (time.time() - last_save) >= float(ck_secs)
        if self.shard_world > 1:                              # save() is a collective: rank 0's clock decides for everyone
            import torch
            import torch.distributed as dist
            dev = torch.device("cuda", self.device) if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
            flag = torch.tensor([1 if due else 0], dtype=torch.int32, device=dev)
            dist.broadcast(flag, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0, group=self.group)
            due = bool(int(flag.item()))
        return due

    def evaluate(self, input_fn, steps=None, hooks=None, checkpoint_path=None, name=None):
        m = self._ensure_model(checkpoint_path, need_trained=True)
        if self.shard_world > 1:
            return self._evaluate_sharded(m, input_fn, steps)
        m.eval_reset()
        n = 0
        from .dataset import TsvTextBatch
        for batch in input_fn():
            text = isinstance(batch, TsvTextBatch)          # parsed on the GPU into slot 0, where eval_accumulate uploads
            if not (batch.has_label if text else batch.label is not None):
                raise ValueError("evaluate needs labelled data (the reference's `pred`-mode test call, train.py:96-101, "
                                 "fails the same way inside TensorFlow)")
            if text:
                m.parse_slot(0, batch)
                m.eval_accumulate_slot(0)
            else:
                m.eval_accumulate(batch)
            n += 1
            if steps and n >= steps:
                break
        out = m.eval_finish()
        out["global_step"] = m.global_step
        self._write_eval(out)
        return out

    def _write_eval(self, out):
        if self.shard_rank == 0:
            from .summary import write_eval
            write_eval(self.model_dir, out)

    # ------------------------------------------------------------------ multi-GPU evaluation and prediction
    # The reference's distributed mode only trains (train.py:215-216).  Here every rank runs the collective forward of the
    # row-sharded model on its lines of the file (input_fn(..., rank, world, keep_tail=True), a ShardPass that also says how many
    # steps every rank runs): the tables are read where they live, in the GPUs that trained them.

    def _rank_pass(self, input_fn):
        data = input_fn()
        if not hasattr(data, "n_valid"):
            raise ValueError("a multi-GPU evaluate() / predict() needs this rank's lines with the file's tail kept: "
                             "input_fn(..., rank=r, world=G, keep_tail=True)")
        return data

    def _fill_slot(self, m, slot, item, n_valid):
        """Slot `slot` <- this step's batch of the rank, or a one-row placeholder once its lines have run out (n_valid 0: the
        rank still serves its peers' ids in the collective forward)."""
        from .dataset import TsvTextBatch
        if n_valid == 0:
            F, Nd = len(self.plan.cat_fields), len(self.plan.dense_fields)
            item = Batch(1, np.zeros(F, dtype=np.uint64), None, np.zeros((1, Nd), dtype=np.float32) if Nd else None,
                         np.zeros(1, dtype=np.float32))
        if isinstance(item, TsvTextBatch):
            m.parse_slot(slot, item)
        else:
            m.upload_slot(slot, item)
        return item

    def _evaluate_sharded(self, m, input_fn, steps):
        """Every rank adds the metrics of its own rows on the device; one collective sums them in rank order.  Returns the same
        dict on every rank.  "loss" is the mean over steps of the sum over the step's rows of all ranks: what one process computes
        with a batch of world x batch_size lines."""
        from .dataset import TsvTextBatch
        data = self._rank_pass(input_fn)
        n = min(data.steps, steps) if steps else data.steps
        it = iter(data)
        self._trainer.eval_reset()
        for s in range(n):
            nv = data.n_valid[s]
            batch = self._fill_slot(m, 0, next(it) if nv else None, nv)
            if nv and not (batch.has_label if isinstance(batch, TsvTextBatch) else batch.label is not None):
                raise ValueError("evaluate needs labelled data (the reference's `pred`-mode test call, train.py:96-101, "
                                 "fails the same way inside TensorFlow)")
            self._trainer.eval_accumulate_slot(0, nv)
        out = self._trainer.eval_finish()
        out["global_step"] = m.global_step
        self._write_eval(out)
        return out

    def _predict_sharded(self, m, input_fn):
        """Every rank runs the collective forward on its lines; rank 0 gathers the logits through the process group and returns
        them in file order, the other ranks None."""
        import torch.distributed as dist
        data = self._rank_pass(input_fn)
        it = iter(data)
        mine = []
        for s in range(data.steps):
            nv = data.n_valid[s]
            self._fill_slot(m, 0, next(it) if nv else None, nv)
            logits, _ = self._trainer.forward_slot(0, max(nv, 1))
            mine.append(logits[:nv])
        mine = np.concatenate(mine) if mine else np.zeros(0, dtype=np.float32)
        parts = [None] * self.shard_world if self.shard_rank == 0 else None
        dst = dist.get_global_rank(self.group, 0) if self.group is not None else 0
        dist.gather_object(mine, parts, dst=dst, group=self.group)
        if self.shard_rank != 0:
            return None
        from .dataset import interleave_ranks
        return interleave_ranks(parts)

    def predict(self, input_fn, predict_keys=None, hooks=None, checkpoint_path=None):
        """Iterator of prediction dicts in input order.  Multi-GPU: a collective, so every rank must drain it; rank 0 yields every
        line's prediction in file order, the other ranks nothing."""
        m = self._ensure_model(checkpoint_path, need_trained=True)
        if self.shard_world > 1:
            logits = self._predict_sharded(m, input_fn)
            batches = [] if logits is None else [logits]
        else:
            batches = (m.forward(batch)[0] for batch in input_fn())
        for logits in batches:
            p = 1.0 / (1.0 + np.exp(-logits.astype(np.float64)))
            for i in range(len(logits)):
                yield {"logits": np.array([logits[i]], dtype=np.float32), "logistic": np.array([p[i]], dtype=np.float32),
                       "probabilities": np.array([1 - p[i], p[i]], dtype=np.float32),
                       "class_ids": np.array([int(logits[i] > 0)]), "classes": np.array([str(int(logits[i] > 0)).encode()])}

    def get_variable_names(self):
        return self.plan.tensor_names.keys()

    def get_variable_value(self, name):
        return self._ensure_model().get_tensor(name)


def build_custom_estimator(model_dir, model_type, **kw):
    """Same signature as the reference's build_custom_estimator (build_estimator.py:264-294)."""
    return WideAndDeepClassifier(model_dir, model_type, **kw)


# eval.py / pred.py of the reference call build_estimator (the canned TF classes); here it is the same object
build_estimator = build_custom_estimator
