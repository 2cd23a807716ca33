"""Data-parallel training over the GPUs of one box (one process per GPU, torch.distributed for plumbing).

The reference trains with an asynchronous TensorFlow parameter server (reference python/lib/build_estimator.py:
172-198, python/train.py:209-217; per-worker input shard python/lib/dataset.py:173-174).  Here the batch is
row-sharded over ranks and every step is synchronous and EXACT: the G-rank result equals the 1-rank result on
the concatenated batch (up to fp32 summation order), because

  * dense gradients (MLP kernels / biases / BN affine / wide bias) are SUM-allreduced — the loss is a sum
    over the global batch (reference python/lib/joint.py:404-406), so partial gradients add;
  * sparse gradients of the replicated tables are exchanged as (row id, summed gradient) lists with one
    all-gather per table space and re-reduced by row on every rank, so each touched row still receives
    exactly one optimizer update per step ("sum duplicates, apply once", SURVEY.md A.8).

``exchange`` is backend-agnostic (NCCL on GPUs, gloo in the CPU tests): it only sees tensors.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

INVALID_ROW = -1  # 0xFFFFFFFF as int32: skipped by the merge


def shard_rows(global_rows, rank, world):
    """Contiguous row range [lo, hi) of ``rank``: the same split the reference's dataset.shard makes in
    spirit (disjoint, covering), but contiguous so a global batch concatenates back in rank order."""
    per = (global_rows + world - 1) // world
    lo = min(rank * per, global_rows)
    return lo, min(lo + per, global_rows)


def exchange_sparse(rows, grads, n, group=None):
    """All-gather variable-length (rows int32[n], grads float32[n, width]) lists.
    Returns (all_rows int32[world*maxn], all_grads float32[world*maxn, width]) where unused tail entries of
    every rank's block carry INVALID_ROW.  ``rows``/``grads`` may be longer than n (capacity buffers)."""
    world = dist.get_world_size(group)
    dev = rows.device
    cnt = torch.tensor([n], dtype=torch.int64, device=dev)
    cnts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(cnts, cnt, group=group)
    maxn = max(int(max(c.item() for c in cnts)), 1)
    width = grads.shape[1]
    r = torch.full((maxn,), INVALID_ROW, dtype=torch.int32, device=dev)
    g = torch.zeros((maxn, width), dtype=torch.float32, device=dev)
    r[:n] = rows[:n]
    g[:n] = grads[:n]
    all_r = torch.empty((world * maxn,), dtype=torch.int32, device=dev)
    all_g = torch.empty((world * maxn, width), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(all_r, r, group=group) if dev.type == "cuda" else _gather_cpu(all_r, r, group)
    dist.all_gather_into_tensor(all_g, g, group=group) if dev.type == "cuda" else _gather_cpu(all_g, g, group)
    return all_r, all_g


def _gather_cpu(out, x, group):
    world = dist.get_world_size(group)
    parts = [torch.empty_like(x) for _ in range(world)]
    dist.all_gather(parts, x, group=group)
    out.copy_(torch.cat(parts, 0))


def merge_sparse_host(all_rows, all_grads):
    """Reference (CPU) merge: unique rows + row-wise sums, skipping INVALID_ROW — what wd_sparse_set does on
    the device.  Used by the gloo tests."""
    keep = all_rows != INVALID_ROW
    rows = all_rows[keep].to(torch.int64)
    grads = all_grads[keep]
    uniq, inv = torch.unique(rows, return_inverse=True)
    out = torch.zeros((uniq.numel(), grads.shape[1]), dtype=torch.float64)
    out.index_add_(0, inv, grads.to(torch.float64))
    return uniq, out.to(torch.float32)


class _DevArray(object):
    """Zero-copy view of library-owned device memory for torch (via __cuda_array_interface__)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def wrap_device(ptr, shape, dtype, device):
    typestr = {torch.float32: "<f4", torch.int32: "<i4"}[dtype]
    return torch.as_tensor(_DevArray(ptr, shape, typestr), device=device)


class DataParallelTrainer(object):
    """Drives one WideDeepModel per rank.  ``step(batch)`` = wd_step_backward -> collectives -> wd_step_apply.

    ``fixed_rows`` = (K_emb, K_wide): static per-rank upper bounds on the number of touched rows per step (e.g.
    batch x embedding columns).  With them the exchange is fully asynchronous: the library pads its row lists with
    INVALID_ROW up to capacity, every rank all-gathers exactly K rows, and no count ever travels to the host.  Without
    them the trainer falls back to the count-based (synchronising) exchange."""

    def __init__(self, model, group=None, fixed_rows=None):
        self.model, self.group = model, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.device = torch.device("cuda", model.device)
        self.stream = torch.cuda.ExternalStream(model.stream(), device=self.device)
        ptr, n = model.dense_grad()
        self.dense_grad = wrap_device(ptr, (n,), torch.float32, self.device) if n else None
        self.lists = [w for w, on in ((0, model.plan.use_deep and len(model.plan.tables) > 0), (1, model.plan.use_wide)) if on]
        self._ext = {}
        self.fixed = None
        if fixed_rows is not None:
            self.fixed = {}
            for which in self.lists:
                rows_ptr, grads_ptr, _, width, cap = model.sparse_grads(which, want_count=False)
                K = int(min(fixed_rows[which], cap))
                self.fixed[which] = dict(
                    K=K,
                    rows=wrap_device(rows_ptr, (cap,), torch.int32, self.device)[:K],
                    grads=wrap_device(grads_ptr, (cap, width), torch.float32, self.device)[:K],
                    all_r=torch.empty((self.world * K,), dtype=torch.int32, device=self.device),
                    all_g=torch.empty((self.world * K, width), dtype=torch.float32, device=self.device))

    def profile_step(self, slot):
        """One step with CUDA-event stamps around its phases (debugging aid): returns {phase: ms}.  Phases of different lists
        overlap; every time is measured from the start of the step on the stream the phase runs on."""
        m = self.model
        ev = lambda: torch.cuda.Event(enable_timing=True)
        t0 = ev(); t0.record(self.stream)
        m.step_backward_slot(slot, want_loss=False)
        marks = {}
        e = ev(); e.record(self.stream); marks["backward(main)"] = e
        for which in sorted(self.lists):
            f = self.fixed[which]
            sptr = m.stream_sparse(which)
            st = self._ext.setdefault(sptr, torch.cuda.ExternalStream(sptr, device=self.device))
            with torch.cuda.stream(st):
                e = ev(); e.record(st); marks["list%d ready" % which] = e
                dist.all_gather_into_tensor(f["all_r"], f["rows"], group=self.group)
                dist.all_gather_into_tensor(f["all_g"], f["grads"], group=self.group)
                e = ev(); e.record(st); marks["list%d gathered" % which] = e
                m.sparse_set_sorted(which, f["all_r"].data_ptr(), f["all_g"].data_ptr(), self.world, f["K"])
                e = ev(); e.record(st); marks["list%d merged" % which] = e
        with torch.cuda.stream(self.stream):
            if self.dense_grad is not None:
                dist.all_reduce(self.dense_grad, op=dist.ReduceOp.SUM, group=self.group)
            e = ev(); e.record(self.stream); marks["dense allreduce"] = e
        m.step_apply()
        e = ev(); e.record(self.stream); marks["apply+join(main)"] = e
        m.sync()
        torch.cuda.synchronize()
        return {k: t0.elapsed_time(v) for k, v in marks.items()}

    def _collectives(self):
        m = self.model
        if self.fixed is not None:
            # asynchronous path: each list is exchanged, merged and later applied on its own side stream.  With the forward +
            # backward replayed from one CUDA graph both lists become ready together, and the collectives of one communicator
            # run in issue order: the embedding list (larger, longest merge + apply chain) goes first, the wide list second,
            # the dense all-reduce (shortest tail) last
            for which in sorted(self.lists):                             # embedding rows (0), then wide rows (1)
                f = self.fixed[which]
                sptr = m.stream_sparse(which)
                if sptr not in self._ext:
                    self._ext[sptr] = torch.cuda.ExternalStream(sptr, device=self.device)
                with torch.cuda.stream(self._ext[sptr]):
                    dist.all_gather_into_tensor(f["all_r"], f["rows"], group=self.group)
                    dist.all_gather_into_tensor(f["all_g"], f["grads"], group=self.group)
                    m.sparse_set_sorted(which, f["all_r"].data_ptr(), f["all_g"].data_ptr(), self.world, f["K"])
            with torch.cuda.stream(self.stream):
                if self.dense_grad is not None:
                    dist.all_reduce(self.dense_grad, op=dist.ReduceOp.SUM, group=self.group)
            return
        with torch.cuda.stream(self.stream):
            if self.dense_grad is not None:
                dist.all_reduce(self.dense_grad, op=dist.ReduceOp.SUM, group=self.group)
            for which in self.lists:
                rows_ptr, grads_ptr, n, width, cap = m.sparse_grads(which)
                rows = wrap_device(rows_ptr, (cap,), torch.int32, self.device)
                grads = wrap_device(grads_ptr, (cap, width), torch.float32, self.device)
                all_r, all_g = exchange_sparse(rows, grads, n, self.group)
                self.stream.synchronize()
                m.sparse_set(which, all_r.data_ptr(), all_g.data_ptr(), all_r.numel())
                self._keep = (all_r, all_g)        # alive until the apply kernels have run
                m.sync()

    def step(self, batch, want_loss=True):
        loss = self.model.step_backward(batch, want_loss=want_loss and self.fixed is None)
        self._collectives()
        self.model.step_apply()
        return loss

    def step_slot(self, slot, want_loss=True):
        m = self.model
        loss = m.step_backward_slot(slot, want_loss=want_loss and self.fixed is None)
        self._collectives()
        m.step_apply()
        return loss
