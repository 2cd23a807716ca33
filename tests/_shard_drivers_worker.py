"""Worker for tests/test_gpu_shard_drivers.py (launched by torch.distributed.run, two processes on cuda:0): every rank runs the same
steps through both drivers of a row-sharded step — first a LocalShardGroup of both ranks in this process (wd_shard_phase segment
by segment, wd_shard_local_sync between segments), then its own rank through ShardedTrainer (wd_shard_train_step_slot: CUDA IPC,
flag barriers, graph replay after two eager steps) — and compares its rank's results byte for byte, and its kernel launches per
step, which differ only by the flag-barrier kernels of the multi-process driver."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS = 6                                  # multi-process: steps 0-1 eager, 2 captured, 3-5 replayed (one slot)
PER = 128                                  # examples per rank: h2_embedding (37 rows) gets rows of more than kChunk occurrences


def _plans(name, world):
    from tests.test_gpu_multi_gpu_optimizers import FTRL
    from tests.test_gpu_parity import small_conf
    from wide_deep_b200.plan import Plan
    if name == "wide_deep-adagrad-ftrl-host":
        model_type, (fc, cross, model), host = "wide_deep", small_conf(dnn_opt="Adagrad", lin_opt=FTRL), ["h2_embedding"]
    else:
        model_type, (fc, cross, model), host = "deep", small_conf(dnn_opt="Adam", lin_opt="Adam"), []
    plans = [Plan(fc, cross, model, model_type, max_batch=PER, max_nnz=PER * 64, max_keys=PER * 64, dense_exchange_max_rows=30,
                  shard_world=world, shard_rank=r, shard_slack=float(world), gemm_engine="ffma", host_tables=host) for r in range(world)]
    return fc, cross, model, model_type, plans


def _tensors(pm):
    return {(n, s): pm.get_tensor(n, slot=s) for n in pm.tensor_names() for s in range(pm.n_slots(n) + 1)}


def _barrier_kernels(plan, train):
    """flag barriers of one step on a rank: A, B, END; a train step adds G, R and Cw / Ce for each sharded space"""
    if not train:
        return 3
    return 5 + int(any(plan.wide_sharded)) + int(any(t["sharded"] for t in plan.tables))


def run(name, rank, world):
    from oracle import model as OM
    from tests.helpers import random_raw_batch, to_product_batch
    from tests.test_gpu_multi_gpu_optimizers import _set_all
    from tests.test_gpu_sharded_host_tables import K_CHUNK, _max_occurrences
    from tests.test_parallel_gloo import slice_raw
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.sharded import LocalShardGroup, ShardedTrainer
    fc, cross, model, model_type, plans = _plans(name, world)
    B = PER * world
    rng = np.random.default_rng(91)
    om = OM.OracleModel(fc, cross, model, model_type).init(11)
    if om.use_wide:                                   # zero-initialised wide weights carry no signal: give them some
        for c in om.wide_cols:
            om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1
    steps = []
    for _ in range(STEPS + 2):                        # train steps, then a forward and an eval batch
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        steps.append([to_product_batch(plans[0], slice_raw(raw, r * PER, (r + 1) * PER), label[r * PER:(r + 1) * PER]) for r in range(world)])
    n_valid = [PER - 7 * r for r in range(world)]
    msgs = []

    # ---- one process, both ranks
    grp = LocalShardGroup([WideDeepModel(p, device=0) for p in plans])
    _set_all(lambda n, v, s: grp.set_tensor(n, v, slot=s), grp.models[0].tensor_names(), om)
    mine = grp.models[rank]
    local_loss, local_launch = [], []
    for i in range(STEPS):
        l0 = mine.launch_count()
        grp.train_step(steps[i])
        local_launch.append(mine.launch_count() - l0)
        local_loss.append(np.float32(mine.last_loss()))
        if i == 0 and plans[0].host_tables and _max_occurrences(grp, "h2_embedding") <= K_CHUNK:
            msgs.append("no row of h2_embedding occurs more than kChunk times")
    l0 = mine.launch_count()
    local_logits = grp.forward(steps[STEPS])[rank]
    local_fwd_launch = mine.launch_count() - l0
    local_tensors = _tensors(mine)
    local_metrics = grp.evaluate([[s] for s in steps[STEPS + 1]], [[nv] for nv in n_valid])[rank]
    for m in grp.models:
        m.close()

    # ---- one process per rank
    pm = WideDeepModel(plans[rank], device=0)
    _set_all(lambda n, v, s: pm.set_tensor(n, v, slot=s), pm.tensor_names(), om)
    trainer = ShardedTrainer(pm)
    bars = _barrier_kernels(plans[rank], True)
    for i in range(STEPS):
        l0 = pm.launch_count()
        loss = np.float32(trainer.step(steps[i][rank]))
        if pm.launch_count() - l0 != local_launch[i] + bars:
            msgs.append("step %d: %d launches, one-process driver %d + %d barriers" % (i, pm.launch_count() - l0, local_launch[i], bars))
        if loss.tobytes() != local_loss[i].tobytes():
            msgs.append("step %d: loss %r vs %r" % (i, loss, local_loss[i]))
    l0 = pm.launch_count()
    logits, _ = trainer.forward(steps[STEPS][rank])
    if pm.launch_count() - l0 != local_fwd_launch + _barrier_kernels(plans[rank], False):
        msgs.append("forward: %d launches, one-process driver %d" % (pm.launch_count() - l0, local_fwd_launch))
    if logits.tobytes() != local_logits.tobytes():
        msgs.append("forward: logits differ")
    for k, v in _tensors(pm).items():
        if v.tobytes() != local_tensors[k].tobytes():
            msgs.append("%s slot %d differs" % k)
    trainer.eval_reset()
    pm.upload_slot(0, steps[STEPS + 1][rank])
    trainer.eval_accumulate_slot(0, n_valid[rank])
    metrics = trainer.eval_finish()
    if metrics.keys() != local_metrics.keys() or \
            np.float64(list(metrics.values())).tobytes() != np.float64([local_metrics[k] for k in metrics]).tobytes():
        msgs.append("eval metrics %r vs %r" % (metrics, local_metrics))
    for m in msgs:
        print("MISMATCH", name, "rank", rank, m, flush=True)
    return not msgs


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dist.init_process_group("gloo")                    # plumbing only: the 64-byte IPC handles and the final verdict
    ok = run(sys.argv[1], rank, world)
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    dist.destroy_process_group()
    if rank == 0:
        print("SHARD_DRIVERS_OK" if flag.item() == 0 else "SHARD_DRIVERS_FAIL", flush=True)
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
