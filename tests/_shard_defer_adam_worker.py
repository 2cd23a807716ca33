"""Worker for tests/test_gpu_host_adam.py::test_sharded_deferred_host_tables_in_separate_processes (launched by
torch.distributed.run): every rank holds two row-sharded Adam models with the same parameters, one with every shard in HBM and one
with its sharded tables in page-locked host memory as deferred Adam tables, trains both through wd_shard_train_step_slot (CUDA IPC + flag barriers,
CUDA-graph replay after two eager steps) on the same batches, and compares losses, logits and its local shards byte for byte."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from oracle import model as OM
    from tests.helpers import random_raw_batch, to_product_batch
    from tests.test_gpu_parity import small_conf
    from tests.test_parallel_gloo import slice_raw
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import Plan
    from wide_deep_b200.sharded import ShardedTrainer
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    same = bool(os.environ.get("WD_SHARD_SAME_GPU"))
    dev = 0 if same else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")                    # plumbing only: the 64-byte IPC handles and the final verdict
    fc, cross, model = small_conf(hidden=(64, 32), dnn_opt="Adam")
    per = 256 // world
    B = per * world
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(5)
    rng = np.random.default_rng(79)
    for c in om.wide_cols:
        om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1

    def plan(host_tables):
        return Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * 64, max_keys=per * 64, dense_exchange_max_rows=30,
                    shard_world=world, shard_rank=rank, shard_slack=float(world), gemm_engine="ffma", host_tables=host_tables,
                    defer_adam=True)

    ref_plan = plan([])
    host = [t["name"] for t in ref_plan.tables if t["sharded"]]
    models = {"hbm": WideDeepModel(ref_plan, device=dev), "host": WideDeepModel(plan(host), device=dev)}
    for pm in models.values():
        for name in pm.tensor_names():
            pm.set_tensor(name, om.params[name])
    trainers = {k: ShardedTrainer(pm) for k, pm in models.items()}
    ok = models["host"].memory_usage()[1] > 0 and models["hbm"].memory_usage()[1] == 0
    lo, hi = rank * per, (rank + 1) * per
    for step in range(8):                              # steps 0-1 eager, 2 captured, 3-7 replayed (one slot)
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        batch = to_product_batch(ref_plan, slice_raw(raw, lo, hi), label[lo:hi])
        losses = {k: np.float32(t.step(batch)) for k, t in trainers.items()}
        if losses["host"].tobytes() != losses["hbm"].tobytes():
            print("LOSS MISMATCH rank", rank, "step", step, losses, flush=True)
            ok = False
    raw = random_raw_batch(fc, B, rng)
    batch = to_product_batch(ref_plan, slice_raw(raw, lo, hi), np.zeros(per, dtype=np.float32))
    logits = {k: t.forward(batch)[0] for k, t in trainers.items()}
    if logits["host"].tobytes() != logits["hbm"].tobytes():
        print("LOGITS MISMATCH rank", rank, flush=True)
        ok = False
    a, b = models["hbm"], models["host"]
    for name in a.tensor_names():                      # this rank's shard of every sharded tensor, every other tensor whole
        for s in range(a.n_slots(name) + 1):
            if a.get_tensor(name, slot=s).tobytes() != b.get_tensor(name, slot=s).tobytes():
                print("MISMATCH rank", rank, name, "slot", s, flush=True)
                ok = False
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    dist.destroy_process_group()
    if rank == 0:
        print("SHARD_DEFER_OK" if flag.item() == 0 else "SHARD_DEFER_FAIL", flush=True)
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
