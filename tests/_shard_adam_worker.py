"""Worker for tests/test_gpu_multi_gpu_optimizers.py::test_multi_process_shard_driver_with_adam (launched by torch.distributed.run):
every rank trains its row shard through wd_shard_train_step_slot (CUDA IPC, flag barriers, graph replay after two eager steps) with
Adam / Adam, then RMSProp / RMSProp; rank 0 compares the gathered tensors with a single-GPU model on the whole batch and checks the
rows of the sharded h3 table that no rank touched in the last step against TensorFlow's formula (which needs the beta powers of
that step: beta^N after N steps)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(pair, rank, world, dev):
    from tests.helpers import to_product_batch
    from tests.test_gpu_multi_gpu_optimizers import (H3, STEPS, _batches, _conf, _oracle, _set_all, _single, _table_ids,
                                                     check_untouched_rows, compare_to_single)
    from tests.test_parallel_gloo import slice_raw
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import Plan
    from wide_deep_b200.sharded import ShardedTrainer
    fc, cross, model = _conf(pair)
    per = 96
    B = per * world
    rng = np.random.default_rng(77)
    om = _oracle(fc, cross, model, "wide_deep", 5, rng)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * 64, max_keys=per * 64, dense_exchange_max_rows=400,
                shard_world=world, shard_rank=rank, shard_slack=float(world), gemm_engine="ffma")
    pm = WideDeepModel(plan, device=dev)
    _set_all(lambda n, v, s: pm.set_tensor(n, v, slot=s), pm.tensor_names(), om)
    trainer = ShardedTrainer(pm)
    single = _single(fc, cross, model, "wide_deep", B, om) if rank == 0 else None
    adam = plan.dnn_opt["kind"] == "adam"
    n = STEPS + 2                                      # steps 0-1 eager, 2 captured, 3-5 replayed (one slot)
    ok = True
    for step, (raw, label) in enumerate(_batches(fc, B, rng, n)):
        if adam and step == n - 1:
            before = tuple(trainer.get_tensor(H3, slot=s) for s in range(3))
        lo, hi = rank * per, (rank + 1) * per
        loss = trainer.step(to_product_batch(plan, slice_raw(raw, lo, hi), label[lo:hi]))
        t = torch.tensor([loss], dtype=torch.float64)
        dist.all_reduce(t)
        if single is not None:
            ref = single.train_step(to_product_batch(single.plan, raw, label))
            if abs(t.item() - ref) > 1e-4 * max(abs(ref), 1.0):
                print("LOSS MISMATCH", pair, step, t.item(), ref, flush=True)
                ok = False
    names = pm.tensor_names()
    got = {(nm, s): trainer.get_tensor(nm, slot=s) for nm in names for s in range(pm.n_slots(nm) + 1)}
    if adam:
        after = tuple(got[(H3, s)] for s in range(3))
    if single is not None:
        try:
            compare_to_single(lambda nm, s: got[(nm, s)], names, pm.n_slots, single, plan)
            if adam:
                check_untouched_rows(before, after, _table_ids(single, "h3_embedding"), plan.dnn_opt, n)
        except AssertionError as e:
            print("MISMATCH", pair, e, flush=True)
            ok = False
        single.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = 0 if os.environ.get("WD_SHARD_SAME_GPU") else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")
    ok = all([run(pair, rank, world, dev) for pair in ("adam-adam", "rmsprop-rmsprop")])
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    dist.destroy_process_group()
    if rank == 0:
        print("SHARD_ADAM_OK" if flag.item() == 0 else "SHARD_ADAM_FAIL", flush=True)
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
