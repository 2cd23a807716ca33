"""Worker for tests/test_gpu_sharded_host_cache.py::test_shard_cache_in_separate_processes (launched by torch.distributed.run).

Every rank holds two row-sharded models with the same parameters and every sharded table's shard in page-locked host memory, one
without and one with the owner's HBM cache (a small one: overflow rows and dirty evictions), trains both through
wd_shard_train_step_slot (CUDA IPC + flag barriers, CUDA-graph replay after two eager steps), evaluates both through
wd_shard_eval_accumulate_slot (graphed) and compares losses, logits, metrics and its local shards byte for byte.  Then a
checkpoint that the estimator saves from a cached sharded model must restore into an HBM-sharded model bit for bit."""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def models_phase(rank, world, dev):
    from oracle import model as OM
    from tests.helpers import random_raw_batch, to_product_batch
    from tests.test_gpu_parity import small_conf
    from tests.test_parallel_gloo import slice_raw
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import Plan
    from wide_deep_b200.sharded import ShardedTrainer
    fc, cross, model = small_conf(hidden=(64, 32))
    per = 256 // world
    B = per * world
    om = OM.OracleModel(fc, cross, model, "wide_deep").init(5)
    rng = np.random.default_rng(83)
    for c in om.wide_cols:
        om.params[om.wname(c)][:] = rng.standard_normal(c.num_buckets).astype(np.float32) * 0.1

    def plan(**kw):
        return Plan(fc, cross, model, "wide_deep", max_batch=per, max_nnz=per * 64, max_keys=per * 64, dense_exchange_max_rows=30,
                    shard_world=world, shard_rank=rank, shard_slack=float(world), gemm_engine="ffma", **kw)

    host = [t["name"] for t in plan().tables if t["sharded"]]
    p0 = plan(host_tables=host)
    stride = max(((t["dim"] + 3) // 4 * 4) * 2 for t in p0.tables if t["name"] in host)        # Adagrad: [w | acc]
    models = {"host": WideDeepModel(p0, device=dev), "cached": WideDeepModel(plan(host_tables=host, shard_cache_bytes=8 * 4 * stride * 4), device=dev)}
    for pm in models.values():
        for name in pm.tensor_names():
            pm.set_tensor(name, om.params[name])
            for s, v in enumerate(om.slots[name].values()):
                pm.set_tensor(name, v, slot=s + 1)
    trainers = {k: ShardedTrainer(pm) for k, pm in models.items()}
    ok = models["cached"].host_cache_stats()["capacity"] == 32
    lo, hi = rank * per, (rank + 1) * per
    for step in range(6):                              # steps 0-1 eager, 2 captured, 3-5 replayed (one slot)
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        batch = to_product_batch(p0, slice_raw(raw, lo, hi), label[lo:hi])
        losses = {k: np.float32(t.step(batch)) for k, t in trainers.items()}
        if losses["host"].tobytes() != losses["cached"].tobytes():
            print("LOSS MISMATCH rank", rank, "step", step, losses, flush=True)
            ok = False
    raw = random_raw_batch(fc, B, rng)
    batch = to_product_batch(p0, slice_raw(raw, lo, hi), np.zeros(per, dtype=np.float32))
    logits = {k: t.forward(batch)[0] for k, t in trainers.items()}
    if logits["host"].tobytes() != logits["cached"].tobytes():
        print("LOGITS MISMATCH rank", rank, flush=True)
        ok = False
    evals = []
    for i in range(3):                                 # slot 1, three batches: eager, captured, replayed
        raw = random_raw_batch(fc, B, rng)
        label = (rng.random(B) < 0.3).astype(np.float32)
        evals.append(to_product_batch(p0, slice_raw(raw, lo, hi), label[lo:hi]))
    metrics = {}
    for k, t in trainers.items():
        t.eval_reset()
        for b in evals:
            models[k].upload_slot(1, b)
            t.eval_accumulate_slot(1, per - 3)
        metrics[k] = t.eval_finish()
    if metrics["host"] != metrics["cached"]:
        print("METRICS MISMATCH rank", rank, metrics, flush=True)
        ok = False
    c = models["cached"].host_cache_stats()
    if not (c["hits"] > 0 and c["overflow"] > 0 and c["evictions"] > 0):
        print("CACHE NOT EXERCISED rank", rank, c, flush=True)
        ok = False
    a, b = models["host"], models["cached"]
    for name in a.tensor_names():                      # this rank's shard of every sharded tensor, every other tensor whole
        for s in range(a.n_slots(name) + 1):
            if a.get_tensor(name, slot=s).tobytes() != b.get_tensor(name, slot=s).tobytes():
                print("MISMATCH rank", rank, name, "slot", s, flush=True)
                ok = False
    for pm in models.values():
        pm.close()
    return ok


def checkpoint_phase(rank, world, dev, mdir):
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import input_fn
    from wide_deep_b200.estimator import build_custom_estimator
    from wide_deep_b200.plan import compile_plan
    cfg = Config()
    names = [t["name"] for t in compile_plan(cfg, "wide_deep", 64, shard_world=world, shard_rank=rank).tables
             if t["sharded"] and t["rows"] <= 100000]
    data = os.path.join(ROOT, "data", "test", "test2")
    est_c = build_custom_estimator(mdir, "wide_deep", config=cfg, max_batch=64, device=dev, shard_world=world, shard_rank=rank,
                                   host_tables=names, shard_cache_bytes=1 << 20)
    est_c.train(input_fn=lambda: input_fn(data, None, "train", 64, config=cfg, plan=est_c.plan, rank=rank, world=world))
    c = est_c._model.host_cache_stats()
    ok = bool(names) and c["capacity"] > 0 and c["loads"] > 0
    if not ok:
        print("NO CACHE rank", rank, names, c, flush=True)
    dist.barrier()                                     # rank 0 has written the checkpoint
    est_d = build_custom_estimator(mdir, "wide_deep", config=cfg, max_batch=64, device=dev, shard_world=world, shard_rank=rank,
                                   host_tables=[])
    md = est_d._ensure_model()                         # restores the checkpoint est_c saved
    ok &= md.memory_usage()[1] == 0
    for name in md.tensor_names():                     # collective reads: every rank compares the whole tensors
        for s in range(md.n_slots(name) + 1):
            if est_d._trainer.get_tensor(name, s).tobytes() != est_c._trainer.get_tensor(name, s).tobytes():
                print("CHECKPOINT MISMATCH rank", rank, name, "slot", s, flush=True)
                ok = False
    md.close()
    est_c._model.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    same = bool(os.environ.get("WD_SHARD_SAME_GPU"))
    dev = 0 if same else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")                    # plumbing only: the 64-byte IPC handles, tensor gathers, the verdict
    ok = models_phase(rank, world, dev)
    parts = [None] * world
    with tempfile.TemporaryDirectory() as tmp:
        dist.all_gather_object(parts, tmp)             # every rank uses rank 0's directory (rank 0 alone writes there)
        ok &= checkpoint_phase(rank, world, dev, os.path.join(parts[0], "m"))
        dist.barrier()
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    dist.destroy_process_group()
    if rank == 0:
        print("SHARD_CACHE_OK" if flag.item() == 0 else "SHARD_CACHE_FAIL", flush=True)
    sys.exit(0 if flag.item() == 0 else 1)


if __name__ == "__main__":
    main()
