"""Evaluation rate of a row-sharded model on the GPUs that hold it, against one process evaluating the same model shape alone.

Run under torch.distributed.run, one process per GPU (or, with --same-gpu, the processes share cuda:0):

    python -m torch.distributed.run --nproc-per-node 2 tools/sharded_eval_bench.py [--same-gpu] [--steps 30] [--out FILE]

Workload: the Criteo shape of wide_deep_b200/synthetic.py, sharded as bench.py --gpus N shards it (tables larger than
bench.DENSE_EXCHANGE_ROWS rows row-sharded, bf16x3 towers, 8192 examples per rank and step).
  * sharded: every rank runs wd_shard_eval_accumulate_slot on a ring of resident batches (graphs captured during the warm-up),
    then the collective wd_shard_eval_finish; a window is timed from a barrier to the finish on the slowest rank.
  * single: rank 0 alone, after the sharded models are freed, evaluates one model of the same shape with a batch of N x 8192
    examples through wd_eval_accumulate_slot, with its tables placed automatically ("auto": host memory only for what does not fit
    in HBM) and with every table above 16384 rows in page-locked host memory ("host", what a model too large for one GPU needs).
Both start from the same init seed; a sharded model draws its shards from per-rank streams, so the parameters differ, which the
rates do not depend on (tests/test_gpu_sharded_eval.py checks the results).  Rates are examples/s over all ranks, best of two
windows.  Rank 0 prints one JSON line with the GPU name, power limit and max SM clock.  With --same-gpu the processes time-slice
one GPU: the sharded rate is then not a multi-GPU rate.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.host_tables_bench import gpu_info    # noqa: E402

RING = 8
SEED = 0x5EED0007


def plans(wl, B, world, rank, host_tables):
    import bench
    from wide_deep_b200.plan import Plan
    return Plan(wl.fc, wl.cross, wl.model, wl.model_type, max_batch=B, embedding_dim_override=wl.emb, gemm_engine="bf16x3",
                max_keys=B * wl.keys_per_row, max_nnz=B * wl.ids_per_row, dense_exchange_max_rows=bench.DENSE_EXCHANGE_ROWS,
                shard_world=world, shard_rank=rank, shard_slack=1.5, host_tables=host_tables)


def timed(run_window, sync, reduce_max):
    best = None
    for _ in range(2):
        sync()
        t0 = time.perf_counter()
        run_window()
        sync()
        dt = reduce_max(time.perf_counter() - t0)
        best = dt if best is None else min(best, dt)
    return best


def sharded_rate(wl, B, steps, dev, world, rank):
    import torch
    import torch.distributed as dist
    from wide_deep_b200.model import Batch, WideDeepModel
    from wide_deep_b200.sharded import ShardedTrainer
    m = WideDeepModel(plans(wl, B, world, rank, []), device=dev)
    m.init(seed=SEED)
    t = ShardedTrainer(m)
    for s in range(RING):
        keys, offs, dense, label = wl.arrays(B, 1000 * rank + s)
        m.upload_slot(s, Batch(B, keys, offs, dense, label))
    t.eval_reset()
    for i in range(3 * RING):                       # two eager calls and the capture per slot
        t.eval_accumulate_slot(i % RING, B)
    t.eval_finish()

    def window():
        t.eval_reset()
        for i in range(steps):
            t.eval_accumulate_slot(i % RING, B)
        window.result = t.eval_finish()

    def reduce_max(x):
        v = torch.tensor([x], dtype=torch.float64)
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        return v.item()

    dt = timed(window, lambda: (m.sync(), dist.barrier()), reduce_max)
    results = [None] * world
    dist.all_gather_object(results, window.result)
    hbm = m.memory_usage()[0]
    m.close()
    return B * world * steps / dt, dt, all(r == results[0] for r in results), hbm


def single_rate(wl, GB, steps, host_tables):
    from wide_deep_b200.model import Batch, WideDeepModel
    from wide_deep_b200.plan import Plan
    plan = Plan(wl.fc, wl.cross, wl.model, wl.model_type, max_batch=GB, embedding_dim_override=wl.emb, gemm_engine="bf16x3",
                max_keys=GB * wl.keys_per_row, max_nnz=GB * wl.ids_per_row, host_tables=host_tables)
    m = WideDeepModel(plan, device=0)
    m.init(seed=SEED)
    for s in range(RING):
        keys, offs, dense, label = wl.arrays(GB, s)
        m.upload_slot(s, Batch(GB, keys, offs, dense, label))
    m.eval_reset()
    for i in range(3 * RING):
        m.eval_accumulate_slot(i % RING)

    def window():
        m.eval_reset()
        for i in range(steps):
            m.eval_accumulate_slot(i % RING)
        m.eval_finish()

    dt = timed(window, m.sync, lambda x: x)
    dev_bytes, host_bytes = m.memory_usage()
    m.close()
    return dict(examples_per_s=GB * steps / dt, step_ms=1e3 * dt / steps, hbm_bytes=dev_bytes, host_bytes=host_bytes)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--same-gpu", action="store_true", help="every process on cuda:0 (overhead and correctness, not scaling)")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file (rank 0)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    import bench
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = 0 if args.same_gpu else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")                 # plumbing only: IPC handles, timings, the results' comparison
    wl = bench.Workload("criteo", world)
    B = wl.batch
    rate, dt, same, hbm = sharded_rate(wl, B, args.steps, dev, world, rank)
    hbms = [None] * world
    dist.all_gather_object(hbms, hbm)
    dist.barrier()                                  # every sharded model freed before rank 0 builds the single-process ones
    ok = same
    if rank == 0:
        host = [t["name"] for t in plans(wl, B, world, 0, []).tables if t["sharded"]]
        res = dict(gpu_info(), workload="criteo", same_gpu=args.same_gpu, world=world, per_rank_batch=B, global_batch=B * world,
                   steps_per_window=args.steps, ring=RING,
                   sharded=dict(examples_per_s=rate, step_ms=1e3 * dt / args.steps, hbm_bytes_per_rank=hbms, identical_on_every_rank=same),
                   single_auto=single_rate(wl, B * world, args.steps, None),
                   single_host=single_rate(wl, B * world, args.steps, host))
        line = json.dumps(res)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
