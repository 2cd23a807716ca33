"""Row-sharded embedding tables with their shards in page-locked host memory against the same shards in HBM.

Run under torch.distributed.run, one process per GPU (or, with --same-gpu, the processes share cuda:0):

    python -m torch.distributed.run --nproc-per-node 2 tools/sharded_host_tables_bench.py [--same-gpu] [--workloads criteo,multihot]
        [--steps 30] [--out FILE]

For each workload (the Criteo and multihot shapes of wide_deep_b200/synthetic.py, sharded as bench.py --gpus N shards them:
tables larger than bench.DENSE_EXCHANGE_ROWS rows row-sharded, bf16x3 towers) every process holds two models with the same
initial parameters, each driven by its own ShardedTrainer: "hbm" with every shard in HBM and "host" with every sharded table's shard
in host memory (Plan(host_tables=[...])).  Both train on the same ring of resident batches; the timed windows alternate
hbm / host / hbm / host.  Reported (rank 0 prints one JSON line per workload):
  * global examples/s of each placement (all ranks' examples over the slowest rank's window, best of two windows);
  * per rank: unique owned host rows per step (from the column ids of every rank's batch shard) and the PCIe bytes each way
    (one record per unique owned host row in each direction);
  * per rank and model: the interval between leaving flag barrier A and entering barrier B of a replayed step (WD_SHARD_TRACE):
    routing delivered -> pooled sums served, which for the host model includes grouping the received rows and the stage-in;
  * pinned host <-> device copy bandwidth of every rank; GPU name, power limit and max SM clock.
At the end every rank compares every parameter and optimizer slot of its local shards byte for byte.
With --same-gpu the processes time-slice one GPU and share one PCIe link: the numbers show overhead and correctness, not scaling.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("WD_SHARD_TRACE", "1")          # read by wd_model_create: flag-barrier stamps of the last step

from tools.host_tables_bench import copy_bandwidth, gpu_info    # noqa: E402

RING = 8
BAR_A, BAR_B = 0, 1


def plans(wl, B, world, rank, host_tables):
    import bench
    from wide_deep_b200.plan import Plan
    return Plan(wl.fc, wl.cross, wl.model, wl.model_type, max_batch=B, embedding_dim_override=wl.emb, gemm_engine="bf16x3",
                max_keys=B * wl.keys_per_row, max_nnz=B * wl.ids_per_row, dense_exchange_max_rows=bench.DENSE_EXCHANGE_ROWS,
                shard_world=world, shard_rank=rank, shard_slack=1.5, host_tables=host_tables)


def a_to_b_us(model):
    tr = np.zeros(16, dtype=np.uint64)
    if model._lib.wd_debug_shard_trace(model._h, tr.ctypes.data_as(ctypes.c_void_p)) != 0:
        return None
    return (int(tr[2 * BAR_B]) - int(tr[2 * BAR_A + 1])) / 1e3


def run(name, steps, dev, world, rank):
    import torch
    import torch.distributed as dist
    import bench
    from wide_deep_b200.model import Batch, WideDeepModel
    from wide_deep_b200.sharded import ShardedTrainer
    wl = bench.Workload(name, world)
    B = wl.batch
    plan_a = plans(wl, B, world, rank, [])
    host = [t["name"] for t in plan_a.tables if t["sharded"]]
    t0 = time.time()
    models = {"hbm": WideDeepModel(plan_a, device=dev), "host": WideDeepModel(plans(wl, B, world, rank, host), device=dev)}
    for m in models.values():
        m.init(seed=0x5EED0005)
    trainers = {k: ShardedTrainer(m) for k, m in models.items()}
    setup_s = time.time() - t0
    for s in range(RING):
        keys, offs, dense, label = wl.arrays(B, 1000 * rank + s)          # each rank's own batch shard
        for m in models.values():
            m.upload_slot(s, Batch(B, keys, offs, dense, label))
    # unique owned host rows per step: the ids of the host tables' columns in every rank's shard of the step, owned by this rank
    cols = [ci for ci, c in enumerate(plan_a.columns) if c.emb_table >= 0 and plan_a.tables[c.emb_table]["name"] in host]
    nslots = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan_a.dnn_opt["kind"]]
    rec = {ci: ((plan_a.tables[plan_a.columns[ci].emb_table]["dim"] + 3) // 4 * 4) * (1 + nslots) * 4 for ci in cols}
    C = len(plan_a.columns)
    urows, ubytes = [], []
    a = models["hbm"]
    step = 0
    for i in range(3 * RING):                       # two eager steps and the capture per slot, the same steps on both models
        for t in trainers.values():
            t.step_slot(step % RING, want_loss=False)
        if i < RING:
            offs, ids = a.column_ids()
            col = np.repeat(np.tile(np.arange(C), B), np.diff(offs))
            mine = {ci: ids[col == ci] for ci in cols}
            allr = [None] * world
            dist.all_gather_object(allr, mine)
            u = by = 0
            for ci in cols:
                g = np.unique(np.concatenate([r[ci] for r in allr]))
                n = int(np.count_nonzero(g % world == rank))
                u += n
                by += n * rec[ci]
            urows.append(u)
            ubytes.append(by)
        step += 1
    times = {k: [] for k in models}
    for w in range(2):                              # hbm / host / hbm / host, each window on the same steps
        for key, t in trainers.items():
            models[key].sync()
            dist.barrier()
            t0 = time.perf_counter()
            for i in range(steps):
                t.step_slot((step + i) % RING, want_loss=False)
            models[key].sync()
            dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64)
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)
            times[key].append(dt.item())
        step += steps
    trace = {}
    for key, t in trainers.items():                 # the trace holds the last step of each model: a replayed one
        t.step_slot(step % RING, want_loss=False)
        models[key].sync()
        trace[key] = a_to_b_us(models[key])
    step += 1
    same, where = True, None
    for nm in a.tensor_names():
        for s in range(a.n_slots(nm) + 1):
            if same and a.get_tensor(nm, slot=s).tobytes() != models["host"].get_tensor(nm, slot=s).tobytes():
                same, where = False, "%s slot %d" % (nm, s)
    mine = dict(rank=rank, unique_owned_host_rows_per_step=float(np.mean(urows)), pcie_bytes_each_way_per_step=float(np.mean(ubytes)),
                a_to_b_us=trace, host_bytes=models["host"].memory_usage()[1], hbm_bytes={k: m.memory_usage()[0] for k, m in models.items()},
                byte_identical=same, first_difference=where)
    allr = [None] * world
    dist.all_gather_object(allr, mine)
    res = dict(workload=name, world=world, per_rank_batch=B, global_batch=B * world, steps_per_window=steps, ring=RING,
               sharded_host_tables=len(host), setup_s=round(setup_s, 1), window_s=times, ranks=allr,
               byte_identical=all(r["byte_identical"] for r in allr))
    for k in models:
        res["examples_per_s_" + k] = B * world * steps / min(times[k])
        res["step_ms_" + k] = 1e3 * min(times[k]) / steps
    for m in models.values():
        m.sync()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--same-gpu", action="store_true", help="every process on cuda:0 (overhead and correctness, not scaling)")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file (rank 0)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = 0 if args.same_gpu else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")                 # plumbing only: IPC handles, ids for the row counts, timings
    bw = copy_bandwidth(256 << 20)
    allbw = [None] * world
    dist.all_gather_object(allbw, bw)
    if rank == 0:
        print(json.dumps(dict(gpu_info(), same_gpu=args.same_gpu, world=world, copy_bandwidth_per_rank=allbw)), flush=True)
    ok = True
    for name in args.workloads.split(","):
        r = run(name, args.steps, dev, world, rank)
        r["same_gpu"] = args.same_gpu
        ok &= r["byte_identical"]
        if rank == 0:
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                with open(args.out, "a") as fh:
                    fh.write(line + "\n")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
