"""Row-sharded embedding tables with their shards in page-locked host memory against the same shards in HBM.

Run under torch.distributed.run, one process per GPU (or, with --same-gpu, the processes share cuda:0):

    python -m torch.distributed.run --nproc-per-node 2 tools/sharded_host_tables_bench.py [--same-gpu] [--workloads criteo,multihot]
        [--steps 30] [--zipf 1.05] [--cache-bytes N] [--out FILE]

For each workload (the Criteo and multihot shapes of wide_deep_b200/synthetic.py, sharded as bench.py --gpus N shards them:
tables larger than bench.DENSE_EXCHANGE_ROWS rows row-sharded, bf16x3 towers) every process holds two models with the same
initial parameters, each driven by its own ShardedTrainer: "hbm" with every shard in HBM and "host" with every sharded table's shard
in host memory (Plan(host_tables=[...])); with --cache-bytes N > 0 also "cache", the host model with an HBM cache of N bytes per
rank in front of each owner's host shards (Plan(shard_cache_bytes=N)).  All train on the same ring of resident batches; the timed
windows alternate hbm / host / cache / hbm / host / cache.  --zipf ALPHA draws the Criteo ids from a Zipf distribution (as
tools/host_tables_bench.py does; multihot ids stay uniform): uniform ids understate what a cache gets.  Reported (rank 0 prints
one JSON line per workload):
  * global examples/s of each placement (all ranks' examples over the slowest rank's window, best of two windows);
  * per rank: unique owned host rows per step (from the column ids of every rank's batch shard) and the PCIe bytes each way
    (one record per unique owned host row in each direction);
  * per rank, for "cache", from its counters over the timed windows: hit rate, loads, evictions and the records it moved over
    PCIe per step in each direction;
  * per rank and model: the interval between leaving flag barrier A and entering barrier B of a replayed step (WD_SHARD_TRACE):
    routing delivered -> pooled sums served, which for the host model includes grouping the received rows and the stage-in;
  * per rank and model: the phase times (ms) of one eager, profiled step (wd_last_timings);
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

from tools.host_tables_bench import batch_of, copy_bandwidth, gpu_info, workload    # noqa: E402

RING = 8
BAR_A, BAR_B = 0, 1


def plans(wl, B, world, rank, host_tables, cache_bytes=0):
    import bench
    from wide_deep_b200.plan import Plan
    return Plan(wl.fc, wl.cross, wl.model, wl.model_type, max_batch=B, embedding_dim_override=wl.emb, gemm_engine="bf16x3",
                max_keys=B * wl.keys_per_row, max_nnz=B * wl.ids_per_row, dense_exchange_max_rows=bench.DENSE_EXCHANGE_ROWS,
                shard_world=world, shard_rank=rank, shard_slack=1.5, host_tables=host_tables, shard_cache_bytes=cache_bytes)


def a_to_b_us(model):
    tr = np.zeros(16, dtype=np.uint64)
    if model._lib.wd_debug_shard_trace(model._h, tr.ctypes.data_as(ctypes.c_void_p)) != 0:
        return None
    return (int(tr[2 * BAR_B]) - int(tr[2 * BAR_A + 1])) / 1e3


def run(name, steps, dev, world, rank, zipf=None, cache_bytes=0):
    import torch
    import torch.distributed as dist
    import bench
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.sharded import ShardedTrainer
    wl = bench.Workload(name, world)
    B = wl.batch
    plan_a = plans(wl, B, world, rank, [])
    host = [t["name"] for t in plan_a.tables if t["sharded"]]
    t0 = time.time()
    models = {"hbm": WideDeepModel(plan_a, device=dev), "host": WideDeepModel(plans(wl, B, world, rank, host), device=dev)}
    if cache_bytes > 0:
        models["cache"] = WideDeepModel(plans(wl, B, world, rank, host, cache_bytes), device=dev)
    for m in models.values():
        m.init(seed=0x5EED0005)
    trainers = {k: ShardedTrainer(m) for k, m in models.items()}
    setup_s = time.time() - t0
    arrays = workload(name, zipf)["arrays"]
    for s in range(RING):
        batch = batch_of(name, arrays(B, 1000 * rank + s), B)             # each rank's own batch shard
        for m in models.values():
            m.upload_slot(s, batch)
    # unique owned host rows per step: the ids of the host tables' columns in every rank's shard of the step, owned by this rank
    cols = [ci for ci, c in enumerate(plan_a.columns) if c.emb_table >= 0 and plan_a.tables[c.emb_table]["name"] in host]
    nslots = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan_a.dnn_opt["kind"]]
    rec = {ci: ((plan_a.tables[plan_a.columns[ci].emb_table]["dim"] + 3) // 4 * 4) * (1 + nslots) * 4 for ci in cols}
    C = len(plan_a.columns)
    urows, ubytes = [], []
    a = models["hbm"]
    step = 0
    for i in range(3 * RING):                       # two eager steps and the capture per slot, the same steps on every model
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
    if "cache" in models:
        models["cache"].host_cache_stats(reset=True)
    times = {k: [] for k in models}
    for w in range(2):                              # hbm / host / cache / hbm / host / cache, each window on the same steps
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
    cache = None
    if "cache" in models:                           # counters of the timed windows and the trace step
        c = models["cache"].host_cache_stats()
        n = 2 * steps + 1
        looked_up = c["hits"] + c["loads"] + c["overflow"]
        cache = dict(counters=c, hit_rate=c["hits"] / looked_up if looked_up else None, loads_per_step=c["loads"] / n,
                     evictions_per_step=c["evictions"] / n, pcie_records_in_per_step=(c["loads"] + c["overflow"]) / n,
                     pcie_records_out_per_step=(c["evictions"] + c["overflow"]) / n)
    phases = {}
    if cache is not None:
        for key, t in trainers.items():             # one profiled (eager) step per model, the same step on each: phase times in ms
            models[key].set_profile(True)
            t.step_slot(step % RING, want_loss=True)
            phases[key] = {nm: round(v, 4) for nm, v in models[key].last_timings().items()}
            models[key].set_profile(False)
        step += 1
    same, where = True, None
    for key in models:
        if key == "hbm":
            continue
        for nm in a.tensor_names():
            for s in range(a.n_slots(nm) + 1):
                if same and a.get_tensor(nm, slot=s).tobytes() != models[key].get_tensor(nm, slot=s).tobytes():
                    same, where = False, ("" if key == "host" else key + ": ") + "%s slot %d" % (nm, s)
    mine = dict(rank=rank, unique_owned_host_rows_per_step=float(np.mean(urows)), pcie_bytes_each_way_per_step=float(np.mean(ubytes)),
                a_to_b_us=trace, host_bytes=models["host"].memory_usage()[1], hbm_bytes={k: m.memory_usage()[0] for k, m in models.items()},
                byte_identical=same, first_difference=where)
    if cache is not None:
        mine.update(cache=cache, phase_ms=phases)
    allr = [None] * world
    dist.all_gather_object(allr, mine)
    res = dict(workload=name, world=world, per_rank_batch=B, global_batch=B * world, steps_per_window=steps, ring=RING,
               sharded_host_tables=len(host), setup_s=round(setup_s, 1), window_s=times, ranks=allr,
               byte_identical=all(r["byte_identical"] for r in allr))
    if zipf is not None or cache_bytes > 0:
        res.update(zipf=zipf, cache_bytes=cache_bytes)
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
    ap.add_argument("--zipf", type=float, default=None, help="Criteo ids from Zipf(ALPHA) instead of uniform")
    ap.add_argument("--cache-bytes", type=int, default=0, help="also run the host model with an HBM cache of this many bytes per rank")
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
        r = run(name, args.steps, dev, world, rank, zipf=args.zipf, cache_bytes=args.cache_bytes)
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
