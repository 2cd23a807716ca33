"""Adam on the Criteo shape (33.76M embedding rows x 32, 26 tables; Adam for both linear_optimizer and dnn_optimizer), one GPU.

    python tools/adam_bench.py [--other DIR] [--runs 3] [--steps 100] [--warmup 10]

Each arm runs in its own process: examples/s over `steps` graph-replayed train steps (batch 8192, a ring of 4 resident batches),
kernel launches per step, then a separate torch.profiler run of 10 steps for the kernels that move the rows no gradient touched
(adam_untouched_*: one pass; adam_decay / adam_step: the two passes of an older build), reported with their achieved bytes/s.  The
bytes are computed here from the shapes: the single pass reads and writes w, m and v of every row, 24 * D bytes per row (wide rows:
D = 1); the two passes move 32 * D.  --other DIR runs a second source tree (e.g. an export of another commit, with its library
built) alternately with this one, `runs` times each.  A last run trains the same model row-sharded over two ranks of a
LocalShardGroup: on one GPU the two ranks time-slice it, so that rate is not a multi-GPU rate.  The card's name and power limit are
read in the same call."""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RING = 4


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def conf():
    from wide_deep_b200 import synthetic
    fc, cross, model, emb = synthetic.criteo_conf()
    model = dict(model, linear_optimizer="Adam", dnn_optimizer="Adam")
    return fc, cross, model, emb


def batches(fc, B, rank=0):
    import numpy as np
    from wide_deep_b200 import synthetic
    from wide_deep_b200.model import Batch
    out = []
    for s in range(RING):
        keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=rank * 1000 + s)
        out.append(Batch(B, np.ascontiguousarray(keys.reshape(-1)), None, dense, label))
    return out


def untouched_bytes(plan):
    """(bytes of one pass over the embedding records, over the wide records), 24 * D per row"""
    emb = sum(24 * t["dim"] * t["rows"] for t in plan.tables)
    wide = 24 * sum(c.buckets for c in plan.wide_columns) if plan.use_wide else 0
    return emb, wide


def child_single(args):
    import torch
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import Plan
    fc, cross, model, emb = conf()
    B = args.batch
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, gemm_engine="bf16x3", max_keys=B * n_cat,
                max_nnz=B * (len(fc) + len(cross)))
    pm = WideDeepModel(plan)
    pm.init(seed=0x5EED0005)
    for s, b in enumerate(batches(fc, B)):
        pm.upload_slot(s, b)
    for i in range(3 * RING):                          # two eager steps and the capture of every slot
        pm.train_step_slot(i % RING, want_loss=False)
    pm.sync()
    l0 = pm.launch_count()
    for i in range(args.warmup):
        pm.train_step_slot(i % RING, want_loss=False)
    pm.sync()
    launches = (pm.launch_count() - l0) // max(args.warmup, 1)
    stream = torch.cuda.ExternalStream(pm.stream(), device=torch.device("cuda", 0))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(args.steps):
        pm.train_step_slot(i % RING, want_loss=False)
    e1.record(stream)
    pm.sync()
    ms = e0.elapsed_time(e1) / args.steps
    loss = pm.train_step_slot(0, want_loss=True)
    # kernel times in a run of their own
    from torch.profiler import ProfilerActivity, profile
    n_prof = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(n_prof):
            pm.train_step_slot(i % RING, want_loss=False)
        pm.sync()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and "adam_" in ev.name:
            key = ev.name.split("(")[0].replace("void ", "").replace("wd::", "")
            kern[key] = kern.get(key, 0.0) + ev.device_time / 1000.0 / n_prof     # ms per step
    eb, wb = untouched_bytes(plan)
    out = {"examples_per_s": B / (ms / 1000.0), "step_ms": ms, "launches_per_step": launches, "loss": loss, "adam_kernels_ms_per_step": kern}
    ue, uw = kern.get("adam_untouched_emb_kernel"), kern.get("adam_untouched_wide_kernel")
    if ue:
        out["untouched_emb_GBps"] = eb / (ue / 1000.0) / 1e9
        out["untouched_emb_bytes"] = eb
    if uw:
        out["untouched_wide_GBps"] = wb / (uw / 1000.0) / 1e9
    dec = sum(v for k, v in kern.items() if k.startswith("adam_decay") or k.startswith("adam_step"))
    if dec:                                            # the two passes of an older build: 32 * D bytes per row
        out["two_pass_ms"] = dec
        out["two_pass_GBps"] = (eb + wb) * 32 / 24 / (dec / 1000.0) / 1e9
    print("RESULT " + json.dumps(out), flush=True)


def child_sharded(args):
    import time
    from wide_deep_b200.model import WideDeepModel
    from wide_deep_b200.plan import Plan
    from wide_deep_b200.sharded import LocalShardGroup
    fc, cross, model, emb = conf()
    G, B = 2, args.batch
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    models = [WideDeepModel(Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, gemm_engine="bf16x3",
                                 max_keys=B * n_cat, max_nnz=B * (len(fc) + len(cross)), dense_exchange_max_rows=16384,
                                 shard_world=G, shard_rank=r, shard_slack=1.5)) for r in range(G)]
    for m in models:
        m.init(seed=0x5EED0005)
    grp = LocalShardGroup(models)
    per_rank = [batches(fc, B, r) for r in range(G)]
    for s in range(RING):
        for r, m in enumerate(models):
            m.upload_slot(s, per_rank[r][s])
    for i in range(2 * RING):
        grp.train_step(slot=i % RING)
    n = max(args.steps // 4, 10)
    t0 = time.perf_counter()
    for i in range(n):
        grp.train_step(slot=i % RING)                  # (ends with a device->host read of every rank's loss)
    dt = (time.perf_counter() - t0) / n
    print("RESULT " + json.dumps({"examples_per_s": G * B / dt, "step_ms": dt * 1000.0, "ranks": G,
                                  "note": "LocalShardGroup, both ranks on one GPU (time-sliced): not a multi-GPU rate"}), flush=True)


def run_child(root, mode, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--child", mode, "--root", root, "--steps", str(args.steps), "--warmup",
           str(args.warmup), "--batch", str(args.batch)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    for line in r.stdout.splitlines():
        if line.startswith("RESULT "):
            return json.loads(line[7:])
    return {"error": (r.stdout[-1500:] + r.stderr[-1500:]).strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", help="a second source tree (its library built) to alternate with this one")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--child", choices=["single", "sharded"])
    ap.add_argument("--root", default=HERE)
    args = ap.parse_args()
    if args.child:
        sys.path.insert(0, os.path.abspath(args.root))
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("no CUDA device")
        return child_single(args) if args.child == "single" else child_sharded(args)
    print("card: " + card(), flush=True)
    arms = [("this", HERE)] + ([("other", os.path.abspath(args.other))] if args.other else [])
    for run in range(args.runs):
        for name, root in arms:
            print(json.dumps({"run": run, "arm": name, "single_gpu": run_child(root, "single", args)}), flush=True)
    print(json.dumps({"arm": "this", "sharded_G2_one_gpu": run_child(HERE, "sharded", args)}), flush=True)
    print("card: " + card(), flush=True)


if __name__ == "__main__":
    main()
