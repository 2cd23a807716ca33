"""Cost of a train step armed for layer summaries on the Criteo shape (bf16x3 engine, batch 8192), one GPU.

    python tools/summary_bench.py [--steps 200] [--armed 20]

Reports the plain step (graph-replayed, device events over `steps` steps), single steps timed one at a time with device events
(plain: graph replay; armed: eager, plus the statistics kernel), the statistics kernel's own time from a torch.profiler run of
`armed` armed steps, and the bytes that kernel reads (every segment once: the deep input, each hidden layer's post-activation
values, the tower and wide logits) over that time, as a share of the H100 SXM's 3.35 TB/s.  The card's name and power limit are
read in the same call."""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)
RING = 4


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def segment_bytes(plan, B):
    """Bytes the statistics kernel reads per armed step: B rows of every segment (the deep input's physical row, its padding
    skipped only after the load of the line)."""
    n = plan.d0_phys if plan.use_deep else 0
    for tw in plan.towers:
        n += sum(plan.out_width(u) for u in tw["hidden"]) + 1
    n += 1 if plan.use_wide else 0
    return 4 * B * n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--armed", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8192)
    args = ap.parse_args()
    import numpy as np
    import torch
    from wide_deep_b200 import synthetic
    from wide_deep_b200.model import Batch, WideDeepModel
    from wide_deep_b200.plan import Plan
    fc, cross, model, emb = synthetic.criteo_conf()
    B = args.batch
    n_cat = sum(1 for c in fc.values() if c["type"] == "category")
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=emb, gemm_engine="bf16x3", max_keys=B * n_cat,
                max_nnz=B * (len(fc) + len(cross)))
    pm = WideDeepModel(plan).init(seed=0x5EED0007)
    for s in range(RING):
        keys, dense, label = synthetic.criteo_batch_arrays(fc, B, step=s)
        pm.upload_slot(s, Batch(B, np.ascontiguousarray(keys.reshape(-1)), None, dense, label))
    for i in range(3 * RING):                          # two eager steps and the capture of every slot
        pm.train_step_slot(i % RING, want_loss=False)
    pm.arm_summary()                                   # first armed step: segment table and buffers
    pm.train_step_slot(0, want_loss=False)
    pm.layer_statistics()
    pm.sync()
    stream = torch.cuda.ExternalStream(pm.stream(), device=torch.device("cuda", 0))
    ev = lambda: torch.cuda.Event(enable_timing=True)
    e0, e1 = ev(), ev()
    l0 = pm.launch_count()
    e0.record(stream)
    for i in range(args.steps):
        pm.train_step_slot(i % RING, want_loss=False)
    e1.record(stream)
    pm.sync()
    plain_ms = e0.elapsed_time(e1) / args.steps
    launches = (pm.launch_count() - l0) / args.steps

    def one(armed, i):
        a, b = ev(), ev()
        pm.sync()
        if armed:
            pm.arm_summary()
        a.record(stream)
        pm.train_step_slot(i % RING, want_loss=False)
        b.record(stream)
        pm.sync()
        if armed:
            pm.layer_statistics()
        return a.elapsed_time(b)
    single = {"plain": [], "armed": []}
    for i in range(args.armed):                        # alternated
        single["plain"].append(one(False, i))
        single["armed"].append(one(True, i))
    med = {k: float(np.median(v)) for k, v in single.items()}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.armed):
            pm.arm_summary()
            pm.train_step_slot(i % RING, want_loss=False)
            pm.sync()
            pm.layer_statistics()
        torch.cuda.synchronize()
    kt = [e.device_time / 1000.0 for e in prof.events() if e.device_type.name == "CUDA" and "summary_stats_kernel" in e.name]
    k_ms = float(np.median(kt)) if kt else None
    nbytes = segment_bytes(plan, B)
    out = {"card": card(), "batch": B, "plain_step_ms_graphed": plain_ms, "launches_per_plain_step": launches,
           "single_step_ms_median": med, "armed_extra_ms": med["armed"] - med["plain"],
           "stats_kernel_ms": k_ms if k_ms is not None else "not measured", "stats_kernel_launches": len(kt), "bytes_read": nbytes,
           "stats_kernel_TBps": nbytes / (k_ms / 1000.0) / 1e12 if k_ms else "not measured",
           "share_of_3.35TBps": nbytes / (k_ms / 1000.0) / 3.35e12 if k_ms else "not measured"}
    print("RESULT " + json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
