"""Host-placed embedding tables against the same tables in HBM, on one GPU.

For each workload (the Criteo and multihot shapes of wide_deep_b200/synthetic.py, as bench.py builds them) two models live in
one process: A with every table in HBM, B with every table larger than --host-min-rows rows in page-locked host memory
(Plan(host_tables=[...])).  Both start from the same init seed and train on the same seeded resident batches; the timed windows
alternate A / B / A / B, so both models take the same sequence of steps.  Reported per workload:
  * examples/s of each model (host clock around windows that end in a device synchronise);
  * unique host-table rows per step (U_host, counted from the column ids of the ring's batches), unique embedding rows per
    step (d_nuniq), and the PCIe bytes per step, U_host x record bytes in each direction;
  * pinned host->device / device->host copy bandwidth measured in the same run, and the PCIe floor of the extra step time;
  * GPU name, power limit and max SM clock (read-only nvidia-smi query).
Afterwards every parameter and optimizer slot of B is compared byte for byte with A's.

    python tools/host_tables_bench.py [--workloads criteo,multihot] [--steps 50] [--warmup 12] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RING = 4


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clk = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:                       # the numbers are still printed, without the card they were taken on
        return {"gpu": "unknown (%s)" % e}


def copy_bandwidth(nbytes=1 << 30, reps=10):
    """Pinned host <-> device copy bandwidth in GB/s (CUDA events around `reps` copies of `nbytes`)."""
    import torch
    h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = {}
    for name, dst, src in (("h2d_gbps", d, h), ("d2h_gbps", h, d)):
        dst.copy_(src, non_blocking=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        out[name] = nbytes * reps / (e0.elapsed_time(e1) / 1e3) / 1e9
    del h, d
    torch.cuda.empty_cache()
    return out


def build(wl, B, host_tables):
    from wide_deep_b200.plan import Plan
    return Plan(wl["fc"], wl["cross"], wl["model"], wl["model_type"], max_batch=B, embedding_dim_override=wl["emb"],
                gemm_engine="bf16x3", max_keys=B * wl["keys_per_row"], max_nnz=B * wl["ids_per_row"], host_tables=host_tables)


def workload(name):
    from wide_deep_b200 import synthetic
    if name == "criteo":
        fc, cross, model, emb = synthetic.criteo_conf()
        n_cat = sum(1 for c in fc.values() if c["type"] == "category")
        return dict(fc=fc, cross=cross, model=model, emb=emb, model_type="wide_deep", ids_per_row=len(fc) + len(cross),
                    keys_per_row=n_cat, batch=8192,
                    arrays=lambda B, s: synthetic.criteo_batch_arrays(fc, B, step=s))
    if name == "multihot":
        fc, cross, model, emb = synthetic.multihot_conf()
        return dict(fc=fc, cross=cross, model=model, emb=emb, model_type="deep", ids_per_row=128, keys_per_row=128, batch=8192,
                    arrays=lambda B, s: synthetic.multihot_batch_arrays(B, step=s))
    raise SystemExit("unknown workload %r" % name)


def batch_of(name, arrays, B):
    from wide_deep_b200.model import Batch
    if name == "criteo":
        keys, dense, label = arrays
        return Batch(B, keys.reshape(-1), None, dense, label)
    keys, offs, label = arrays
    return Batch(B, keys, offs, None, label)


def all_equal(a, b):
    for name in a.tensor_names():
        for s in range(a.n_slots(name) + 1):
            if a.get_tensor(name, slot=s).tobytes() != b.get_tensor(name, slot=s).tobytes():
                return False, "%s slot %d" % (name, s)
    return True, None


def run(name, steps, warmup, host_min_rows, seed=7):
    from wide_deep_b200.model import WideDeepModel
    wl = workload(name)
    B = wl["batch"]
    plan_a = build(wl, B, [])
    host = [t["name"] for t in plan_a.tables if t["rows"] > host_min_rows]
    plan_b = build(wl, B, host)
    batches = [batch_of(name, wl["arrays"](B, s), B) for s in range(RING)]
    t0 = time.time()
    a = WideDeepModel(plan_a).init(seed)
    b = WideDeepModel(plan_b).init(seed)
    setup_s = time.time() - t0
    for m in (a, b):
        for s in range(RING):
            m.upload_slot(s, batches[s])
    # U_host: unique ids of the host tables' columns in each ring batch
    by_table = {i: t for i, t in enumerate(plan_a.tables)}
    host_cols = [ci for ci, c in enumerate(plan_a.columns) if c.emb_table >= 0 and by_table[c.emb_table]["name"] in host]
    rec_bytes = {}
    nslots = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan_a.dnn_opt["kind"]]
    for ci in host_cols:
        t = by_table[plan_a.columns[ci].emb_table]
        rec_bytes[ci] = ((t["dim"] + 3) // 4 * 4) * (1 + nslots) * 4
    u_host, bytes_way, nuniq = [], [], []
    step = 0
    for i in range(warmup):                      # same steps on both models; the first RING steps also count the rows
        for m in (a, b):
            m.train_step_slot(step % RING, want_loss=True)
        if i < RING:
            offs, ids = a.column_ids()
            C = len(plan_a.columns)
            u, by = 0, 0
            col = np.repeat(np.tile(np.arange(C), B), np.diff(offs))
            for ci in host_cols:
                n = len(np.unique(ids[col == ci]))
                u += n
                by += n * rec_bytes[ci]
            u_host.append(u)
            bytes_way.append(by)
            nuniq.append(a.sparse_grads(0)[2])
        step += 1
    times = {"hbm": [], "host": []}
    for w in range(4):                            # A / B / A / B
        m, key = (a, "hbm") if w % 2 == 0 else (b, "host")
        s0 = step - (steps if w % 2 else 0)
        m.sync()
        t = time.perf_counter()
        for i in range(steps):
            m.train_step_slot((s0 + i) % RING, want_loss=False)
        m.sync()
        times[key].append(time.perf_counter() - t)
        if w % 2 == 0:
            step += steps
    rate = {k: B * steps / min(v) for k, v in times.items()}
    same, where = all_equal(a, b)
    dev_b, host_b = b.memory_usage()
    dev_a, _ = a.memory_usage()
    a.close()
    b.close()
    return dict(workload=name, batch=B, steps_per_window=steps, host_tables=len(host), host_table_bytes=host_b,
                hbm_bytes_hbm_model=dev_a, hbm_bytes_host_model=dev_b, setup_s=round(setup_s, 1),
                examples_per_s_hbm=rate["hbm"], examples_per_s_host=rate["host"],
                step_ms_hbm=1e3 * min(times["hbm"]) / steps, step_ms_host=1e3 * min(times["host"]) / steps,
                window_s=times, unique_rows_per_step=float(np.mean(nuniq)), unique_host_rows_per_step=float(np.mean(u_host)),
                pcie_bytes_per_step_each_way=float(np.mean(bytes_way)), byte_identical=same, first_difference=where)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=12, help="steps before timing (3 per ring slot: two eager, then the graph)")
    ap.add_argument("--host-min-rows", type=int, default=16384, help="tables with more rows than this go to host memory")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    info = gpu_info()
    bw = copy_bandwidth()
    print(json.dumps(dict(info, **bw)), flush=True)
    ok = True
    for name in args.workloads.split(","):
        r = run(name, args.steps, args.warmup, args.host_min_rows)
        extra = (r["step_ms_host"] - r["step_ms_hbm"]) / 1e3
        by = r["pcie_bytes_per_step_each_way"]
        r.update(info)
        r["pcie_floor_ms"] = 1e3 * (by / (bw["h2d_gbps"] * 1e9) + by / (bw["d2h_gbps"] * 1e9))
        r["achieved_pcie_gbps_over_extra_time"] = 2 * by / extra / 1e9 if extra > 0 else None
        ok &= r["byte_identical"]
        line = json.dumps(r)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
