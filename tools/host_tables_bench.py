"""Host-placed embedding tables against the same tables in HBM, on one GPU.

For each workload (the Criteo and multihot shapes of wide_deep_b200/synthetic.py, as bench.py builds them) up to three models
live in one process: A with every table in HBM, B with every table larger than --host-min-rows rows in page-locked host memory
(Plan(host_tables=[...])), and with --cache-bytes N > 0 also C, which is B plus an HBM cache of N bytes for the host records
(Plan(host_cache_bytes=N)).  All start from the same init seed and train on the same seeded resident batches (a ring of --ring
distinct batches, so a cache sees as many distinct rows as --ring steps of a real stream); the timed windows alternate
A / B / C / A / B / C, so every model takes the same sequence of steps.  --zipf ALPHA draws the Criteo ids from a Zipf
distribution (synthetic.criteo_batch_arrays(zipf=...)); multihot ids stay uniform.  Reported per workload:
  * examples/s of each model (host clock around windows that end in a device synchronise);
  * for C, from its cache counters over the timed windows: hit rate, and PCIe records and bytes per step in each direction
    (in: loads + overflow rows; out: dirty evictions + overflow rows);
  * unique host-table rows per step (U_host, counted from the column ids of the ring's batches), unique embedding rows per
    step (d_nuniq), and the PCIe bytes per step, U_host x record bytes in each direction;
  * pinned host->device / device->host copy bandwidth measured in the same run, and the PCIe floor of the extra step time;
  * GPU name, power limit and max SM clock (read-only nvidia-smi query).
Afterwards every parameter and optimizer slot of B and C is compared byte for byte with A's.

--dnn-opt OPT replaces the workload's dnn_optimizer (e.g. Adam).  With Adam, B and C are deferred Adam tables
(Plan(defer_adam=True)): rows no gradient touched catch up on their missed steps when next staged.  Then also reported: the
catch-up counters per timed step of B and C (rows caught up, steps replayed, steps skipped by the early exit, longest gap), and
the time of one settling read of B's largest host table (a whole-table read first replays every row's missed steps).

    python tools/host_tables_bench.py [--workloads criteo,multihot] [--steps 50] [--ring 64] [--zipf 1.05] [--cache-bytes N]
                                      [--dnn-opt Adam] [--out FILE]
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


def build(wl, B, host_tables, cache_bytes=0):
    from wide_deep_b200.plan import Plan
    return Plan(wl["fc"], wl["cross"], wl["model"], wl["model_type"], max_batch=B, embedding_dim_override=wl["emb"],
                gemm_engine="bf16x3", max_keys=B * wl["keys_per_row"], max_nnz=B * wl["ids_per_row"], host_tables=host_tables,
                host_cache_bytes=cache_bytes, defer_adam=bool(host_tables))


def workload(name, zipf=None, dnn_opt=None):
    wl = _workload(name, zipf)
    if dnn_opt:
        wl["model"] = dict(wl["model"], dnn_optimizer=dnn_opt)
    return wl


def _workload(name, zipf=None):
    from wide_deep_b200 import synthetic
    if name == "criteo":
        fc, cross, model, emb = synthetic.criteo_conf()
        n_cat = sum(1 for c in fc.values() if c["type"] == "category")
        return dict(fc=fc, cross=cross, model=model, emb=emb, model_type="wide_deep", ids_per_row=len(fc) + len(cross),
                    keys_per_row=n_cat, batch=8192,
                    arrays=lambda B, s: synthetic.criteo_batch_arrays(fc, B, step=s, zipf=zipf))
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


def run(name, steps, warmup, host_min_rows, ring, zipf=None, cache_bytes=0, seed=7, dnn_opt=None):
    from wide_deep_b200.model import WideDeepModel
    wl = workload(name, zipf, dnn_opt)
    B = wl["batch"]
    plan_a = build(wl, B, [])
    host = [t["name"] for t in plan_a.tables if t["rows"] > host_min_rows]
    plans = {"hbm": plan_a, "host": build(wl, B, host)}
    if cache_bytes > 0:
        plans["cache"] = build(wl, B, host, cache_bytes)
    batches = [batch_of(name, wl["arrays"](B, s), B) for s in range(ring)]
    t0 = time.time()
    models = {k: WideDeepModel(p).init(seed) for k, p in plans.items()}
    setup_s = time.time() - t0
    a = models["hbm"]
    for m in models.values():
        for s in range(ring):
            m.upload_slot(s, batches[s])
    # U_host: unique ids of the host tables' columns in each ring batch
    by_table = {i: t for i, t in enumerate(plan_a.tables)}
    host_cols = [ci for ci, c in enumerate(plan_a.columns) if c.emb_table >= 0 and by_table[c.emb_table]["name"] in host]
    rec_bytes = {}
    nslots = {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan_a.dnn_opt["kind"]]
    adam = plan_a.dnn_opt["kind"] == "adam"
    for ci in host_cols:
        t = by_table[plan_a.columns[ci].emb_table]
        rec_bytes[ci] = (((t["dim"] + 3) // 4 * 4) * (1 + nslots) + (4 if adam else 0)) * 4     # (deferred Adam: + the stamp)
    u_host, bytes_way, nuniq = [], [], []
    step = 0
    for i in range(warmup):                      # same steps on every model; the first steps also count the rows
        for m in models.values():
            m.train_step_slot(step % ring, want_loss=True)
        if i < min(ring, 8):
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
    if "cache" in models:
        models["cache"].host_cache_stats(reset=True)
    for m in models.values():
        m.deferred_adam_stats(reset=True)
    times = {k: [] for k in models}
    for w in range(2):                            # A / B / C / A / B / C, each window on the same steps
        for key, m in models.items():
            m.sync()
            t = time.perf_counter()
            for i in range(steps):
                m.train_step_slot((step + i) % ring, want_loss=False)
            m.sync()
            times[key].append(time.perf_counter() - t)
        step += steps
    rate = {k: B * steps / min(v) for k, v in times.items()}
    catch_up = {k: {c: (v if c == "max_gap" else v / (2 * steps)) for c, v in m.deferred_adam_stats().items()}
                for k, m in models.items() if k != "hbm"}
    phases = {}
    for key, m in models.items():                 # one profiled (eager) step per model, the same step on each: phase times in ms
        m.set_profile(True)
        m.train_step_slot(step % ring, want_loss=True)
        phases[key] = {n: round(v, 4) for n, v in m.last_timings().items()}
        m.set_profile(False)
    step += 1
    res = dict(workload=name, zipf=zipf, ring=ring, batch=B, steps_per_window=steps, host_tables=len(host), setup_s=round(setup_s, 1),
               unique_rows_per_step=float(np.mean(nuniq)), unique_host_rows_per_step=float(np.mean(u_host)),
               pcie_bytes_per_step_each_way=float(np.mean(bytes_way)), window_s=times, phase_ms=phases)
    for k, m in models.items():
        dev, hb = m.memory_usage()
        res["examples_per_s_" + k] = rate[k]
        res["step_ms_" + k] = 1e3 * min(times[k]) / steps
        res["hbm_bytes_" + k] = dev
        res["host_bytes_" + k] = hb
    if "cache" in models:
        c = models["cache"].host_cache_stats()
        n = 2 * steps
        rec = float(np.mean(bytes_way)) / max(float(np.mean(u_host)), 1.0)       # mean record bytes of the host rows
        looked_up = c["hits"] + c["loads"] + c["overflow"]
        res.update(cache_bytes=cache_bytes, cache_slots=c["capacity"], cache_counters=c,
                   hit_rate=c["hits"] / looked_up if looked_up else None,
                   pcie_records_in_per_step=(c["loads"] + c["overflow"]) / n,
                   pcie_records_out_per_step=(c["evictions"] + c["overflow"]) / n,
                   pcie_bytes_in_per_step=(c["loads"] + c["overflow"]) / n * rec,
                   pcie_bytes_out_per_step=(c["evictions"] + c["overflow"]) / n * rec)
    if adam and host:
        res["catch_up_per_step"] = catch_up
        largest = max((t for t in plan_a.tables if t["name"] in host), key=lambda t: t["rows"] * t["dim"])
        from wide_deep_b200.plan import T_EMB_TABLE
        tname = [n for n, v in plan_a.tensor_names.items() if v[0] == T_EMB_TABLE and plan_a.tables[v[1]]["name"] == largest["name"]][0]
        mb = models["host"]
        mb.sync()
        mb.deferred_adam_stats(reset=True)
        t = time.perf_counter()
        mb.get_tensor(tname)
        res["settle_read_s"] = time.perf_counter() - t
        res["settle_table"] = dict(name=largest["name"], rows=largest["rows"], dim=largest["dim"], counters=mb.deferred_adam_stats())
        t = time.perf_counter()
        mb.get_tensor(tname)
        res["second_read_s"] = time.perf_counter() - t
    for k in models:
        if k == "hbm":
            continue
        same, where = all_equal(a, models[k])
        res["byte_identical_" + k] = same
        res["first_difference_" + k] = where
    res["byte_identical"] = all(res["byte_identical_" + k] for k in models if k != "hbm")
    for m in models.values():
        m.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--ring", type=int, default=64, help="distinct resident batches the steps cycle through (at most 64)")
    ap.add_argument("--warmup", type=int, default=None, help="steps before timing (default 3 per ring slot: two eager, then the graph)")
    ap.add_argument("--zipf", type=float, default=None, help="Criteo ids from Zipf(ALPHA) instead of uniform")
    ap.add_argument("--cache-bytes", type=int, default=0, help="also run the host model with an HBM cache of this many bytes")
    ap.add_argument("--host-min-rows", type=int, default=16384, help="tables with more rows than this go to host memory")
    ap.add_argument("--dnn-opt", default=None, help="dnn optimizer of every workload (e.g. Adam: deferred Adam host tables)")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    info = gpu_info()
    bw = copy_bandwidth()
    print(json.dumps(dict(info, **bw)), flush=True)
    ok = True
    for name in args.workloads.split(","):
        r = run(name, args.steps, 3 * args.ring if args.warmup is None else args.warmup, args.host_min_rows, args.ring,
                zipf=args.zipf, cache_bytes=args.cache_bytes, dnn_opt=args.dnn_opt)
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
