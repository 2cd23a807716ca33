"""Save and restore time and host memory of the two checkpoint layouts, on one GPU.

For each workload (the Criteo and multihot shapes of wide_deep_b200/synthetic.py, tables scaled by --scale) and each placement
(hbm: every table in HBM; host: the tables of more than --host-min-rows rows in page-locked host memory; cache: the same behind an
HBM cache of --cache-bytes, whose slot metadata every chunk's tensor IO scans once) one model is built, trained --steps steps on
seeded batches, and then:
  * sharded layout (wide_deep_b200/checkpoint.py): save and restore seconds, and GB/s of checkpoint bytes (one process is one
    rank here, so these are per-rank figures);
  * .npz layout (checkpoint.save_npz / restore_npz, WideAndDeepClassifier's flat file), only when the model's checkpoint bytes are at most --npz-max-gb: the same;
  * peak traced host bytes (tracemalloc) of every save and restore.
After the restores every tensor is compared byte for byte with what was saved.  The card's name and power limit are printed with
the numbers.  Checkpoints go to --dir (a temporary directory by default), which is removed afterwards.

    python tools/checkpoint_bench.py [--workloads criteo,multihot] [--scale 0.1] [--steps 2] [--npz-max-gb 8] [--dir D] [--out FILE]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import tracemalloc

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from host_tables_bench import batch_of, gpu_info  # noqa: E402


def workload(name, scale):
    from wide_deep_b200 import synthetic
    if name == "criteo":
        fc, cross, model, emb = synthetic.criteo_conf(scale=scale)
        n_cat = sum(1 for c in fc.values() if c["type"] == "category")
        return dict(fc=fc, cross=cross, model=model, emb=emb, model_type="wide_deep", ids_per_row=len(fc) + len(cross), keys_per_row=n_cat,
                    arrays=lambda B, s: synthetic.criteo_batch_arrays(fc, B, step=s))
    if name == "multihot":
        fc, cross, model, emb = synthetic.multihot_conf(rows=int(12_500_000 * scale))
        return dict(fc=fc, cross=cross, model=model, emb=emb, model_type="deep", ids_per_row=128, keys_per_row=128,
                    arrays=lambda B, s: synthetic.multihot_batch_arrays(B, step=s))
    raise SystemExit("unknown workload %r" % name)


def build(wl, B, host_tables, cache_bytes=0):
    from wide_deep_b200.plan import Plan
    return Plan(wl["fc"], wl["cross"], wl["model"], wl["model_type"], max_batch=B, embedding_dim_override=wl["emb"], gemm_engine="bf16x3",
                max_keys=B * wl["keys_per_row"], max_nnz=B * wl["ids_per_row"], host_tables=host_tables, defer_adam=bool(host_tables),
                host_cache_bytes=cache_bytes)


def traced(fn):
    """(result, seconds, peak traced host bytes) of fn()."""
    tracemalloc.start()
    try:
        tracemalloc.reset_peak()
        t0 = time.perf_counter()
        out = fn()
        return out, time.perf_counter() - t0, tracemalloc.get_traced_memory()[1]
    finally:
        tracemalloc.stop()


def dir_bytes(path):
    if os.path.isfile(path):
        return os.path.getsize(path)
    return sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))


def state(m):
    return {(n, s): m.get_tensor(n, s).tobytes() for n in m.tensor_names() for s in range(m.n_slots(n) + 1)}


def run(name, placement, args, root):
    from wide_deep_b200 import checkpoint
    from wide_deep_b200.model import WideDeepModel
    wl = workload(name, args.scale)
    B = args.batch
    plan = build(wl, B, [])
    if placement in ("host", "cache"):
        plan = build(wl, B, [t["name"] for t in plan.tables if t["rows"] > args.host_min_rows],
                     args.cache_bytes if placement == "cache" else 0)
    m = WideDeepModel(plan).init(7)
    for s in range(args.steps):
        m.train_step(batch_of(name, wl["arrays"](B, s), B))
    m.sync()
    out = dict(workload=name, placement=placement, host_bytes=m.memory_usage()[1], cache_slots=m.host_cache_stats()["capacity"],
               steps=args.steps)
    before = state(m) if args.check else None
    for layout in ("sharded", "npz"):
        d = os.path.join(root, "%s_%s_%s" % (name, placement, layout))
        if layout == "sharded":
            path, t_save, p_save = traced(lambda: checkpoint.save(d, [m]))
        else:
            total = sum(4 * int(np.prod(plan.tensor_names[n][3])) * (1 + m.n_slots(n)) for n in m.tensor_names())
            if total > args.npz_max_gb * 1e9:
                out[layout] = "skipped: %.1f GB of tensors > --npz-max-gb" % (total / 1e9)
                continue
            path, t_save, p_save = traced(lambda: checkpoint.save_npz(d, m))
        nbytes = dir_bytes(path)
        if layout == "sharded":
            _, t_restore, p_restore = traced(lambda: checkpoint.restore(path, [m]))
        else:
            _, t_restore, p_restore = traced(lambda: checkpoint.restore_npz(path, m))
        same = (state(m) == before) if args.check else None
        out[layout] = dict(bytes=nbytes, save_s=round(t_save, 3), restore_s=round(t_restore, 3),
                           save_gbps_per_rank=round(nbytes / t_save / 1e9, 3), restore_gbps_per_rank=round(nbytes / t_restore / 1e9, 3),
                           save_peak_traced_bytes=p_save, restore_peak_traced_bytes=p_restore, restored_bytes_equal=same)
        shutil.rmtree(d, ignore_errors=True)
    m.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--placements", default="hbm,host,cache")
    ap.add_argument("--cache-bytes", type=int, default=1 << 30)
    ap.add_argument("--scale", type=float, default=0.1, help="multiplies every table's rows (1.0: the full single-GPU shapes)")
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--host-min-rows", type=int, default=100_000)
    ap.add_argument("--npz-max-gb", type=float, default=8.0)
    ap.add_argument("--no-check", dest="check", action="store_false", help="skip the byte comparison after each restore")
    ap.add_argument("--dir", default=None, help="where checkpoints are written (default: a temporary directory)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    root = tempfile.mkdtemp(prefix="wd_ckpt_bench_", dir=args.dir)
    res = dict(card=gpu_info(), chunk_bytes=None, results=[])
    try:
        from wide_deep_b200 import checkpoint
        res["chunk_bytes"] = checkpoint.CHUNK_BYTES
        for name in args.workloads.split(","):
            for placement in args.placements.split(","):
                r = run(name, placement, args, root)
                print(json.dumps(dict(r, card=res["card"])), flush=True)
                res["results"].append(r)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
