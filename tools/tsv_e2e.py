#!/usr/bin/env python
"""End to end FROM TSV BYTES (the product input path, not a bench.py line): lines/s of `estimator.train` over the bundled
training files repeated R times, for both input paths, next to each pipeline alone and the train step alone:

  host    file bytes -> wd_tsv_parse_lines (C++ worker threads, pinned ring) -> prefetch thread -> wd_batch_prefetch_slot
  device  file bytes -> wd_tsv_gather_lines (pinned text ring) -> prefetch thread -> wd_tsv_parse_slot (H2D of the text, parse
          and hash on the GPU into the slot, beside the running step)

then wd_train_step_slot, loss read every step.  The two arms run alternately (--rounds times each, best kept) in one process,
and the card's name and power limit are read in the same run.

    python tools/tsv_e2e.py [--repeat 40] [--batch 2048 8192] [--rounds 2] [--model_type wide_deep] [--arms host device]

The bundled configuration (conf/*.yaml: 43 raw fields, 20 string crosses, towers 1024-512-256) is the reference's own; the
synthetic Criteo workload of bench.py has no text form, so this is the only number that includes parsing + hashing."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from wide_deep_b200.config import Config  # noqa: E402
from wide_deep_b200.dataset import input_fn, list_files  # noqa: E402
from wide_deep_b200.estimator import build_custom_estimator  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(path, batch, args, cfg, tmp):
    est = build_custom_estimator(os.path.join(tmp, "model%d" % batch), args.model_type, config=cfg, max_batch=batch)
    m = est._ensure_model()

    def fn(arm, **kw):
        if arm == "device":
            return lambda: input_fn(path, None, "train", batch, config=cfg, plan=est.plan, device_parse=True, **kw)
        return lambda: input_fn(path, None, "train", batch, config=cfg, plan=est.plan, pinned=True, **kw)

    def pipeline(arm):                    # read + index + shuffle + parse / hash into a slot, no step
        t0 = time.time()
        for i, item in enumerate(fn(arm)()):
            m.feed_slot(i % 2, item)
        m.sync()
        return time.time() - t0

    def e2e(arm):
        t0 = time.time()
        est.train(input_fn=fn(arm))
        return time.time() - t0

    for arm in args.arms:                 # warm-up: graph captures, first launches of the parser kernels
        print("batch %d: warm-up, %s arm" % (batch, arm), file=sys.stderr, flush=True)
        est.train(input_fn=fn(arm), steps=12)
    save, est.save = est.save, (lambda: None)          # the end-of-pass checkpoint (all tables -> npz) is not input-path work
    res = {a: {"pipeline": [], "e2e": []} for a in args.arms}
    for _ in range(args.rounds):
        for arm in args.arms:
            print("batch %d: timed pipeline and e2e, %s arm" % (batch, arm), file=sys.stderr, flush=True)
            res[arm]["pipeline"].append(pipeline(arm))
            res[arm]["e2e"].append(e2e(arm))
    est.save = save
    stats = m.tsv_parse_stats()
    # the train step alone on one resident batch
    b = next(iter(input_fn(path, None, "train", batch, config=cfg, plan=est.plan)))
    m.upload_slot(0, b)
    for _ in range(5):
        m.train_step_slot(0, want_loss=False)
    m.sync()
    t0 = time.time()
    for _ in range(50):
        m.train_step_slot(0, want_loss=False)
    m.sync()
    t_step = (time.time() - t0) / 50
    return res, stats, t_step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=40)
    ap.add_argument("--batch", type=int, nargs="+", default=[2048, 8192])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--model_type", default="wide_deep")
    ap.add_argument("--arms", nargs="+", default=["host", "device"], choices=["host", "device"])
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    cfg = Config()
    run = cfg.runconfig
    run["save_checkpoints_steps"], run["save_checkpoints_secs"] = None, 10 ** 9          # no checkpoint inside the timed pass
    src = b"".join(open(f, "rb").read() for f in list_files(os.path.join(ROOT, "data", "train")))
    gpu = card()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "train.tsv")
        with open(path, "wb") as fh:
            for _ in range(args.repeat):
                fh.write(src)
        n_lines = src.count(b"\n") * args.repeat
        nbytes = len(src) * args.repeat
        for batch in args.batch:
            res, stats, t_step = measure(path, batch, args, cfg, tmp)
            line = {"gpu": gpu, "lines": n_lines, "mbytes": round(nbytes / 1e6, 1), "batch": batch,
                    "step_only_lines_per_s": round(batch / t_step), "device_parsed_batches": stats["device"],
                    "host_fallback_batches": stats["host"]}
            for arm, r in res.items():
                line["%s_pipeline_lines_per_s" % arm] = round(n_lines / min(r["pipeline"]))
                line["%s_e2e_lines_per_s" % arm] = round(n_lines / min(r["e2e"]))
                line["%s_e2e_lines_per_s_all" % arm] = [round(n_lines / t) for t in r["e2e"]]
            line["note"] = ("pipeline = read file + line index + shuffle + parse/hash into a batch slot (no step); e2e = pipeline + train "
                            "step + loss readback every step; best of %d alternated rounds; no checkpoint inside the timed pass" % args.rounds)
            print(json.dumps(line), flush=True)
            if args.out:
                with open(args.out, "a") as fh:
                    fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
