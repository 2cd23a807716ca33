#!/usr/bin/env python
"""Evaluation entry point — drop-in for the reference's python/eval.py (same flags; prints the sorted metric
dict, reference eval.py:56-83).  Evaluates what train.py wrote under <model_dir>/<model_type>.
Multi-GPU: `torchrun --nproc-per-node G eval.py ...` (main_distributed below) evaluates the checkpoint with its large tables
row-sharded over the G ranks; --batch_size is then per rank."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wide_deep_b200.config import Config  # noqa: E402
from wide_deep_b200.dataset import input_fn  # noqa: E402
from wide_deep_b200.estimator import build_estimator  # noqa: E402
from train import distributed_env  # noqa: E402

CONF = Config()
CONFIG = CONF.train
parser = argparse.ArgumentParser(description="Evaluate Wide and Deep Model.")
parser.add_argument("--model_dir", type=str, default=CONFIG["model_dir"], help="Model checkpoint dir for evaluating.")
parser.add_argument("--model_type", type=str, default=CONFIG["model_type"], help="Valid model types: {'wide', 'deep', 'wide_deep'}.")
parser.add_argument("--test_data", type=str, default=CONFIG["test_data"], help="Evaluating data dir.")
parser.add_argument("--image_test_data", type=str, default=CONFIG.get("image_test_data"))
parser.add_argument("--batch_size", type=int, default=CONFIG["batch_size"], help="Number of examples per batch.")
parser.add_argument("--checkpoint_path", type=str, default=CONFIG["checkpoint_path"],
                    help="Path of a specific checkpoint to evaluate. If None, the latest checkpoint in model_dir is used.")


def evaluate(log, rank=0, world=1, **kw):
    log("Model type: {}".format(FLAGS.model_type))
    model_dir = os.path.join(FLAGS.model_dir, FLAGS.model_type)
    log("Model directory: {}".format(model_dir))
    model = build_estimator(model_dir, FLAGS.model_type, config=CONF, max_batch=FLAGS.batch_size, shard_world=world, shard_rank=rank, **kw)
    if not (FLAGS.checkpoint_path or model.latest_checkpoint()):
        raise ValueError("No model checkpoint found, please check the model dir.")
    log("INFO: " + "=" * 30 + " START TESTING" + "=" * 30)
    s_time = time.time()
    results = model.evaluate(input_fn=lambda: input_fn(FLAGS.test_data, None, "eval", FLAGS.batch_size, config=CONF, plan=model.plan,
                                                       rank=rank, world=world, keep_tail=world > 1, device_parse=True),
                             checkpoint_path=FLAGS.checkpoint_path)
    log("INFO: " + "=" * 30 + "FINISH TESTING, TAKE {} mins".format(round((time.time() - s_time) / 60, 2)) + "=" * 30)
    log("-" * 80)
    for key in sorted(results):
        log("%s: %s" % (key, results[key]))


def main():
    rank, world, local = distributed_env()
    if world > 1:
        return main_distributed(rank, world, local)
    print("Using wide_deep_b200 (CUDA sm_90a) in place of TensorFlow")
    evaluate(print)


def main_distributed(rank, world, local):
    """torchrun --nproc-per-node G eval.py ...: the checkpoint's tables larger than 16384 rows are row-sharded over the G ranks (as
    train.py's distributed mode trains them), rank r evaluates lines r, r + G, ... of the data, and one collective sums the
    metrics of all ranks; rank 0 alone prints.  The metrics equal a single process's with a batch of G x --batch_size lines.
    WD_SHARD_SAME_GPU=1 puts every rank on cuda:0 (a test setup, not a multi-GPU rate)."""
    import torch
    import torch.distributed as dist
    device = 0 if os.environ.get("WD_SHARD_SAME_GPU") else local
    torch.cuda.set_device(device)
    dist.init_process_group("gloo")                    # plumbing only (IPC handles); metrics are summed over NVLink
    log = print if rank == 0 else (lambda *a, **k: None)
    log("Using wide_deep_b200 (CUDA sm_90a) in place of TensorFlow: rank {} of {}".format(rank, world))
    evaluate(log, rank, world, device=device)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    FLAGS, unparsed = parser.parse_known_args()
    main()
