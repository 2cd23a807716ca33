#!/usr/bin/env python
"""Training entry point — drop-in for the reference's python/train.py (same flags, same loops).

  python train.py [--model_dir --model_type --train_epochs --epochs_per_eval --batch_size --train_data
                   --eval_data --test_data --keep_train ...]        (run from the python/ directory)

Loop semantics follow reference python/train.py:65-164: `dynamic_train` (train on file i, evaluate on file
i+1), `train_and_eval`, `train`; the model directory is wiped unless --keep_train (train.py:188-191).
Multi-GPU: `torchrun --nproc-per-node G train.py ...` (main_distributed below): every rank trains on its shard of each file
(dataset.shard semantics) with synchronous, exact steps over row-sharded tables (wide_deep_b200/sharded.py) instead of the
reference's asynchronous parameter servers (train.py:197-217); train only, as in the reference.
"""
import argparse
import os
import shutil
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wide_deep_b200.config import Config  # noqa: E402
from wide_deep_b200.dataset import input_fn, list_files  # noqa: E402
from wide_deep_b200.estimator import build_custom_estimator  # noqa: E402

CONF = Config()
CONFIG = CONF.train
parser = argparse.ArgumentParser(description="Train Wide and Deep Model.")
parser.add_argument("--model_dir", type=str, default=CONFIG["model_dir"], help="Base directory for the model.")
parser.add_argument("--model_type", type=str, default=CONFIG["model_type"], help="Valid model types: {'wide', 'deep', 'wide_deep'}.")
parser.add_argument("--train_epochs", type=int, default=CONFIG["train_epochs"], help="Number of training epochs.")
parser.add_argument("--epochs_per_eval", type=int, default=CONFIG["epochs_per_eval"], help="The number of training epochs to run between evaluations.")
parser.add_argument("--batch_size", type=int, default=CONFIG["batch_size"], help="Number of examples per batch.")
parser.add_argument("--train_data", type=str, default=CONFIG["train_data"], help="Path to the train data.")
parser.add_argument("--eval_data", type=str, default=CONFIG["eval_data"], help="Path to the validation data.")
parser.add_argument("--test_data", type=str, default=CONFIG["test_data"], help="Path to the test data.")
parser.add_argument("--image_train_data", type=str, default=CONFIG.get("image_train_data"))
parser.add_argument("--image_eval_data", type=str, default=CONFIG.get("image_eval_data"))
parser.add_argument("--image_test_data", type=str, default=CONFIG.get("image_test_data"))
parser.add_argument("--keep_train", type=int, default=CONFIG["keep_train"], help="Whether to keep training on previous trained model.")


def elapse_time(t0):
    return round((time.time() - t0) / 60, 2)


def _fn(model, path, mode):
    return lambda: input_fn(path, None, mode, FLAGS.batch_size, config=CONF, plan=model.plan, device_parse=True)


def _show(results):
    print("-" * 80)
    for key in sorted(results):
        print("{}: {}".format(key, results[key]))


def train_and_eval(model):
    for n in range(FLAGS.train_epochs):
        print("INFO: " + "=" * 30 + " START EPOCH {} ".format(n + 1) + "=" * 30 + "\n")
        for f in list_files(FLAGS.train_data):
            t0 = time.time()
            print("INFO: <EPOCH {}>: Start training {}".format(n + 1, f))
            model.train(input_fn=_fn(model, f, "train"))
            print("INFO: <EPOCH {}>: Finish training {}, take {} mins".format(n + 1, f, elapse_time(t0)))
            print("-" * 80)
            print("INFO: <EPOCH {}>: Start evaluating {}".format(n + 1, FLAGS.eval_data))
            t0 = time.time()
            results = model.evaluate(input_fn=_fn(model, FLAGS.eval_data, "eval"))
            print("INFO: <EPOCH {}>: Finish evaluation {}, take {} mins".format(n + 1, FLAGS.eval_data, elapse_time(t0)))
            _show(results)
        if (n + 1) % FLAGS.epochs_per_eval == 0:
            print("INFO: <EPOCH {}>: Start testing {}".format(n + 1, FLAGS.test_data))
            t0 = time.time()
            # the reference passes mode 'pred' here (train.py:96-101, quirk Q10), which cannot be evaluated; use 'eval'
            results = model.evaluate(input_fn=_fn(model, FLAGS.test_data, "eval"))
            print("INFO: <EPOCH {}>: Finish testing {}, take {} mins".format(n + 1, FLAGS.test_data, elapse_time(t0)))
            _show(results)


def dynamic_train(model):
    data_files = list_files(FLAGS.train_data)
    data_files.sort()
    assert len(data_files) > 1, "Dynamic train mode need more than 1 data file"
    for i in range(len(data_files) - 1):
        train_data, test_data = data_files[i], data_files[i + 1]
        print("INFO: " + "=" * 30 + " START TRAINING DATA: {} ".format(train_data) + "=" * 30 + "\n")
        for n in range(FLAGS.train_epochs):
            t0 = time.time()
            print("INFO: START TRAIN DATA <{}> <EPOCH {}>".format(train_data, n + 1))
            model.train(input_fn=_fn(model, train_data, "train"))
            print("INFO: FINISH TRAIN DATA <{}> <EPOCH {}> take {} mins".format(train_data, n + 1, elapse_time(t0)))
            print("-" * 80)
            print("INFO: START EVALUATE TEST DATA <{}> <EPOCH {}>".format(test_data, n + 1))
            t0 = time.time()
            results = model.evaluate(input_fn=_fn(model, test_data, "eval"))
            print("INFO: FINISH EVALUATE TEST DATA <{}> <EPOCH {}>: take {} mins".format(test_data, n + 1, elapse_time(t0)))
            _show(results)


def train(model):
    for n in range(FLAGS.train_epochs):
        print("INFO: " + "=" * 30 + " START EPOCH {} ".format(n + 1) + "=" * 30 + "\n")
        for f in list_files(FLAGS.train_data):
            t0 = time.time()
            print("INFO: <EPOCH {}>: Start training {}".format(n + 1, f))
            model.train(input_fn=_fn(model, f, "train"))
            print("INFO: <EPOCH {}>: Finish training {}, take {} mins".format(n + 1, f, elapse_time(t0)))


def distributed_env():
    """(rank, world, local_rank) when launched by torchrun / torch.distributed.run, else (0, 1, 0).  Counterpart of the reference's
    `distribution` block (conf/train.yaml, python/train.py:201-217): workers there, ranks here; no parameter servers."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return 0, 1, 0
    return int(os.environ["RANK"]), world, int(os.environ.get("LOCAL_RANK", "0"))


def main():
    rank, world, local = distributed_env()
    if world > 1:
        return main_distributed(rank, world, local)
    print("Using wide_deep_b200 (CUDA sm_90a) in place of TensorFlow")
    print("\nModel Type: {}".format(FLAGS.model_type))
    model_dir = os.path.join(FLAGS.model_dir, FLAGS.model_type)
    print("\nModel Directory: {}".format(model_dir))
    print("\nUsing Train Config:")
    for k, v in CONF.train.items():
        print("{}: {}".format(k, v))
    print("\nUsing Model Config:")
    for k, v in CONF.model.items():
        print("{}: {}".format(k, v))
    if not FLAGS.keep_train:
        shutil.rmtree(model_dir, ignore_errors=True)
        print("Remove model directory: {}".format(model_dir))
    model = build_custom_estimator(model_dir, FLAGS.model_type, config=CONF, max_batch=FLAGS.batch_size)
    print("INFO: Build estimator: {}".format(model))
    if CONF.train["dynamic_train"]:
        print("Using dynamic train mode.")
        dynamic_train(model)
    else:
        train_and_eval(model)


def main_distributed(rank, world, local):
    """torchrun --nproc-per-node G train.py ...: rank r trains on every G-th line of each file (dataset.shard semantics, reference
    python/lib/dataset.py:173-174) with synchronous, exact steps; tables larger than 16384 rows are row-sharded over the ranks
    (the reference partitions them over its parameter servers, python/lib/joint.py:141-143).  As in the reference, distributed
    runs train only ("distributed can not including eval", python/train.py:215-216); rank 0 alone touches the model directory and
    writes the TensorBoard summaries (those of the global batch).  WD_SHARD_SAME_GPU=1 puts every rank on cuda:0 (a test setup, not
    a multi-GPU rate)."""
    import torch
    import torch.distributed as dist
    device = 0 if os.environ.get("WD_SHARD_SAME_GPU") else local
    torch.cuda.set_device(device)
    dist.init_process_group("gloo")                    # plumbing only (IPC handles, checkpoint gather); data moves over NVLink
    log = print if rank == 0 else (lambda *a, **k: None)
    log("Using wide_deep_b200 (CUDA sm_90a) in place of TensorFlow: rank {} of {}".format(rank, world))
    model_dir = os.path.join(FLAGS.model_dir, FLAGS.model_type)
    if not FLAGS.keep_train and rank == 0:
        shutil.rmtree(model_dir, ignore_errors=True)
        log("Remove model directory: {}".format(model_dir))
    dist.barrier()
    model = build_custom_estimator(model_dir, FLAGS.model_type, config=CONF, max_batch=FLAGS.batch_size, device=device,
                                   shard_world=world, shard_rank=rank)
    log("INFO: Build estimator: {}".format(model))
    for n in range(FLAGS.train_epochs):
        log("INFO: " + "=" * 30 + " START EPOCH {} ".format(n + 1) + "=" * 30 + "\n")
        for f in list_files(FLAGS.train_data):
            t0 = time.time()
            log("INFO: <EPOCH {}>: Start training {}".format(n + 1, f))
            model.train(input_fn=lambda f=f: input_fn(f, None, "train", FLAGS.batch_size, config=CONF, plan=model.plan, rank=rank, world=world, device_parse=True))
            log("INFO: <EPOCH {}>: Finish training {}, take {} mins".format(n + 1, f, elapse_time(t0)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    FLAGS, unparsed = parser.parse_known_args()
    main()
