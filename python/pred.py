#!/usr/bin/env python
"""Prediction entry point — drop-in for the reference's python/pred.py (reference pred.py:52-74).
Multi-GPU: `torchrun --nproc-per-node G pred.py ...` runs the forward with the checkpoint's large tables row-sharded over the G
ranks, each rank on lines r, r + G, ... (--batch_size per rank); rank 0 prints every prediction in file order.
WD_SHARD_SAME_GPU=1 puts every rank on cuda:0 (a test setup)."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wide_deep_b200.config import Config  # noqa: E402
from wide_deep_b200.dataset import input_fn  # noqa: E402
from wide_deep_b200.estimator import build_estimator  # noqa: E402
from train import distributed_env  # noqa: E402

CONF = Config()
CONFIG = CONF.train
parser = argparse.ArgumentParser(description="Wide and Deep Model Prediction")
parser.add_argument("--model_dir", type=str, default=CONFIG["model_dir"])
parser.add_argument("--model_type", type=str, default=CONFIG["model_type"])
parser.add_argument("--data_dir", type=str, default="../data/pred")
parser.add_argument("--image_data_dir", type=str, default=None)
parser.add_argument("--batch_size", type=int, default=CONFIG["batch_size"])
parser.add_argument("--checkpoint_path", type=str, default=CONFIG["checkpoint_path"])

def main():
    rank, world, local = distributed_env()
    kw = {}
    if world > 1:                                      # gloo for plumbing only (IPC handles, the gather of the logits to rank 0)
        import torch
        import torch.distributed as dist
        kw["device"] = 0 if os.environ.get("WD_SHARD_SAME_GPU") else local
        torch.cuda.set_device(kw["device"])
        dist.init_process_group("gloo")
    model_dir = os.path.join(FLAGS.model_dir, FLAGS.model_type)
    model = build_estimator(model_dir, FLAGS.model_type, config=CONF, max_batch=FLAGS.batch_size, shard_world=world, shard_rank=rank, **kw)
    preds = model.predict(input_fn=lambda: input_fn(FLAGS.data_dir, None, "pred", FLAGS.batch_size, config=CONF, plan=model.plan,
                                                    rank=rank, world=world, keep_tail=world > 1),
                          checkpoint_path=FLAGS.checkpoint_path)
    for pred_dict in preds:                            # (a collective with world > 1: every rank drains it, rank 0 alone yields)
        cid = int(pred_dict["class_ids"][0])
        print("Prediction is \"{}\" ({:.1f}%)".format(cid, 100 * float(pred_dict["probabilities"][cid])))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    FLAGS, unparsed = parser.parse_known_args()
    main()
