"""The two drivers of a row-sharded step run the same rank-step (shard.cu shard_step): multi-process ranks run it whole, under flag
barriers and graph replay; ranks of one process (LocalShardGroup) run it segment by segment, with wd_shard_local_sync between the
segments.  On the same plan, parameters and batches they must agree byte for byte — losses, logits, eval metrics, every tensor and
optimizer slot — and launch the same kernels, but for the multi-process driver's barrier kernels.  Two processes share cuda:0
(tests/_shard_drivers_worker.py), so this runs on a single-GPU box."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("plan", ["wide_deep-adagrad-ftrl-host", "deep-adam"])
def test_shard_drivers_bit_identical(plan):
    """wide_deep-adagrad-ftrl-host: both table spaces sharded, h2_embedding's shards in host memory, rows of more than kChunk
    occurrences; deep-adam: Adam / Adam, every shard in HBM.  6 train steps (multi-process: eager, eager, capture, replay x 3),
    then a forward and an evaluation."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29677", os.path.join(ROOT, "tests", "_shard_drivers_worker.py"), plan]
    env = dict(os.environ)
    env.pop("WD_SHARD_TRACE", None)                    # (its stamp kernels would count as launches)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0 and "SHARD_DRIVERS_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
