"""Results of the 3xBF16 GEMM engine (csrc/gemm_bf16.cu) held bit for bit, and its tile-schedule edges.

Every output element of the engine gets one fixed wgmma sequence (m64n128k16, ascending k-steps, lo*hi + hi*lo + hi*hi into one
fp32 accumulator), so which CTA or warp group computes a tile must never change a bit of what a step trains.  The trained
tensors of four small models are held to SHA-256 digests recorded on an H100 80GB HBM3, and the edges of the tile schedule
(odd tile counts, B = 1, fewer tiles than SMs, weight-gradient splits without k-blocks, multi-segment inputs) go through the
float64 criteria of tests/kernel_ref.py.  `python -m tests.test_gpu_gemm_schedule` prints the digests of the current build."""
import hashlib

import numpy as np
import pytest

from tests import kernel_ref as KR
from tests.test_gpu_kernel_parity import build, probe
from tests.helpers import to_product_batch
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

SGD = "tf.train.GradientDescentOptimizer(learning_rate=0.05)"
# name -> (hidden units, connection mode, wide deep input, max_batch, batch sizes of the three steps)
CASES = {
    "odd_row_tiles": ((129, 33, 8), "simple", False, 2100, (300, 1, 200)),
    "wide_partial": ((257, 200, 520, 100), "dense", True, 1024, (129, 300, 1000)),
    "seven_segments": ((24, 24, 24, 24, 24, 24, 24), "dense", False, 512, (200, 511, 64)),
    "empty_wgrad_splits": ((100,), "resnet", False, 16384, (300, 1, 2049)),
}
DIGESTS = {
    "odd_row_tiles": "a6e62abb21d8f94f4037ebdfc848eebc537f9c76863b7890dc99fd018be5454d",
    "wide_partial": "dea3edd5f72ac0ce2fe3e890ab7b0f270ce015a4abda860da7a44567ba022a4f",
    "seven_segments": "97df8b8e953cba411d8ebb5fcea4d46a1b72037bb94ea1c4e1c38c532adf1bbd",
    "empty_wgrad_splits": "182b7e24a6a771082ae09e508d5e0e1fb2619b13bbef39a1ed1928274b668482",
}


def trained_digest(name):
    """SHA-256 of the three losses and of every trained tensor (sorted by name, float32 bytes) after three SGD steps."""
    hidden, mode, wide_input, max_batch, sizes = CASES[name]
    fc, cross, model = KR.parity_conf(hidden, mode=mode, opt=SGD)
    emb = 64 if wide_input else 8
    plan = Plan(fc, cross, model, "wide_deep", max_batch=max_batch, embedding_dim_override=emb, max_nnz=max_batch * 40,
                max_keys=max_batch * 40, gemm_engine="bf16x3")
    pm = WideDeepModel(plan)
    rng = np.random.default_rng(sorted(CASES).index(name) + 100)
    for n, v in KR.random_params([(n, s[3]) for n, s in plan.tensor_names.items()], rng, plan.activation).items():
        pm.set_tensor(n, v)
    h = hashlib.sha256()
    for B in sizes:
        raw = KR.raw_batch(B, rng)
        loss = pm.train_step(to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32)))
        h.update(np.float32(loss).tobytes())
    for n in sorted(plan.tensor_names):
        h.update(n.encode())
        h.update(np.ascontiguousarray(pm.get_tensor(n), dtype=np.float32).tobytes())
    assert pm.gemm_fallback_count() == 0
    return h.hexdigest()


@pytest.mark.parametrize("name", sorted(CASES))
def test_trained_tensors_match_recorded_digest(name):
    assert trained_digest(name) == DIGESTS[name]


def test_odd_tile_counts_and_b1():
    """B = 300, 1300 and 200 give 3, 11 and 2 row tiles, B = 1 one row tile; widths 129 and 33 give 2 and 1 column tiles, and
    the first weight gradient has one row tile (K = 32)."""
    plan, pm = build("bf16x3", (129, 33, 8))
    rng = np.random.default_rng(21)
    for B in (300, 1, 200, 1300):
        probe("bf16x3", plan, pm, B, rng)


def test_seven_segment_input():
    """dense mode over seven hidden layers: the last one reads 7 input segments, the most a hidden layer can have (the logits
    layer then reads kMaxSegs = 8)."""
    plan, pm = build("bf16x3", (24,) * 7, mode="dense", max_batch=512)
    probe("bf16x3", plan, pm, 300, np.random.default_rng(22))


def test_fewer_tile_pairs_than_clusters_and_empty_splits():
    """max_batch 16384 gives 32 weight-gradient splits of which B = 300 fills one; every GEMM has fewer tiles than the GPU has
    SMs."""
    plan, pm = build("bf16x3", (100, 40), max_batch=16384)
    rng = np.random.default_rng(23)
    for B in (300, 1):
        probe("bf16x3", plan, pm, B, rng)


if __name__ == "__main__":
    for name in sorted(CASES):
        print('    "%s": "%s",' % (name, trained_digest(name)))
