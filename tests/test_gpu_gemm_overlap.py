"""Results of the 3xBF16 GEMM engine (csrc/gemm_bf16.cu) held bit for bit where a CTA runs several tiles in a row.

A schedule that carries work from one tile into the next (an epilogue under the next main loop, a second accumulator set)
must not change a bit, and the small models of tests/test_gpu_gemm_schedule.py give each CTA one or two tiles only.  These cases
give CTAs 3 and 4 tiles (B = 8192 and 8064 on 1024-wide layers: 512 and 504 tiles over 132 SMs), 1 and 2 tiles (the 512- and
256-wide layers), layers with one k-block (K = 32 and 64), with 5 and 8, and with more than 16 (dense layers over 224 + 1024
and 224 + 1024 + 512 physical inputs: 20 and 28), a partial column tile (N = 320), the non-relu epilogue (tanh), and
weight-gradient splits without k-blocks behind splits with them (B = 300).  Each case's trained tensors after three SGD steps
are held to a SHA-256 digest recorded on an H100 80GB HBM3.  `python -m tests.test_gpu_gemm_overlap` prints the digests of
the current build."""
import hashlib

import numpy as np
import pytest

from tests import kernel_ref as KR
from tests.helpers import to_product_batch
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

SGD = "tf.train.GradientDescentOptimizer(learning_rate=0.05)"
# name -> (hidden units, connection mode, activation, wide deep input, batch sizes of the three steps); max_batch 8192
CASES = {
    "simple_relu": ((1024, 512, 256), "simple", "relu", False, (8192, 8064, 8192)),
    "dense_tanh": ((1024, 512, 256), "dense", "tanh", True, (8064, 300, 8192)),
    "k64_partial_n": ((64, 1024, 320, 256), "simple", "relu", False, (8192, 300, 8064)),
}
DIGESTS = {
    "dense_tanh": "ea1400ef8185f3543a150f7c6391fb5e2b2ec9124e1526f822429f60eb6aa1d6",
    "k64_partial_n": "bba881c141c4530160c127ab2d3c05f5272635e338bec339ee7128192c39b092",
    "simple_relu": "7846efc3192b32975c3509b75f389f746a3519217706d24e48a10b54ac668269",
}


def trained_digest(name):
    """SHA-256 of the three losses and of every trained tensor (sorted by name, float32 bytes) after three SGD steps."""
    hidden, mode, act, wide_input, sizes = CASES[name]
    fc, cross, model = KR.parity_conf(hidden, mode=mode, act=act, opt=SGD)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=8192, embedding_dim_override=64 if wide_input else 8,
                max_nnz=8192 * 40, max_keys=8192 * 40, gemm_engine="bf16x3")
    pm = WideDeepModel(plan)
    rng = np.random.default_rng(sorted(CASES).index(name) + 200)
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


if __name__ == "__main__":
    for name in sorted(CASES):
        print('    "%s": "%s",' % (name, trained_digest(name)))
