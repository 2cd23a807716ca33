"""Each GEMM engine allocates only the operand copies it reads (the operand-family table at the top of csrc/mlp.cu).

The fp32 family (ffma, tc1x, tc3x) keeps fp32 activations, their transposed copies and the transposed / tf32-split weights; the
bf16 family (bf16x3) keeps bf16 hi / lo copies instead.  The engines of one family must allocate the same HBM, and bf16x3 must
allocate exactly the fp32 family's bytes minus its fp32-only buffers plus its bf16-only ones, computed here from the plan's shapes.
"""
import pytest

from tests import kernel_ref as KR
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

F32, BF16 = 4, 2


def pad(n, m):
    return (n + m - 1) // m * m


def family_bytes(plan):
    """(bytes only the fp32 family allocates, bytes only the bf16 family allocates) for the plan's deep towers."""
    bp = pad(plan.max_batch, 128)
    own_a = plan.batch_norm or plan.dropout > 0.0         # post-activation values kept apart from the layer output
    fp32_only = bp * plan.d0_phys * F32                     # X0T
    bf16_only = 2 * bp * plan.d0_phys * BF16               # X0 hi / lo
    wt = 0
    for tw in plan.towers:
        hu = tw["hidden"]
        srcs = plan.layer_sources(tw["mode"], len(hu))
        n_phys = [pad(plan.out_width(h), 32) for h in hu]
        for l in range(len(hu)):
            wt += sum(plan.d0_phys if s == "x" else n_phys[s] for s in srcs[l]) * n_phys[l]
            n = bp * n_phys[l]
            fp32_only += 3 * n * F32                        # HT, dZ, dZT
            if own_a and l not in srcs[-1]:
                fp32_only += n * F32                        # H: the bf16 family keeps it only where the logits layer reads it
            bf16_only += 4 * n * BF16                       # H and dZ hi / lo
    fp32_only += 5 * wt * F32                               # Wt and the tf32 hi / lo splits of W and Wt
    bf16_only += 2 * wt * BF16                              # W hi / lo
    return fp32_only, bf16_only


@pytest.mark.parametrize("hidden,mode,bn,dropout", [
    ((129, 33, 8), "first_dense", 1, 0.0),
    ([(96, 40), (64,)], "resnet", 0, 0.0),
    ((200, 48), "dense", 0, 0.25),
])
def test_bf16_family_allocates_only_its_copies(hidden, mode, bn, dropout):
    fc, cross, model = KR.parity_conf(hidden, mode=mode, bn=bn, dropout=dropout)
    used = {}
    for engine in ("ffma", "tc1x", "tc3x", "bf16x3"):
        plan = Plan(fc, cross, model, "wide_deep", max_batch=300, embedding_dim_override=8, max_nnz=300 * 40, max_keys=300 * 40,
                    gemm_engine=engine)
        pm = WideDeepModel(plan)
        used[engine] = pm.memory_usage()[0]
        del pm
    assert used["ffma"] == used["tc1x"] == used["tc3x"], used
    fp32_only, bf16_only = family_bytes(plan)
    assert used["tc3x"] - used["bf16x3"] == fp32_only - bf16_only, (used, fp32_only, bf16_only)
