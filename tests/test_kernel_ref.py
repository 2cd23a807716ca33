"""CPU self-tests of the float64 kernel checker (tests/kernel_ref.py): emulated healthy engines pass both criteria at the layer shapes
of the GPU matrix, emulated defects fail them, the derivative-from-a formulas match the oracle's derivative-from-z, and the
reference backward restates the oracle's gradients."""
import numpy as np
import pytest

from oracle import model as OM
from tests import kernel_ref as KR

# Criterion-2 bounds predicted by the emulation: 4x the worst tile of test_emulated_engines_pass (ffma and tc3x 3.9e-7 = 2^-21.3,
# bf16x3 6.0e-6 = 2^-17.3).  tests/test_gpu_kernel_parity.py sets its own from the H100 and compares them with these.
TAU_PRED = {"ffma": 1.6e-6, "tc3x": 1.6e-6, "bf16x3": 2.4e-5}
KBLOCK = {"tc3x": 32, "bf16x3": 64}
WIDTHS = [1, 8, 33, 100, 129, 200, 257, 520, 400]


def _operands(rng, M, K, N):
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = (rng.uniform(-1, 1, size=(K, N)) * np.sqrt(6.0 / (K + N))).astype(np.float32)
    return a, b


def _ref(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return a @ b, np.abs(a) @ np.abs(b), np.sqrt((a * a) @ (b * b))


def _check(got, a, b, engine, name="gemm"):
    ref, M, R = _ref(a, b)
    return KR.compare(name, got, ref, M, R, KR.c_gemm(engine, a.shape[1]))


@pytest.mark.parametrize("engine", ["ffma", "tc3x", "bf16x3"])
@pytest.mark.parametrize("K", [32, 192])
def test_emulated_engines_pass(engine, K):
    """Forward GEMMs of every hidden width of the matrix (B = 300) and a weight gradient reduced over B = 2100 rows."""
    rng = np.random.default_rng(K)
    worst = 0.0
    for N in WIDTHS:
        a, b = _operands(rng, 300, K, N)
        c = _check(KR.emulated_gemm(a, b, engine), a, b, engine, "fwd N=%d" % N)
        assert c.worst1 <= 1.0 and c.worst2 <= TAU_PRED[engine], c
        worst = max(worst, c.worst2)
    x, dz = rng.standard_normal((2100, K)).astype(np.float32), rng.standard_normal((2100, 129)).astype(np.float32)
    c = _check(KR.emulated_gemm(x.T, dz, engine), x.T, dz, engine, "wgrad")
    assert c.worst1 <= 1.0 and c.worst2 <= TAU_PRED[engine], c
    print("%s K=%d: worst tile %.3g (2^%.1f)" % (engine, K, max(worst, c.worst2), np.log2(max(worst, c.worst2))))


@pytest.mark.parametrize("engine,bad", [("tc3x", "tf32"), ("bf16x3", "bf16"), ("bf16x3", "tf32")])
def test_single_pass_fails_by_8x(engine, bad):
    """A single-pass product (tc1x = tf32, or bf16) misses the three-pass engines' criterion 2 by at least 8x."""
    rng = np.random.default_rng(3)
    a, b = _operands(rng, 300, 192, 200)
    c = _check(KR.emulated_gemm(a, b, "tc3x" if bad == "tf32" else "bf16x3", single_pass=True), a, b, engine)
    assert c.worst2 >= 8 * TAU_PRED[engine], c


@pytest.mark.parametrize("engine", ["tc3x", "bf16x3"])
def test_missing_lohi_term_in_one_kblock_fails(engine):
    rng = np.random.default_rng(4)
    a, b = _operands(rng, 300, 192, 257)
    c = _check(KR.emulated_gemm(a, b, engine, drop_lohi_kblock=1, kblock=KBLOCK[engine]), a, b, engine)
    assert c.worst2 > TAU_PRED[engine], c


@pytest.mark.parametrize("engine", ["ffma", "tc3x", "bf16x3"])
@pytest.mark.parametrize("defect", ["drop_last_row", "stale_row"])
@pytest.mark.parametrize("B", [65, 300, 2100])
def test_weight_gradient_row_defects_fail(engine, defect, B):
    """Weight gradient x^T dz over the batch: leaving out the last row, or reducing one stale row of an earlier batch too."""
    rng = np.random.default_rng(B)
    x, dz = rng.standard_normal((B, 100)), rng.standard_normal((B, 129))
    if defect == "drop_last_row":
        got = KR.emulated_gemm(x[:-1].T, dz[:-1], engine)
    else:
        xs, ds = rng.standard_normal((B + 1, 100)), rng.standard_normal((B + 1, 129))
        xs[:B], ds[:B] = x, dz
        got = KR.emulated_gemm(xs.T, ds, engine)
    c = _check(got, x.T.astype(np.float32), dz.astype(np.float32), engine)
    assert c.worst1 > 1.0 or c.worst2 > TAU_PRED[engine], c
    assert c.worst2 > 8 * TAU_PRED[engine], c


@pytest.mark.parametrize("B", [129, 300, 2100])
def test_bias_partial_skipping_last_row_tile_fails(B):
    rng = np.random.default_rng(B)
    dz = rng.standard_normal((B, 200)).astype(np.float32)
    rts = (B + 127) // 128
    got = dz[:(rts - 1) * 128].sum(0, dtype=np.float32).astype(np.float64)
    d = dz.astype(np.float64)
    c = KR.compare("bias", got, d.sum(0), np.abs(d).sum(0), np.sqrt((d * d).sum(0)), KR.c_gemm("ffma", B))
    assert c.worst1 > 1.0 and c.worst2 > 8 * TAU_PRED["bf16x3"], c


def test_nan_fails_both_criteria():
    rng = np.random.default_rng(5)
    a, b = _operands(rng, 64, 32, 33)
    got = KR.emulated_gemm(a, b, "tc3x")
    got[63, 32] = np.nan
    c = _check(got, a, b, "tc3x")
    assert c.worst1 == np.inf and c.worst2 == np.inf and c.where1 == (63, 32) and c.tile2 == (0, 0)


@pytest.mark.parametrize("act", OM.ACTS if hasattr(OM, "ACTS") else
                         ["relu", "relu6", "sigmoid", "tanh", "leaky_relu", "elu", "selu", "softplus", "softsign", "crelu"])
def test_derivative_from_a_matches_oracle_derivative_from_z(act):
    rng = np.random.default_rng(6)
    z = np.concatenate([rng.standard_normal((200, 64)) * 3, rng.uniform(-8, 8, size=(200, 64))])
    if act == "crelu":
        a = OM.act_fwd(act, z)
        d = KR.act_bwd_from_a(act, a)
        u = z.shape[1]
        np.testing.assert_array_equal(d[:, :u], (z > 0).astype(np.float64))
        np.testing.assert_array_equal(d[:, u:], (z < 0).astype(np.float64))
        return
    a = OM.act_fwd(act, z)
    np.testing.assert_allclose(KR.act_bwd_from_a(act, a), OM.act_bwd(act, z, a), rtol=1e-9, atol=1e-12)


def test_rounding_helpers():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -9, -3.1415926], dtype=np.float32)
    np.testing.assert_array_equal(KR.bf16_round(x), np.array([1.0, 1.0, 1.0 + 4 * 2 ** -8, 1.0, -3.140625], dtype=np.float32))
    np.testing.assert_array_equal(KR.tf32_round(np.array([1.0 + 2 ** -11, 1.0 + 2 ** -12], dtype=np.float32)),
                                  np.array([1.0 + 2 ** -10, 1.0], dtype=np.float32))     # (a tie goes up; below half an ulp goes down)
    hi, lo = KR.split_hi_lo(x, KR.bf16_round)
    assert np.all(np.abs(x.astype(np.float64) - hi - lo) <= 2.0 ** -16 * np.abs(x))


# ---------------------------------------------------------------------------------------- the reference backward vs the oracle
class _OracleAsGpu(object):
    """Stands in for a WideDeepModel after a step: serves the oracle's forward values through the debug getters."""

    def __init__(self, plan, om, raw, cache):
        self.plan, self.om, self.cache, self.raw = plan, om, cache, raw
        self.B = cache["B"]
        ids = om.transform(raw)
        C = len(plan.columns)
        per = []
        for c in plan.columns:
            per.append(ids.get(c.name, (np.zeros(self.B + 1, dtype=np.int64), np.zeros(0, dtype=np.int64))))
        offs, flat = [0], []
        for b in range(self.B):
            for o, i in per:
                flat.extend(i[o[b]:o[b + 1]])
                offs.append(len(flat))
        self._offs, self._ids = np.array(offs, dtype=np.int32), np.array(flat, dtype=np.int64)
        assert len(self._offs) == self.B * C + 1

    def column_ids(self):
        return self._offs, self._ids

    def deep_input(self, B):
        X = np.zeros((B, self.plan.d0_phys))
        for name, (lo, po, w) in self.plan.deep_layout.items():
            X[:, po:po + w] = self.cache["X"][:, lo:lo + w]
        return X

    def hidden_output(self, t, l, B):
        h = self.cache["towers"][t]["H"][l]
        out = np.zeros((B, (h.shape[1] + 31) // 32 * 32))
        out[:, :h.shape[1]] = h
        return out


@pytest.mark.parametrize("mode,act,bn,dropout,hidden", [
    ("simple", "relu", 1, 0.0, (33, 8)),
    ("first_dense", "tanh", 1, 0.0, (20, 12)),
    ("last_dense", "sigmoid", 0, 0.0, (16, 8)),
    ("dense", "crelu", 1, 0.0, (12, 10)),
    ("resnet", "selu", 0, 0.25, (16, 9, 5)),
    ("dense", "relu", 1, 0.25, ((16, 8), (9,))),
])
def test_reference_backward_restates_the_oracle(mode, act, bn, dropout, hidden):
    """StepRef's gradients, computed from the forward values alone (a recovered from H), equal the oracle's backward."""
    from tests.helpers import to_product_batch
    from wide_deep_b200.plan import Plan
    fc, cross, model = KR.parity_conf(hidden, mode=mode, act=act, bn=bn, dropout=dropout)
    B = 150
    rng = np.random.default_rng(7)
    om = OM.OracleModel(fc, cross, model, "wide_deep", embedding_dim_override=8).init(8)
    plan = Plan(fc, cross, model, "wide_deep", max_batch=B, embedding_dim_override=8, max_nnz=B * 64, max_keys=B * 64)
    params = KR.random_params([(n, s[3]) for n, s in plan.tensor_names.items()], rng, act)
    for n, v in params.items():
        om.params[n] = v.copy()
    om.global_step = 3
    raw = KR.raw_batch(B, rng)
    label = (rng.random(B) < 0.3).astype(np.float32)
    weight = (rng.random(B) + 0.5).astype(np.float32)
    _, cache = om.forward(raw, train=True)
    grads = om.backward(cache, label, weight)
    fake = _OracleAsGpu(plan, om, raw, cache)
    ref = KR.StepRef(fake, to_product_batch(plan, raw, label, weight), params, "ffma", step=3 if dropout else None)
    got, M, R, C = ref.gradients()
    assert set(got) <= set(params)
    for name, g in grads.items():
        if isinstance(g, tuple):
            dense = np.zeros(om.params[name].shape)
            dense[g[0]] = np.asarray(g[1]).reshape((len(g[0]),) + dense.shape[1:])
            g = dense
        g = np.asarray(g, dtype=np.float64).reshape(got[name].shape)
        np.testing.assert_allclose(got[name], g, rtol=1e-5, atol=1e-7 * max(1.0, np.abs(g).max()), err_msg=name)
        assert np.all(M[name] + 1e-12 >= np.abs(got[name])), name
    for c in ref.forward_checks():          # (the kernels' BN scale is fp32 gamma * fp32 inv, the oracle's exact: 2^-24 apart)
        assert c.worst1 <= 0.05 and c.worst2 <= 1e-6, c
