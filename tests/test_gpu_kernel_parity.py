"""Every MLP layer output and every train-step gradient against float64, per GEMM engine and at tile edges (tests/kernel_ref.py).

Each step is probed with SGD at a learning rate of 2^24, so the gradients come back through the public API; the reference is
recomputed from the GPU's own deep input and hidden outputs.  Criterion 1 (elementwise, worst-case C * M) needs no calibration.
Criterion 2 (per 128 x 128 tile RMS of |gpu - ref| / R) is held to TAU, 4x the worst tile measured over this whole file on an
H100 80GB HBM3 (700 W power limit):

    worst tile          ffma      tc3x      bf16x3
    layer outputs       6.0e-7    8.1e-6    7.0e-6
    gradients           2.5e-6    6.5e-5    3.9e-5

The numpy emulation of the engines (tests/test_kernel_ref.py) predicts 3.9e-7 for ffma and tc3x and 6.0e-6 for bf16x3 on a single
GEMM.  ffma and bf16x3 land there; tc3x does not: its worst tile grows with K (8.1e-6 at K = 1174, the last layer of
test_wide_layers_partial_tiles, against ~2e-6 at K <= 300), which fits an accumulation in the wgmma pipe that is not
round-to-nearest fp32 rather than the tf32 split.  It stays far inside criterion 1.  The single-pass tf32 engine tc1x (worst
forward tile 8.2e-4) misses the tc3x and bf16x3 forward bounds by 25x and 29x.
"""
from collections import defaultdict

import numpy as np
import pytest

from tests import kernel_ref as KR
from tests.helpers import to_product_batch
from wide_deep_b200.model import WideDeepModel
from wide_deep_b200.plan import Plan

pytestmark = pytest.mark.gpu

ENGINES = ["ffma", "tc3x", "bf16x3"]
TAU = {"forward": {"ffma": 2.4e-6, "tc3x": 3.3e-5, "bf16x3": 2.8e-5}, "gradient": {"ffma": 1.0e-5, "tc3x": 2.6e-4, "bf16x3": 1.6e-4}}
WORST = defaultdict(float)                                # (engine, kind) -> worst criterion-2 tile seen
ACTS = ["relu", "relu6", "sigmoid", "tanh", "leaky_relu", "elu", "selu", "softplus", "softsign", "crelu"]
MODES = ["simple", "first_dense", "last_dense", "dense", "resnet"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (e, kind), w in sorted(WORST.items()):
        tau = TAU[kind].get(e)
        print("\n%-7s %-8s worst criterion-2 tile %.3g (%s)" % (e, kind, w, "tau %.3g, %.2fx" % (tau, w / tau) if tau else "control"))


def build(engine, hidden, mode="simple", act="relu", bn=1, dropout=0.0, wide_input=False, max_batch=2100, opt=KR.SGD_PROBE):
    fc, cross, model = KR.parity_conf(hidden, mode=mode, act=act, bn=bn, dropout=dropout, opt=opt)
    emb = 64 if wide_input else 8
    plan = Plan(fc, cross, model, "wide_deep", max_batch=max_batch, embedding_dim_override=emb, max_nnz=max_batch * 40,
                max_keys=max_batch * 40, gemm_engine=engine)
    assert plan.d0_phys == (224 if wide_input else 32)
    return plan, WideDeepModel(plan)


def batch(plan, B, rng, dense_scale=1.0):
    raw = KR.raw_batch(B, rng, dense_scale)
    return to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32), (rng.random(B) + 0.5).astype(np.float32))


def params_for(plan, rng):
    return KR.random_params([(n, s[3]) for n, s in plan.tensor_names.items()], rng, plan.activation)


def assert_checks(engine, checks, what):
    bad = []
    for c in checks:
        kind = "forward" if c.name.startswith("tower") else "gradient"
        WORST[engine, kind] = max(WORST[engine, kind], c.worst2)
        if not (c.worst1 <= 1.0 and c.worst2 <= TAU[kind][engine]):
            bad.append(c)
    assert not bad, "%s (%s): %s" % (what, engine, "\n".join(map(repr, bad)))


def probe(engine, plan, pm, B, rng, dense_scale=1.0, split=False, b=None, params=None):
    """One probed step: forward check of every layer and check of every gradient.  -> (gradients, batch, params)"""
    b = b or batch(plan, B, rng, dense_scale)
    params = params or params_for(plan, rng)
    step = pm.global_step
    grads, _ = KR.probe_step(pm, b, params, split=split)
    ref = KR.StepRef(pm, b, params, engine, step=step)
    assert_checks(engine, ref.forward_checks() + ref.gradient_checks(grads, params), "B=%d" % B)
    assert pm.gemm_fallback_count() == 0
    return grads, b, params


@pytest.mark.parametrize("engine", ENGINES)
def test_narrow_widths_every_batch_edge(engine):
    """Widths 129, 33, 8 and 1 on a 32-wide deep input, one plan of max_batch 2100 at B = 1 ... 2100: ragged row tiles of the bias,
    gamma and beta partials, weight gradients reduced over 1 to 2100 rows, and one graph per batch size."""
    plan, pm = build(engine, (129, 33, 8, 1))
    rng = np.random.default_rng(1)
    for B in (1, 17, 64, 65, 127, 129, 300, 2100):
        probe(engine, plan, pm, B, rng)


@pytest.mark.parametrize("engine", ENGINES)
def test_wide_layers_partial_tiles(engine):
    """Widths 257, 200, 520 and 100 densely connected to a 197-wide deep input (d0_phys 224): partial N tiles, K up to 1174."""
    plan, pm = build(engine, (257, 200, 520, 100), mode="dense", act="tanh", wide_input=True)
    probe(engine, plan, pm, 300, np.random.default_rng(2))


@pytest.mark.parametrize("engine", ENGINES)
def test_crelu_200_units(engine):
    """crelu of 200 units hands on 400 features (N_phys 416) through resnet connections."""
    plan, pm = build(engine, (200, 48), mode="resnet", act="crelu", wide_input=True)
    probe(engine, plan, pm, 129, np.random.default_rng(3))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("act", ACTS)
def test_activations_and_modes(engine, act):
    """All ten activations over the five connection modes; BN on and off; two towers on every other case (dX0 summed over them)."""
    i = ACTS.index(act)
    hidden = ((100, 40), (33,)) if i % 2 else (100, 40, 24)
    plan, pm = build(engine, hidden, mode=MODES[i % 5], act=act, bn=(i // 2) % 2 == 0, wide_input=i % 3 == 0)
    probe(engine, plan, pm, 300, np.random.default_rng(10 + i))


@pytest.mark.parametrize("engine", ENGINES)
def test_dropout(engine):
    plan, pm = build(engine, (129, 64), mode="first_dense", dropout=0.25)
    rng = np.random.default_rng(4)
    probe(engine, plan, pm, 300, rng)
    probe(engine, plan, pm, 129, rng)                       # (second step: the mask counter has advanced)


@pytest.mark.parametrize("engine", ENGINES)
def test_weight_gradient_splits_without_rows(engine):
    """max_batch 16384 and one 100-unit layer on d0_phys 32 give 32 weight-gradient splits; at B = 300 most of them get no rows."""
    plan, pm = build(engine, (100,), max_batch=16384)
    probe(engine, plan, pm, 300, np.random.default_rng(5))


@pytest.mark.parametrize("engine", ENGINES)
def test_fused_and_split_steps(engine):
    """The unfused wd_step_backward + wd_step_apply path (dense_reduce) meets the same bounds as the fused step, bit for bit."""
    plan, pm = build(engine, (129, 33), mode="dense", wide_input=True)
    rng = np.random.default_rng(6)
    g1, b, params = probe(engine, plan, pm, 300, rng)
    g2, _, _ = probe(engine, plan, pm, 300, rng, split=True, b=b, params=params)
    for n in g1:
        np.testing.assert_array_equal(g1[n], g2[n], err_msg=n)


def _sequence(engine, rng_seed):
    plan, pm = build(engine, (129, 33), mode="first_dense")
    rng = np.random.default_rng(rng_seed)
    out = []
    for i, B in enumerate((2100, 2100, 2100, 300, 1, 2100, 65)):
        out.append(probe(engine, plan, pm, B, rng, dense_scale=1e4 if i < 3 else 1.0)[0])
    return out


@pytest.mark.parametrize("engine", ENGINES)
def test_batch_sequence_graph_and_eager(engine, monkeypatch):
    """B = 2100, 2100, 2100, 300, 1, 2100, 65 on one handle: graph capture, replay and re-capture as B changes.  The first batches
    carry a dense feature of scale 1e4, so a row they leave behind in an activation buffer would stand far above the bounds of
    the smaller steps after them.  The same sequence without graphs gives bit-identical gradients."""
    graph = _sequence(engine, 7)
    monkeypatch.setenv("WD_NO_GRAPH", "1")
    eager = _sequence(engine, 7)
    for s, (a, b) in enumerate(zip(graph, eager)):
        for n in a:
            np.testing.assert_array_equal(a[n], b[n], err_msg="step %d %s" % (s, n))


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("act", ["relu", "crelu"])
def test_weight_copies_after_optimizer(engine, act):
    """Three Adagrad steps (single tower, so bf16x3 splits the dense update over two streams; crelu: crelu_mirror), then the
    forward of every layer against get_tensor's weights.  Then set_tensor on the handle that is replaying its graph, and the
    forward of the next step against the uploaded weights."""
    plan, pm = build(engine, (129, 64), act=act, opt="Adagrad")
    rng = np.random.default_rng(8)
    for _ in range(3):
        pm.train_step(batch(plan, 300, rng))
    b = batch(plan, 300, rng)
    pm.forward(b)
    now = {n: pm.get_tensor(n) for n in pm.tensor_names()}
    assert_checks(engine, KR.StepRef(pm, b, now, engine).forward_checks(), "after Adagrad")
    new = params_for(plan, rng)
    for n, v in new.items():
        pm.set_tensor(n, v)
    pm.train_step(b)
    assert_checks(engine, KR.StepRef(pm, b, new, engine).forward_checks(), "after set_tensor")
    assert pm.gemm_fallback_count() == 0


def test_tc1x_misses_the_three_pass_bounds():
    """Negative control: single-pass tf32 fails the forward criterion 2 of tc3x and of bf16x3 by at least 8x."""
    plan, pm = build("tc1x", (257, 200), wide_input=True)
    b = batch(plan, 300, np.random.default_rng(9))
    params = params_for(plan, np.random.default_rng(9))
    KR.probe_step(pm, b, params)
    worst = max(c.worst2 for c in KR.StepRef(pm, b, params, "tc3x").forward_checks())
    WORST["tc1x", "forward"] = worst
    tau = TAU["forward"]
    print("\ntc1x worst tile %.3g: %.1fx tau(tc3x), %.1fx tau(bf16x3)" % (worst, worst / tau["tc3x"], worst / tau["bf16x3"]))
    assert worst >= 8 * tau["tc3x"] and worst >= 8 * tau["bf16x3"]


def test_hidden_output_wider_than_4096_columns():
    """hidden_output sizes its buffer from the layer: crelu of 2100 units is 4200 features (N_phys 4224)."""
    plan, pm = build("bf16x3", (2100, 8), act="crelu", max_batch=64)
    b = batch(plan, 5, np.random.default_rng(10))
    pm.forward(b)
    h = pm.hidden_output(0, 0, 5)
    assert h.shape == (5, 4224) and np.isfinite(h).all() and not h[:, 4200:].any()
