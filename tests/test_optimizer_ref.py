"""The optimizer reference and its bound (tests/optimizer_ref.py) pinned down on the CPU.

The fp32 emulation of the update kernels passes the derived bound on about 1e5 random elements per optimizer plus adversarial
ones (FTRL's |z1| within 1% of l1 on both signs, accumulators from 1e-8 to 1e4, zero mean squares and second moments, zero and
tiny gradients, Adam at t = 0, 1 and 5000).  Each planted defect fails on the same inputs by at least DEFECT_MARGIN times the
bound.  Run with -s to see the worst ratios.
"""
import numpy as np
import pytest

from tests import optimizer_ref as R

N = 100000
DEFECT_MARGIN = 4.0
ADAM_STEPS = (0, 1, 5000)
HP = {
    "sgd": [dict(lr=0.05)],
    "adagrad": [dict(lr=0.05)],
    "ftrl": [dict(lr=0.1, l1=0.5, l2=1.0), dict(lr=0.1, l1=0.0, l2=0.0), dict(lr=0.05, l1=0.01, l2=0.1)],
    "rmsprop": [dict(lr=0.05, rho=0.8, momentum=0.0, epsilon=1e-10), dict(lr=0.05, rho=0.9, momentum=0.5, epsilon=1e-10)],
    "adam": [dict(lr=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8), dict(lr=0.05, beta1=0.8, beta2=0.999, epsilon=1e-8)],
}


def _logu(rng, lo, hi, n):
    return 10.0 ** rng.uniform(lo, hi, n)


def elements(kind, hp, seed, n=N):
    """(w, s1, s2, g) float32 arrays: random states and gradients over many decades, then the adversarial elements."""
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(n) * _logu(rng, -3, 1, n)
    g = rng.standard_normal(n) * _logu(rng, -6, 1, n)
    q = n // 20
    g[:q] = 0.0                                                      # zero gradients
    g[q:2 * q] = rng.standard_normal(q) * _logu(rng, -30, -12, q)     # tiny gradients (products underflow)
    s1 = np.zeros(n)
    s2 = np.zeros(n)
    if kind in ("adagrad", "ftrl"):
        s1 = _logu(rng, -8, 4, n)
    if kind == "ftrl":
        s2 = rng.standard_normal(n) * _logu(rng, -3, 1, n)
        # |z1| within 1% of l1, both signs: z = target - (g - (sqrt(n1) - sqrt(n)) / lr * w)
        k = slice(2 * q, 4 * q)
        lr, l1 = R.f32(hp["lr"]), R.f32(hp["l1"])
        n1 = s1[k] + g[k] ** 2
        target = np.where(rng.random(2 * q) < 0.5, -1.0, 1.0) * l1 * (1 + rng.uniform(-0.01, 0.01, 2 * q))
        s2[k] = target - (g[k] - (np.sqrt(n1) - np.sqrt(s1[k])) / lr * w[k])
    if kind == "rmsprop":
        s1 = _logu(rng, -8, 2, n)
        s1[2 * q:4 * q] = 0.0                                         # ms = 0 (half of them with g = 0 or tiny, below)
        g[3 * q:4 * q] = rng.standard_normal(q) * _logu(rng, -7, -4, q)
        s2 = rng.standard_normal(n) * _logu(rng, -4, 0, n)
    if kind == "adam":
        s1 = rng.standard_normal(n) * _logu(rng, -4, 0, n)
        s2 = _logu(rng, -8, 2, n)
        s2[2 * q:4 * q] = 0.0                                         # v = 0, some with m = 0 too
        s1[2 * q:3 * q] = 0.0
        g[3 * q:3 * q + q // 2] = 0.0
    return tuple(np.asarray(x, dtype=np.float32) for x in (w, s1, s2, g))


def cases(kind):
    """(label, hp, steps, touched, dense, inputs) for every hyper-parameter set, Adam form and step count."""
    out = []
    for i, hp in enumerate(HP[kind]):
        if kind != "adam":
            out.append(("%s hp%d" % (kind, i), hp, 0, True, False, elements(kind, hp, 100 + i)))
            continue
        for t in ADAM_STEPS:
            for form, touched, dense in (("sparse", True, False), ("untouched", False, False), ("dense", True, True)):
                out.append(("adam hp%d t=%d %s" % (i, t, form), hp, t, touched, dense, elements(kind, hp, 200 + 10 * i + t % 7, N // 9)))
    return out


def worst(kind, hp, steps, touched, dense, inp, defect=None):
    w, s1, s2, g = inp
    after = R.emulate(kind, hp, w, s1, s2, g, steps=steps, touched=touched, dense=dense, defect=defect)
    res = R.check(kind, hp, (w, s1, s2), g, after, steps=steps, touched=touched, dense=dense)
    return res.worst(), res


def test_hyperparameter_constants_are_fp32_exact_where_the_bound_says():
    """1 - beta and 1 - rho are exact in fp32 for the values used (Sterbenz): one_minus asserts the range."""
    for kind in ("rmsprop", "adam"):
        for hp in HP[kind]:
            for key in ("rho", "beta1", "beta2"):
                if key in hp:
                    x = np.float32(hp[key])
                    assert float(np.float32(1) - x) == 1.0 - float(x)


def test_depths_match_the_documented_table():
    for kind in R.KINDS:
        hp = HP[kind][-1]
        if kind == "adam":
            assert R.depths(kind, hp, dense=True) == R.DEPTH["adam_dense"]
            assert R.depths(kind, hp, touched=False) == R.DEPTH["adam_untouched"]
        assert R.depths(kind, hp) == R.DEPTH[kind], kind


def test_adam_beta_powers_underflow_at_late_steps():
    """beta1^5001 underflows in fp32 (to a subnormal that 0.9 no longer moves); lr_t is then lr * sqrt(1 - beta2^5001), and the
    device's fp32 lr_t stays within 5 roundings of the reference's."""
    p1, p2 = R.beta_powers(HP["adam"][0], 5000)
    assert 0 <= p1 < np.finfo(np.float32).tiny and 0 < p2 < 0.01
    lr = R.adam_lr_t(HP["adam"][0], 5000)
    assert abs(float(R.adam_lr_t32(HP["adam"][0], 5000)) - lr) <= 5 * R.U * lr


def test_ref_update_first_adam_step_and_untouched_row():
    """From zero moments, Adam's first step moves w by lr * g / (|g| + eps / sqrt(1 - b2)) in both forms, and an untouched row
    with zero moments stays; check()'s reference is ref_update's."""
    hp = HP["adam"][0]
    w, g = np.float32([0.5, -0.25, 1.0]), np.float32([1e-2, -3.0, 0.0])
    z = np.zeros(3, dtype=np.float32)
    step = R.f32(hp["lr"]) * g.astype(np.float64) / (np.abs(g.astype(np.float64)) + R.f32(hp["epsilon"]) / np.sqrt(1 - R.f32(hp["beta2"])))
    for dense in (False, True):
        w1, m1, v1 = R.ref_update("adam", hp, w, z, z, g, steps=0, dense=dense)
        np.testing.assert_allclose(w1, w - step, rtol=0, atol=1e-12)
        np.testing.assert_allclose(m1, (1 - R.f32(hp["beta1"])) * g.astype(np.float64), rtol=1e-15)
        res = R.check("adam", hp, (w, z, z), g, R.emulate("adam", hp, w, z, z, g, dense=dense), dense=dense)
        np.testing.assert_array_equal(res.ref["w"], w1)
    w1, m1, v1 = R.ref_update("adam", hp, w, z, z, g, steps=3, touched=False)
    np.testing.assert_array_equal(w1, w)
    assert not m1.any() and not v1.any()


@pytest.mark.parametrize("kind", R.KINDS)
def test_emulated_kernels_pass_the_bound(kind):
    lines, bad = [], []
    for label, hp, steps, touched, dense, inp in cases(kind):
        wr, res = worst(kind, hp, steps, touched, dense, inp)
        lines.append("%-28s worst ratio %s%s" % (label, " ".join("%s %.3g" % kv for kv in wr.items()),
                                                 ", %d FTRL elements near l1" % res.ambiguous.sum() if kind == "ftrl" else ""))
        if max(wr.values()) > 1.0:
            bad.append(label)
    print("\n" + "\n".join(lines))
    assert not bad, bad


def test_ftrl_adversarial_elements_reach_the_branch_on_both_sides():
    """The near-threshold elements put |z1| on both sides of l1 (w' = 0 and w' != 0) and some inside the ambiguity band."""
    hp = HP["ftrl"][0]
    w, s1, s2, g = elements("ftrl", hp, 100)
    after = R.emulate("ftrl", hp, w, s1, s2, g)
    q = N // 20
    near = slice(2 * q, 4 * q)
    z = after[2][near].astype(np.float64)
    assert np.any((np.abs(z) > 0.5) & (z > 0)) and np.any((np.abs(z) > 0.5) & (z < 0))
    assert np.any(np.abs(z) <= 0.5) and np.any(after[0][near] == 0) and np.any(after[0][near] != 0)


# defect -> (kind, the cases it applies to: labels containing one of these).  l2 and l1 only act where they are nonzero (hp0),
# the momentum term where momentum is (hp1).  Adam's bias correction is off by one step only while it still matters: at t = 5000
# an extra beta2 factor moves lr_t by ~1e-7 relative, which no per-element bound resolves.
DEFECT_CASES = {
    "adagrad_old_acc": ("adagrad", ("",)),
    "ftrl_new_n_twice": ("ftrl", ("",)),
    "ftrl_no_l2": ("ftrl", ("ftrl hp0",)),
    "ftrl_l1_sign": ("ftrl", ("ftrl hp0",)),
    "ftrl_skip_zero_g": ("ftrl", ("",)),
    "rmsprop_eps_outside": ("rmsprop", ("",)),
    "rmsprop_no_momentum": ("rmsprop", ("rmsprop hp1",)),
    "adam_bias_off_by_one": ("adam", ("t=0 ", "t=1 ")),
    "adam_untouched_no_decay": ("adam", ("untouched",)),
    "adam_untouched_double_decay": ("adam", ("untouched",)),
}


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_planted_defect_fails_the_bound(defect):
    kind, sel = DEFECT_CASES[defect]
    ratios = []
    for label, hp, steps, touched, dense, inp in cases(kind):
        if not any(x in label for x in sel):
            continue
        wr, _ = worst(kind, hp, steps, touched, dense, inp, defect=defect)
        ratios.append((max(wr.values()), label))
    # every case the defect applies to must expose it, not just the worst one
    least = min(ratios)
    print("\n%-28s worst ratio %.3g (%s); least over its cases %.3g (%s)" % ((defect,) + max(ratios) + least))
    assert least[0] >= DEFECT_MARGIN, (defect, ratios)
