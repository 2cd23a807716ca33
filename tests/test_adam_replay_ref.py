"""The float32 emulation of deferred Adam's replayed steps (tests/adam_replay_ref.py) against float64 Adam, and its early exit
against the full loop."""
import numpy as np
import pytest

from tests.adam_replay_ref import lr_t_table, replay


def _f64_untouched(w, m, v, s, g, lr, b1, b2, eps):
    w, m, v = (np.asarray(a, dtype=np.float64).copy() for a in (w, m, v))
    for j in range(s + 1, g + 1):
        lt = lr * np.sqrt(1 - b2 ** j) / (1 - b1 ** j)
        m, v = m * b1, v * b2
        w = w - lt * m / (np.sqrt(v) + eps)
    return w, m, v


def _state(rng, n):
    w = rng.standard_normal(n).astype(np.float32) * 0.1
    m = rng.standard_normal(n).astype(np.float32) * 1e-2
    v = (rng.random(n).astype(np.float32) * 1e-3 + 1e-5).astype(np.float32)
    return w, m, v


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.5, 0.9), (0.8, 0.999)])
def test_lr_t_table_matches_float64_and_ends_at_lr(betas):
    lr = 0.05
    lr_t, last = lr_t_table(lr, *betas)
    j = np.arange(1, last + 1)
    b1, b2 = (float(np.float32(b)) for b in betas)          # (the betas the library holds)
    ref = lr * np.sqrt(1 - b2 ** j) / (1 - b1 ** j)
    assert np.allclose(lr_t[1:], ref, rtol=1e-4)
    assert lr_t[last] == np.float32(lr)
    # the last step is the first at which both 1 - beta^j round to 1 (beta powers multiplied up in fp32 from beta^1)
    f = np.float32
    p1, p2 = f(betas[0]), f(betas[1])
    done = [f(1) - p1 == f(1) and f(1) - p2 == f(1)]
    for _ in range(last - 1):
        p1, p2 = f(p1 * f(betas[0])), f(p2 * f(betas[1]))
        done.append(f(1) - p1 == f(1) and f(1) - p2 == f(1))
    assert done[-1] and not any(done[:-1])


@pytest.mark.parametrize("s,g", [(0, 1), (3, 20), (10, 400), (0, 3000)])
def test_replay_matches_float64_adam(s, g):
    rng = np.random.default_rng(s * 1000 + g)
    w, m, v = _state(rng, 256)
    lr, b1, b2, eps = 0.05, 0.9, 0.999, 1e-8
    ew, em, ev, run = replay(w, m, v, s, g, lr, b1, b2, eps)
    assert run == g - s                      # (all steps before the table's end: no early exit)
    rw, rm, rv = _f64_untouched(w, m, v, s, g, lr, b1, b2, eps)
    assert np.allclose(ew, rw, rtol=1e-4, atol=1e-6)
    assert np.allclose(em, rm, rtol=1e-4, atol=1e-30)
    assert np.allclose(ev, rv, rtol=1e-4, atol=1e-30)


@pytest.mark.parametrize("betas,s,k", [((0.5, 0.5), 0, 2000), ((0.5, 0.9), 7, 5000), ((0.9, 0.999), 0, 17500)])
def test_early_exit_equals_the_full_loop(betas, s, k):
    rng = np.random.default_rng(k)
    w, m, v = _state(rng, 64)
    w[:8] = 0.5
    m[:8] = 0
    v[:8] = 0                                 # rows no gradient ever touched: the map is the identity from the start
    table = lr_t_table(0.05, *betas)
    full = replay(w, m, v, s, s + k, 0.05, betas[0], betas[1], 1e-8, early_exit=False, table=table)
    fast = replay(w, m, v, s, s + k, 0.05, betas[0], betas[1], 1e-8, early_exit=True, table=table)
    for a, b in zip(full[:3], fast[:3]):
        assert a.tobytes() == b.tobytes()
    assert full[3] == k
    if s + k > table[1] + 1000:
        assert fast[3] < k                   # the exit did fire
