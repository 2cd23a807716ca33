"""numpy float32 emulation of Adam's untouched-row steps, as deferred host tables replay them (WD_PLACE_DEFER_ADAM).

A row that no gradient touched takes, at Adam step j (1-based), m = m*b1; v = v*b2; w -= lr_t[j]*m/(sqrt(v)+eps) with
lr_t[j] = lr*sqrt(1 - b2^j)/(1 - b1^j), the beta powers multiplied up in fp32 from b^1.  numpy float32 `*`, `/` and `sqrt` round
like the library's kernels (built without fast-math, denormals kept), so this emulation is bit-exact, not just close.
"""
import numpy as np

F = np.float32


def lr_t_table(lr, beta1, beta2, cap=1 << 22):
    """(lr_t, last): lr_t[j] for j = 1 .. last (lr_t[0] unused), last = the first step at which both 1 - beta^j round to 1 in
    fp32; every later step has lr_t == lr exactly."""
    b1, b2 = F(beta1), F(beta2)
    p1, p2 = [F(0), b1], [F(0), b2]
    while not (F(1) - p1[-1] == F(1) and F(1) - p2[-1] == F(1)):
        if len(p1) > cap:
            raise ValueError("betas too close to 1")
        p1.append(F(p1[-1] * b1))
        p2.append(F(p2[-1] * b2))
    p1, p2 = np.array(p1, dtype=F), np.array(p2, dtype=F)
    lr_t = (F(lr) * np.sqrt(F(1) - p2)) / (F(1) - p1)
    return lr_t.astype(F), len(p1) - 1


def replay(w, m, v, s, g, lr, beta1, beta2, eps, early_exit=True, table=None):
    """Steps s+1 .. g of the untouched update on float32 arrays w, m, v (copies returned) -> (w, m, v, steps run).  early_exit:
    stop once a step past the table's end leaves every value's bits unchanged (every later step is the same map)."""
    lr_t, last = table if table is not None else lr_t_table(lr, beta1, beta2)
    w, m, v = (np.array(a, dtype=F, copy=True) for a in (w, m, v))
    b1, b2, e, lr = F(beta1), F(beta2), F(eps), F(lr)
    run = 0
    for j in range(s + 1, g + 1):
        lt = lr_t[j] if j <= last else lr
        w0, m0, v0 = w, m, v
        m = m * b1
        v = v * b2
        w = w - (lt * m) / (np.sqrt(v) + e)
        run += 1
        if early_exit and j > last and w.tobytes() == w0.tobytes() and m.tobytes() == m0.tobytes() and v.tobytes() == v0.tobytes():
            break
    return w, m, v, run
