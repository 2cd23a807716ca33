"""Float64 reference of one optimizer update per element, with an error bound derived from the kernels' operation order.

The update kernels (csrc/sparse_dev.cuh opt_update / adam_untouched4, csrc/mlp.cu opt_update_d) apply TensorFlow's training ops
element by element in fp32:

    sgd       w -= lr * g
    adagrad   acc += g^2;  w -= lr * g / sqrt(acc)                                             (ApplyAdagrad)
    ftrl      n1 = n + g^2;  z1 = z + g - (sqrt(n1) - sqrt(n)) / lr * w;                        (ApplyFtrl, lr_power -0.5)
              w = |z1| > l1 ? (sign(z1) l1 - z1) / (sqrt(n1) / lr + 2 l2) : 0
    rmsprop   ms += (g^2 - ms)(1 - rho);  mom = mom * momentum + g * lr / sqrt(ms + eps);  w -= mom   (ApplyRMSProp)
    adam      dense (ApplyAdam):  m += (g - m)(1 - b1);  v += (g^2 - v)(1 - b2);  w -= lr_t m / (sqrt(v) + eps)
              sparse (AdamOptimizer._apply_sparse_shared), a touched row:  m = m b1 + g (1 - b1);  v = v b2 + g^2 (1 - b2);  step
              an untouched row: decay and step only.  lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) from the fp32 beta powers the
              device holds, beta^(t+1) after t steps, multiplied up in fp32 (wd_set_opt_step, adam_tick_kernel).

One transcription of these formulas (``_update``), in the kernels' operation order, runs on three kinds of numbers:

* ``Q``: the float64 value of each intermediate, its magnitude M and its depth k (rounded fp32 operations on its longest
  path).  The outputs' values are the reference; M and k give the bound.
* float64 arrays: the reference at g +- dg, for the gradient's own uncertainty.
* float32 arrays: an emulation of the kernel (numpy rounds every operation to fp32), which the CPU suite holds to the bound.

The bound of every output is  ``|gpu - ref| <= k * 2^-24 * M + sens_g + ulp32(ref)``.  Every rounded fp32 operation errs by at
most u (|x| + 2^-126), u = 2^-24 (the 2^-126 covers subnormal results).  By induction over the expression, an intermediate
of depth k is then within k u M of its exact value, to first order, when M follows

    a +- b:  M_a + M_b                      a / b:  M_a / |b| + |a / b| M_b / |b|
    a * b:   M_a |b| + |a| M_b              (M_a |b| when b is exact, k_b = 0)
    sqrt(a): M_a / sqrt(a)                  (a > 0: |sqrt(a') - sqrt(a)| <= |a' - a| / sqrt(a); for a = 0: sqrt(M_a / u))

plus 2^-126 per rounded operation.  Each rule makes M at least the value's magnitude and at least what the operands' errors
contribute, k_a u M_a |b| + k_b u |a| M_b for a product, so the operation's own rounding, u |result|, raises the depth by one.  A difference of square roots thus counts as sqrt(n1) + sqrt(n0), so FTRL's cancellation is
covered.  Operations that are exact are not counted: 1 - beta and 1 - rho for beta, rho in [0.5, 1] (Sterbenz), 2 * l2 and
copysign.  Contracting a multiply and an add into an FMA (the build allows it; it uses IEEE division and sqrtf) removes a
rounding and never raises the bound, so it holds either way.  The depth k of each output, the constant C of its bound, is:

    kind      w    s1   s2        kind            w    s1   s2
    sgd       2    -    -         rmsprop         9    4    8
    adagrad   5    2    -         adam (dense)    8    3    4
    ftrl      9    2    7         adam (sparse)   8    2    3         (untouched rows: w 8, m 1, v 1)

Adam's lr_t is one fp32 expression per step, of depth 5 and relative error below 5u (both subtractions are exact or err
relatively by u); it enters as a leaf of that depth with M = lr_t.  ``DEPTH`` holds the table and the CPU suite checks it
against the depths the transcription derives.

The gradient is known to within dg (the SGD probe's read-back, tests/kernel_ref.py); sens_g = max |ref(g +- dg) - ref(g)|
carries it, |d out / d g| dg to first order.  FTRL's branch: where |z1| lies within its own bound of l1 either branch is
accepted (w' = 0 or the formula's value); everywhere else the branch must match, and a w' the reference puts at 0 must be 0.
"""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -126
KINDS = ("sgd", "adagrad", "ftrl", "rmsprop", "adam")
OUTS = ("w", "s1", "s2")
DEPTH = {"sgd": (2, 0, 0), "adagrad": (5, 2, 0), "ftrl": (9, 2, 7), "rmsprop": (9, 4, 8),
         "adam_dense": (8, 3, 4), "adam": (8, 2, 3), "adam_untouched": (8, 1, 1)}
LR_T_DEPTH = 5
SECOND_ORDER = 1.0 + 2.0 ** -16            # the first-order bound's neglected O(k^2 u^2) terms, with room to spare
DEFECTS = ("adagrad_old_acc", "ftrl_new_n_twice", "ftrl_no_l2", "ftrl_l1_sign", "ftrl_skip_zero_g", "rmsprop_eps_outside",
           "rmsprop_no_momentum", "adam_bias_off_by_one", "adam_untouched_no_decay", "adam_untouched_double_decay")


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def f32(x):
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------ the three kinds of numbers
class Q(object):
    """float64 value v, magnitude M (>= |v|) and depth k of an intermediate of the update."""
    __slots__ = ("v", "M", "k")

    def __init__(self, v, M=None, k=0):
        self.v = np.asarray(v, dtype=np.float64)
        self.M = np.abs(self.v) if M is None else np.asarray(M, dtype=np.float64)
        self.k = k

    def __add__(self, o):
        return Q(self.v + o.v, self.M + o.M + TINY, max(self.k, o.k) + 1)

    def __sub__(self, o):
        return Q(self.v - o.v, self.M + o.M + TINY, max(self.k, o.k) + 1)

    def __mul__(self, o):
        if self.k and o.k:                # both inexact: each one's error is scaled by the other's value
            M = self.M * np.abs(o.v) + np.abs(self.v) * o.M
        else:
            M = self.M * o.M
        return Q(self.v * o.v, M + TINY, max(self.k, o.k) + 1)

    def __truediv__(self, o):
        v = self.v / o.v
        return Q(v, self.M / np.abs(o.v) + np.abs(v) * o.M / np.abs(o.v) + TINY, max(self.k, o.k) + 1)

    def __neg__(self):
        return Q(-self.v, self.M, self.k)


class _QOps(object):
    def const(self, x):
        return Q(f32(x))

    def exact(self, x):                  # an fp32 operation whose result is exact (1 - beta for beta in [0.5, 1], 2 * l2)
        return Q(f32(x))

    def sqrt(self, a):
        pos = a.v > 0
        r = np.sqrt(np.maximum(a.v, 0.0))
        with np.errstate(divide="ignore", invalid="ignore"):
            M = np.where(pos, a.M / np.where(pos, r, 1.0), np.sqrt(a.M / U))
        return Q(r, M + TINY, a.k + 1)

    def copysign(self, mag, x):
        return Q(np.copysign(mag.v, x.v), mag.M, mag.k)

    def leaf(self, x):
        return Q(np.asarray(x, dtype=np.float32))


class _FloatOps(object):
    """Plain arithmetic in one numpy float type (float32: the kernel's rounding; float64: the reference's values)."""

    def __init__(self, dtype):
        self.t = dtype

    def const(self, x):
        return self.t(np.float32(x))

    def exact(self, x):
        return self.t(np.float32(x))

    def sqrt(self, a):
        return np.sqrt(a)

    def copysign(self, mag, x):
        return np.copysign(mag, x).astype(self.t)

    def leaf(self, x):
        return np.asarray(np.asarray(x, dtype=np.float32), dtype=self.t)


QOPS, F64, F32 = _QOps(), _FloatOps(np.float64), _FloatOps(np.float32)


def one_minus(X, x):
    """1 - x as the kernels compute it ("1.f - o.beta1"): exact by Sterbenz for x in [0.5, 2]."""
    x = f32(x)
    assert 0.5 <= x <= 2.0, "1 - %g would round: count it as an operation" % x
    return X.exact(1.0 - x)


# ------------------------------------------------------------------------------------------------ Adam's step size
def beta_powers(hp, steps):
    """The fp32 beta powers {beta1^(t+1), beta2^(t+1)} the device holds after `steps` steps (wd_set_opt_step's loop)."""
    b1, b2 = np.float32(hp["beta1"]), np.float32(hp["beta2"])
    p1, p2 = b1, b2
    for _ in range(int(steps)):
        p1, p2 = np.float32(p1 * b1), np.float32(p2 * b2)
    return p1, p2


def adam_lr_t(hp, steps):
    """float64 lr_t of the step after `steps` steps, from the fp32 beta powers the device holds."""
    p1, p2 = beta_powers(hp, steps)
    return f32(hp["lr"]) * np.sqrt(1.0 - float(p2)) / (1.0 - float(p1))


def adam_lr_t32(hp, steps):
    """The kernels' fp32 lr_t (with_lr_t / opt_update_d): lr * sqrtf(1 - bpow[1]) / (1 - bpow[0])."""
    p1, p2 = beta_powers(hp, steps)
    one = np.float32(1)
    return np.float32(np.float32(np.float32(hp["lr"]) * np.sqrt(np.float32(one - p2))) / np.float32(one - p1))


# ------------------------------------------------------------------------------------------------ the formulas
def _update(kind, hp, w, s1, s2, g, lr_t, touched, dense, X, defect=None):
    """(w', s1', s2', extra) of one update in the kernels' operation order; extra = (z1, formula w) for FTRL, else None."""
    c = X.const
    if kind == "sgd":
        return w - c(hp["lr"]) * g, s1, s2, None
    if kind == "adagrad":                                      # s1 += g * g; w -= o.lr * g / sqrtf(s1)
        acc = s1 + g * g
        return w - c(hp["lr"]) * g / X.sqrt(s1 if defect == "adagrad_old_acc" else acc), acc, s2, None
    if kind == "ftrl":
        lr = c(hp["lr"])
        n1 = s1 + g * g
        r1 = X.sqrt(n1)
        r0 = r1 if defect == "ftrl_new_n_twice" else X.sqrt(s1)
        z1 = s2 + g - (r1 - r0) / lr * w
        quad = X.sqrt(n1) / lr
        if defect != "ftrl_no_l2":
            quad = quad + X.exact(2.0 * f32(hp["l2"]))
        l1 = X.copysign(c(hp["l1"]), z1)
        if defect == "ftrl_l1_sign":
            l1 = -l1
        wn = (l1 - z1) / quad
        return wn, n1, z1, (z1, wn)
    if kind == "rmsprop":
        ms = s1 + (g * g - s1) * one_minus(X, hp["rho"])
        den = X.sqrt(ms) + c(hp["epsilon"]) if defect == "rmsprop_eps_outside" else X.sqrt(ms + c(hp["epsilon"]))
        mom = (g * c(hp["lr"])) / den
        if defect != "rmsprop_no_momentum":
            mom = s2 * c(hp["momentum"]) + mom
        return w - mom, ms, mom, None
    if kind == "adam":
        b1, b2 = c(hp["beta1"]), c(hp["beta2"])
        if dense:                                              # ApplyAdam
            m = s1 + (g - s1) * one_minus(X, hp["beta1"])
            v = s2 + (g * g - s2) * one_minus(X, hp["beta2"])
        else:
            m, v = s1 * b1, s2 * b2                            # the decay of every row (adam_decay)
            if touched:
                m = m + g * one_minus(X, hp["beta1"])
                v = v + g * g * one_minus(X, hp["beta2"])
            elif defect == "adam_untouched_no_decay":
                m, v = s1, s2
            elif defect == "adam_untouched_double_decay":
                m, v = m * b1, v * b2
        return w - lr_t * m / (X.sqrt(v) + c(hp["epsilon"])), m, v, None
    raise ValueError(kind)


def _lr_t(kind, hp, steps, X, defect=None):
    if kind != "adam":
        return None
    if defect == "adam_bias_off_by_one":                       # beta powers advanced before the update
        steps = steps + 1
    if X is F32:
        return adam_lr_t32(hp, steps)
    v = adam_lr_t(hp, steps)
    return Q(v, v, LR_T_DEPTH) if X is QOPS else np.float64(v)


def _run(kind, hp, w, s1, s2, g, steps, touched, dense, X, defect=None):
    L = X.leaf
    return _update(kind, hp, L(w), L(s1), L(s2), L(g), _lr_t(kind, hp, steps, X, defect), touched, dense, X, defect)


# ------------------------------------------------------------------------------------------------ the API
def ref_update(kind, hp, w, s1, s2, g, steps=0, touched=True, dense=False):
    """float64 (w', s1', s2') of one update from fp32 inputs.  Adam: `steps` steps done before this one (lr_t from
    ``adam_lr_t``), touched = the row took a gradient (sparse form), dense = ApplyAdam.  FTRL: w' with its branch."""
    w1, a, b, extra = _run(kind, hp, w, s1, s2, g, steps, touched, dense, F64)
    if extra is not None:
        w1 = np.where(np.abs(extra[0]) > f32(hp["l1"]), w1, 0.0)
    return w1, a, b


def emulate(kind, hp, w, s1, s2, g, steps=0, touched=True, dense=False, defect=None):
    """The kernels' fp32 update (numpy float32, every operation rounded, no contraction); `defect` plants one of DEFECTS."""
    w1, a, b, extra = _run(kind, hp, w, s1, s2, g, steps, touched, dense, F32, defect)
    if extra is not None:
        w1 = np.where(np.abs(extra[0]) > np.float32(hp["l1"]), w1, np.float32(0))
    if defect == "ftrl_skip_zero_g":
        z = np.asarray(g, dtype=np.float32) == 0
        w1, a, b = np.where(z, w, w1), np.where(z, s1, a), np.where(z, s2, b)
    return tuple(np.asarray(x, dtype=np.float32) for x in (w1, a, b))


def depths(kind, hp, steps=0, touched=True, dense=False):
    """The depth k of (w', s1', s2') the transcription derives."""
    one = np.ones(1, dtype=np.float32)
    out = _run(kind, hp, one, one, one, one, steps, touched, dense, QOPS)
    return tuple(q.k for q in out[:3])


class Result(object):
    """ref, bound: dicts of float64 arrays by output; ratio: |gpu - ref| / bound per output (<= 1 passes; inf for a wrong FTRL
    branch or a non-finite value); ambiguous: FTRL elements whose |z1| lies within its bound of l1."""

    def __init__(self, ref, bound, ratio, ambiguous):
        self.ref, self.bound, self.ratio, self.ambiguous = ref, bound, ratio, ambiguous

    def worst(self):
        return {o: float(r.max(initial=0.0)) for o, r in self.ratio.items()}


def _ratio(gpu, ref, bound):
    gpu = np.asarray(gpu, dtype=np.float64)
    err = np.abs(gpu - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    r[~np.isfinite(gpu)] = np.inf
    return r


def check(kind, hp, before, g, after, dg=0.0, steps=0, touched=True, dense=False):
    """Compare one update: before = (w, s1, s2) the kernel read (fp32), g its gradient (known to within dg), after = (w', s1',
    s2') it wrote.  Adam: `steps` steps done before this one, touched = the row took a gradient (sparse form only).  Slots an
    optimizer does not have (s1, s2 of SGD; s2 of Adagrad) must come back unchanged: they are checked with a zero bound."""
    w, s1, s2 = before
    q = _run(kind, hp, w, s1, s2, g, steps, touched, dense, QOPS)
    lt = _lr_t(kind, hp, steps, F64)
    dg = np.asarray(dg, dtype=np.float64)
    gm = np.asarray(g, dtype=np.float64)
    sens = [np.zeros_like(q[i].v) for i in range(3)]
    if np.any(dg > 0):
        for sgn in (1.0, -1.0):
            alt = _update(kind, hp, F64.leaf(w), F64.leaf(s1), F64.leaf(s2), gm + sgn * dg, lt, touched, dense, F64)
            for i in range(3):
                sens[i] = np.maximum(sens[i], np.abs(alt[i] - q[i].v))
    ref, bound, ratio = {}, {}, {}
    for i, o in enumerate(OUTS):
        ref[o] = np.broadcast_to(q[i].v, np.shape(after[i])).astype(np.float64)
        bound[o] = q[i].k * U * q[i].M * SECOND_ORDER + sens[i] + ulp32(q[i].v) if q[i].k else np.zeros_like(ref[o])
        bound[o] = np.broadcast_to(bound[o], ref[o].shape)
        ratio[o] = _ratio(after[i], ref[o], bound[o])
    amb = np.zeros(np.shape(after[0]), dtype=bool)
    if kind == "ftrl":
        z, wn = q[3]
        l1 = f32(hp["l1"])
        bz = z.k * U * z.M * SECOND_ORDER + sens[2] + ulp32(z.v)
        amb = np.abs(np.abs(z.v) - l1) <= bz
        live = np.abs(z.v) > l1
        ref["w"] = np.where(live, wn.v, 0.0)
        gw = np.asarray(after[0], dtype=np.float64)
        r_live = _ratio(gw, wn.v, bound["w"])
        r_zero = np.where(gw == 0, 0.0, np.inf)
        ratio["w"] = np.where(amb, np.minimum(r_live, r_zero), np.where(live, r_live, r_zero))
        ratio["w"][~np.isfinite(gw)] = np.inf
    return Result(ref, bound, ratio, amb)
