"""Float64 reference of the sparse half of the forward and of what the head hands back: the deep input X0, the wide logit, the
logits, the batch loss and the eval metrics, recomputed from the values the GPU itself read.

The ids are the GPU's own (``pm.column_ids()``; ``check_transform`` holds them to the oracle's ``transform``), the tables are the
fp32 values ``get_tensor`` returns, the dense features are the raw fp32 batch, and the loss and the metrics start from the GPU's
own fp32 logits.  So every kernel is judged on its own error only.  U = 2^-24 (unit roundoff of fp32); every bound below is
derived from the operations of the kernel, none is fitted to a measurement.

Deep input X0 [B, d0_phys] (``x0_reference``), per element a reference and a bound (bound 0: bit-exact):

- Embedding bag, combiner mean, n ids with rows r_i (emb_pool_fwd_rows_kernel, emb_pool_fwd_kernel, the host-table staging
  through the same kernels, shard_serve_emb + shard_combine_emb): ref = sum r_i / n.
  n = 0: exactly 0 (the kernels store a zero accumulator).  n = 1: the row itself, bit for bit (no add, no scale: the local kernels
  skip the mean at n = 1 and the combine's scale is fl(1/1) = 1 on a zero-initialised accumulator).
  n >= 2: any order of n - 1 fp32 adds errs by at most (n - 1) U sum|r_i| (sequential walk, lane-group striding plus xor tree,
  per-owner runs: all are binary trees of the n rows); the kernels then multiply by fl(1/n) = (1 + d1) / n and round the product
  (1 + d2): 2 U |sum| / n more.  So |gpu - ref| <= (n + 1) U sum|r_i| / n, plus ulp32(ref) for the second-order terms.  A
  row-sharded bag adds up to G owner partials onto a zero accumulator: at most G more roundings, (n + G + 1).
- Lanes between a table's logical width and the next multiple of 4, and every column the layout leaves unused: exactly 0.
- Indicator columns: exact integer counts of the GPU's ids (vocab OOV tokens and identity -1 are dropped by the id transform, so
  they count nothing; identity values below -1 or >= buckets map to id 0, as TensorFlow's default_value does).
- Numeric columns: none, min_max and standard are bit-exact to numpy's correctly rounded fp32 (x - a) / b (``__fsub_rn`` and
  ``__fdiv_rn`` in the kernel; for min_max b is the span hi - lo the plan computes on the host).  log: CUDA's logf has a maximum
  error of 1 ulp (CUDA C Programming Guide, mathematical functions); the float64 log is not rounded to fp32, which adds at most
  half an ulp: bound 2 ulp32(ref).  x = 0 gives -inf and x < 0 NaN, exactly, on both sides.

Wide logit (``wide_reference``; wide_fwd_kernel: lanes stride over the example's entries, ``warp_sum``, then + bias):
bias + sum w over the example's n_b wide ids.  The adds of zeros for the entries of non-wide columns are exact, so the n_b weights
and the bias go through a binary tree: lane sums, five xor levels and the bias add; (n_b + 7) U (|bias| + sum|w|) bounds it with
room to spare.  A row-sharded wide column adds its owner partials onto the logit: + G.

Logits of towers (``logit_reference``): the head is an fp32 FMA chain over the logits layer's inputs plus the wide logit; the kernel
reference ``StepRef.head`` gives the logit, Mlogit (the same sums on absolute values) and Khead (the longest accumulation), and
|gpu - ref| <= (Khead + 2) U Mlogit + ulp32(ref), the quantity the gradient check already carries for dlogit.

Loss (``loss_reference``; logits_head_kernel):  t_b = fl(w * fl(fl(max(x, 0) - fl(x y)) + log1pf(expf(-|x|)))).
With a = max(x, 0), e = exp(-|x|), l1 = log1p(e):  fl(x y) errs by U |x y|; the subtraction by U (|a| + |x y|); expf has a
maximum error of 2 ulp (the Programming Guide's table), i.e. 4 U e, which moves log1p by at most 4 U e (its derivative is <= 1);
log1pf adds 1 ulp = 2 U l1; the add U (|a| + |x y| + l1) and the weight product U |w| (|a| + |x y| + l1).  To first order
    E_b = |w| U (3 |a| + 4 |x y| + 4 e + 4 l1),
scaled by (1 + 2^-20) for the second-order terms (and valid when the compiler contracts x y into an FMA: one rounding fewer).  The
sum: lig-0 lanes add their examples in sequence (n_l = ceil(B / (4 * 8 * blocks)) terms), two xor levels combine a warp's four
lanes, thread 0 adds the block's eight warp partials onto 0 (seven roundings), and the last block sums the partials in double
(2^-44 of the sum covers 512 double adds) before one rounding to fp32: (n_l + 8) U sum|t_b| + sum E_b + 2^-44 sum|t_b| +
ulp32(ref).  A LocalShardGroup's loss is the double sum of its ranks' fp32 losses: the sum of their bounds (+ 2^-44).

Eval metrics (``metrics_reference``; metrics_kernel + metrics_finish).  The kernel bins p' = fl(1 / fl(1 + expf(-x))) by the
count of fp32 thresholds strictly below it.  p' = p (1 + d) with |d| <= 2 U + 4 U (1 - p) (expf's 4 U relative error enters
through e / (1 + e) = 1 - p; the add and the division one U each), so an example whose float64 p lies within
dp = (2 + 4 (1 - p)) U p (1 + 2^-20) of a threshold may land in either neighbouring bin: it is *ambiguous*.  (This is the derived
width of the ambiguity band; it is up to six fp32 ulps of p, wider than the two ulps a naive estimate gives.)  AUC and AUPR are
evaluated with the kernel's own trapezoid formulas for every assignment of the ambiguous examples, and the GPU value must lie in
[min, max] +- 1e-12.  accuracy, precision, recall, label/mean and accuracy_baseline depend only on x > 0 and the labels: 1e-12
relative (the accumulators are double).  average_loss, loss and prediction/mean carry the per-element E_b and dp.

The fp32 emulations (``emu_*``) compute what each kernel computes, in its own summation order.  They let the CPU suite pin the
checker down before any GPU runs: the healthy kernels pass every bound, planted defects fail by a wide margin.  They are not
compared bit for bit with the GPU.
"""
import itertools

import numpy as np

from tests.kernel_ref import StepRef, ulp32

U = 2.0 ** -24
F32 = np.float32
NORM_NONE, NORM_MINMAX, NORM_STANDARD, NORM_LOG = 0, 1, 2, 3
N_THR = 200
# the kernel's fp32 thresholds (misc.cu metrics_setup): -1e-7, i / 199 for i = 1 .. 198, 1 + 1e-7
THR32 = np.array([0.0 - 1e-7] + [(i + 1) * 1.0 / (N_THR - 1) for i in range(N_THR - 2)] + [1.0 + 1e-7],
                 dtype=np.float32).astype(np.float64)
METRIC_KEYS = ["accuracy", "accuracy_baseline", "auc", "auc_precision_recall", "average_loss", "label/mean", "loss",
               "precision", "prediction/mean", "recall"]


# ------------------------------------------------------------------------------------------------ judging
class Result(object):
    """worst = max |gpu - ref| / bound over the compared elements (passes at <= 1; inf where an exact element differs)."""

    def __init__(self, name, worst, where, n):
        self.name, self.worst, self.where, self.n = name, worst, where, n

    def __repr__(self):
        return "%s: worst %.3g at %s (%d elements)" % (self.name, self.worst, self.where, self.n)


def judge(name, gpu, ref, bound):
    """bound 0 means bit-exact (NaN matches NaN, -inf matches -inf); otherwise |gpu - ref| <= bound with finite gpu."""
    gpu, ref = np.asarray(gpu, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), ref.shape)
    assert gpu.shape == ref.shape, (name, gpu.shape, ref.shape)
    if gpu.size == 0:
        return Result(name, 0.0, None, 0)
    exact = bound == 0
    same = (gpu == ref) | (np.isnan(gpu) & np.isnan(ref))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(exact, np.where(same, 0.0, np.inf), np.abs(gpu - ref) / np.where(exact, 1.0, bound))
    r[~exact & ~np.isfinite(gpu)] = np.inf
    i = np.unravel_index(int(np.argmax(r)), r.shape)
    return Result(name, float(r[i]), tuple(int(v) for v in i), int(r.size))


# ------------------------------------------------------------------------------------------------ ids
def column_bags(plan, offs, ids, B, col):
    """(example of each id, id, count per example) of one column of the GPU's CSR."""
    C = len(plan.columns)
    ci = plan._col_index[id(col)]
    s, e = offs[ci:B * C:C].astype(np.int64), offs[ci + 1:B * C + 1:C].astype(np.int64)
    n = e - s
    rows = np.repeat(np.arange(B), n)
    pos = np.concatenate([np.arange(a, b) for a, b in zip(s, e)] + [np.zeros(0, dtype=np.int64)])
    return rows, np.asarray(ids)[pos].astype(np.int64), n


def check_transform(om, plan, offs, ids, raw, B):
    """The GPU's ids equal the oracle's transform of the raw batch, column by column (so the reference cannot drift from it)."""
    ref = om.transform(raw)
    C = len(plan.columns)
    for ci, col in enumerate(plan.columns):
        if col.name not in ref:
            continue
        ro, ri = ref[col.name]
        got_n = offs[ci + 1:B * C + 1:C] - offs[ci:B * C:C]
        assert np.array_equal(got_n, np.diff(ro)), "column %s: id counts differ from the oracle" % col.name
        _, got, _ = column_bags(plan, offs, ids, B, col)
        assert np.array_equal(got, ri), "column %s: ids differ from the oracle" % col.name


# ------------------------------------------------------------------------------------------------ deep input
def numeric_fp32(kind, a, b, x):
    """The kernel's normalise in fp32: (x - a) / b correctly rounded for min_max / standard, x for none (log: not exact)."""
    x = np.asarray(x, dtype=np.float32)
    if kind in (NORM_MINMAX, NORM_STANDARD):
        return (x - F32(a)) / F32(b)
    assert kind == NORM_NONE
    return x


def bag_reference(S, A, n, extra=0):
    """-> (ref, bound) of mean-combined bags from their float64 row sums S [B, w], sums of |rows| A and id counts n [B]; extra:
    the owner partials a row-sharded combine adds (G)."""
    nn = np.maximum(n, 1)[:, None].astype(np.float64)
    val = S / nn
    bnd = (n[:, None] + 1 + extra) * U * A / nn + ulp32(val)
    bnd[n <= 1] = 0.0
    return val, bnd


def x0_reference(plan, offs, ids, B, tables, dense, G=1):
    """-> (ref, bound, kind) [B, d0_phys]: float64 reference, bound (0 = bit-exact) and the kind of each element ('bag',
    'indicator', 'numeric', 'log', 'pad').  tables: embedding table name -> fp32 [rows, dim] (full tables); dense: fp32 [B, n_dense]
    raw features; G: ranks of a row-sharded group (its sharded tables take the combine's extra roundings)."""
    P = plan.d0_phys
    ref, bound = np.zeros((B, P)), np.zeros((B, P))
    kind = np.full(P, "pad", dtype=object)
    for tb in plan.tables:
        lo, po, w = plan.deep_layout[tb["name"]]
        rows, idv, n = column_bags(plan, offs, ids, B, tb["column"])
        W = np.asarray(tables[tb["name"]], dtype=np.float64)
        assert W.shape[1] == w, (tb["name"], W.shape, w)
        r = W[idv]
        S, A = np.zeros((B, w)), np.zeros((B, w))
        np.add.at(S, rows, r)
        np.add.at(A, rows, np.abs(r))
        ref[:, po:po + w], bound[:, po:po + w] = bag_reference(S, A, n, G if tb["sharded"] and G > 1 else 0)
        kind[po:po + w] = "bag"
    for c in plan.columns:
        if c.ind_off >= 0:
            rows, idv, _ = column_bags(plan, offs, ids, B, c)
            np.add.at(ref, (rows, c.ind_off + idv), 1.0)
            kind[c.ind_off:c.ind_off + c.buckets] = "indicator"
    dense = np.asarray(dense, dtype=np.float32).reshape(B, -1)
    for nm in plan.numerics:
        k, a, b = nm["norm"]
        x = dense[:, nm["field"]]
        o = nm["x0_off"]
        if k == NORM_LOG:
            x64 = x.astype(np.float64)
            with np.errstate(divide="ignore", invalid="ignore"):
                v = np.log(x64)
            ref[:, o] = v
            bound[:, o] = np.where(x64 > 0, 2 * ulp32(v), 0.0)
            bound[:, o][(x64 > 0) & (v == 0)] = 0.0          # logf(1) = 0 exactly
            kind[o] = "log"
        else:
            ref[:, o] = numeric_fp32(k, a, b, x)
            kind[o] = "numeric"
    return ref, bound, kind


def check_x0(name, X0, ref, bound, kind):
    """-> {kind: Result} over the whole physical row (every padding column is compared too)."""
    out = {}
    for kd in ("bag", "indicator", "numeric", "log", "pad"):
        cols = np.nonzero(kind == kd)[0]
        if len(cols):
            out[kd] = judge("%s %s" % (name, kd), X0[:, cols], ref[:, cols], bound[:, cols])
    return out


# ------------------------------------------------------------------------------------------------ wide logit, logits, loss
def wide_reference(plan, offs, ids, B, wide, bias, G=1):
    """-> (ref, bound) of the wide logit.  wide: wide column name -> fp32 weights (full); bias: the fp32 bias."""
    ref, A, nb = np.full(B, float(bias)), np.full(B, abs(float(bias))), np.zeros(B)
    sharded = False
    for ci, c in enumerate(plan.columns):
        if c not in plan.wide_columns:
            continue
        rows, idv, n = column_bags(plan, offs, ids, B, c)
        w = np.asarray(wide[c.name], dtype=np.float64)
        np.add.at(ref, rows, w[idv])
        np.add.at(A, rows, np.abs(w[idv]))
        nb += n
        sharded |= G > 1 and bool(plan.wide_sharded[ci])
    return ref, wide_bound(A, nb, G if sharded else 0)


def wide_bound(A, nb, extra=0):
    """Bound of a wide logit: A = |bias| + sum |w| per example, nb = its wide ids, extra = the owner partials of sharded columns."""
    return (nb + 7 + extra) * U * A


def logit_reference(pm, batch, params, engine):
    """-> (ref, bound) of the logits a wide_deep / deep forward returns, from the GPU's deep input and hidden outputs."""
    logit, Mlogit, _, Khead, _ = StepRef(pm, batch, params, engine).head()
    return logit, (Khead + 2) * U * Mlogit + ulp32(logit)


def loss_terms(x, y, w):
    """-> (float64 w * loss per example, its per-element fp32 error bound E_b)."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    w = np.ones_like(x) if w is None else np.asarray(w, dtype=np.float64)
    a, e = np.maximum(x, 0.0), np.exp(-np.abs(x))          # (exp of a non-positive number cannot overflow)
    l1 = np.log1p(e)
    t = w * (a - x * y + l1)
    E = np.abs(w) * U * (3 * np.abs(a) + 4 * np.abs(x * y) + 4 * e + 4 * l1) * (1 + 2.0 ** -20)
    return t, E


def head_blocks(B):
    return min(max((B * 8 + 255) // 256, 1), 512)


def loss_reference(x, y, w):
    """-> (ref, bound) of the batch loss logits_head_kernel returns for the fp32 logits x."""
    B = len(x)
    t, E = loss_terms(x, y, w)
    n_l = -(-B // (4 * 8 * head_blocks(B)))
    ref = t.sum()
    T = np.abs(t).sum()
    return ref, (n_l + 8) * U * T + E.sum() + 2.0 ** -44 * T + float(ulp32(ref))


# ------------------------------------------------------------------------------------------------ eval metrics
def _auc_aupr(pos, neg):
    """metrics_finish's trapezoids over the 201-bin histograms (float64)."""
    eps = 1e-7
    P, N = pos.sum(), neg.sum()
    tp = np.cumsum(pos[::-1])[::-1][1:]                 # tp[t] = sum_{k > t} pos[k]
    fp = np.cumsum(neg[::-1])[::-1][1:]
    rec = (tp + eps) / (P + eps)
    fpr = fp / (N + eps)
    prec = (tp + eps) / (tp + fp + eps)
    auc = ((fpr[:-1] - fpr[1:]) * (rec[:-1] + rec[1:]) / 2.0).sum()
    aupr = ((rec[:-1] - rec[1:]) * (prec[:-1] + prec[1:]) / 2.0).sum()
    return auc, aupr


def prob_bound(p):
    return (2 + 4 * (1 - p)) * U * p * (1 + 2.0 ** -20)


def metrics_reference(x, y, w, n_batches, max_ambiguous=12):
    """-> dict key -> (lo, hi): the interval each of the ten metrics must lie in (before the 1e-12 tolerances of
    ``check_metrics``), for the fp32 logits x of every evaluated example, labels y, weights w (None: ones)."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    w = np.ones_like(x) if w is None else np.asarray(w, dtype=np.float64)
    with np.errstate(over="ignore"):
        p = 1.0 / (1.0 + np.exp(-x))
    dp = prob_bound(p)
    # p' lies in [p - dp, p + dp] and, being 1 / fl(1 + e) with e >= 0, in [0, 1]: its bin is the count of thresholds below it
    lo_bin = np.searchsorted(THR32, np.maximum(p - dp, 0.0), side="left")
    hi_bin = np.searchsorted(THR32, np.minimum(p + dp, 1.0), side="left")
    amb = np.nonzero(lo_bin != hi_bin)[0]
    assert len(amb) <= max_ambiguous, "%d ambiguous examples: too many to enumerate" % len(amb)
    ispos = y > 0.5
    pos, neg = np.zeros(N_THR + 1), np.zeros(N_THR + 1)
    sure = np.setdiff1d(np.arange(len(x)), amb)
    np.add.at(pos, lo_bin[sure][ispos[sure]], w[sure][ispos[sure]])
    np.add.at(neg, lo_bin[sure][~ispos[sure]], w[sure][~ispos[sure]])
    aucs, auprs = [], []
    for choice in itertools.product((0, 1), repeat=len(amb)):
        ps, ns = pos.copy(), neg.copy()
        for i, c in zip(amb, choice):
            (ps if ispos[i] else ns)[hi_bin[i] if c else lo_bin[i]] += w[i]
        a, b = _auc_aupr(ps, ns)
        aucs.append(a)
        auprs.append(b)
    t, E = loss_terms(x, y, w)
    sw = w.sum()
    cls = (x > 0).astype(np.float64)
    lm = (w * y).sum() / sw
    tp, fp, fn = (w * cls * y).sum(), (w * cls * (1 - y)).sum(), (w * (1 - cls) * y).sum()
    pt = lambda v: (v, v)
    out = {"accuracy": pt((w * (cls == y)).sum() / sw), "accuracy_baseline": pt(max(lm, 1 - lm)),
           "auc": (min(aucs), max(aucs)), "auc_precision_recall": (min(auprs), max(auprs)), "label/mean": pt(lm),
           "precision": pt(tp / (tp + fp) if tp + fp > 0 else 0.0), "recall": pt(tp / (tp + fn) if tp + fn > 0 else 0.0)}
    el = E.sum() / abs(sw)
    out["average_loss"] = (t.sum() / sw - el, t.sum() / sw + el)
    eb = E.sum() / n_batches
    out["loss"] = (t.sum() / n_batches - eb, t.sum() / n_batches + eb)
    ep = (np.abs(w) * dp).sum() / abs(sw)
    out["prediction/mean"] = ((w * p).sum() / sw - ep, (w * p).sum() / sw + ep)
    return out


def check_metrics(got, ref):
    """-> Result: worst over the ten metrics of the distance outside [lo, hi], over the allowed tolerance (1e-12 absolute for AUC
    and AUPR, 1e-12 relative otherwise, on top of the interval)."""
    ratio = {}
    for k in METRIC_KEYS:
        lo, hi = ref[k]
        tol = 1e-12 if k.startswith("auc") else 1e-12 * max(abs(lo), abs(hi), 1e-300)
        g = got[k]
        d = 0.0 if lo <= g <= hi else min(abs(g - lo), abs(g - hi))
        ratio[k] = d / tol if np.isfinite(g) else np.inf
    where = max(ratio, key=ratio.get)
    return Result("metrics", ratio[where], where, len(METRIC_KEYS))


# ------------------------------------------------------------------------------------------------ fp32 emulations
def _f4(v):
    return np.asarray(v, dtype=np.float32)


def emu_rows_bag(rows, defect=None):
    """emb_pool_fwd_rows_kernel on one bag: sequential fp32 walk, then * fl(1/n) for n > 1."""
    n = len(rows)
    if n == 0:
        return None if defect == "stale_empty" else np.zeros(rows.shape[1], dtype=np.float32)
    acc = _f4(rows[0]).copy()
    for j in range(1, n):
        acc = acc + _f4(rows[j])
    if n > 1 and not (defect == "no_mean_2" and n == 2):
        acc = acc * (F32(1.0) / F32(n))
    return acc


def emu_warp_bag(rows, G, defect=None):
    """emb_pool_fwd_kernel on one bag: lane group g sums rows g, g + 32/G, ... of each 32-id chunk in turn (RND rows in flight
    change no order), then the xor tree over the groups, then * fl(1/n) for n > 1."""
    n, D = rows.shape
    GROUPS = 32 // G
    acc = np.zeros((GROUPS, D), dtype=np.float32)
    for j0 in range(0, n, 32):
        cnt = min(32, n - j0)
        for r in range(cnt):
            if defect == "drop_33" and j0 + r == 32:
                continue
            acc[r % GROUPS] = acc[r % GROUPS] + _f4(rows[j0 + r])
    s = 1
    while s < GROUPS:
        acc = acc + acc[np.arange(GROUPS) ^ s]
        s <<= 1
    out = acc[0]
    if n > 1 and not (defect == "no_mean_2" and n == 2):
        out = out * (F32(1.0) / F32(n))
    return out


def emu_shard_bag(rows, ids, G, defect=None):
    """shard_serve_emb + shard_combine_emb on one bag: owner o = id mod G sums its ids of the bag in order, the requester adds
    the partials of the owners present in bagmask in rank order onto 0, then * fl(1/n) (a zero scale for an empty bag)."""
    n, D = rows.shape
    acc = np.zeros(D, dtype=np.float32)
    owners = [o for o in range(G) if np.any(ids % G == o)]
    if defect == "drop_owner" and len(owners) > 1:
        owners = owners[1:]
    for o in owners:
        sel = np.nonzero(ids % G == o)[0]
        part = _f4(rows[sel[0]]).copy()
        for j in sel[1:]:
            part = part + _f4(rows[j])
        acc = acc + part
    scale = F32(1.0) / F32(n) if n else F32(0.0)
    return acc * scale


def emu_wide(entries, bias, defect=None):
    """wide_fwd_kernel on one example: lane l sums entries l, l + 32, ... (0 for entries of non-wide columns), warp_sum's xor
    tree (16, 8, 4, 2, 1), then + bias."""
    lanes = np.zeros(32, dtype=np.float32)
    for j, v in enumerate(entries):
        lanes[j % 32] = lanes[j % 32] + F32(v)
    for d in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ d]
    out = lanes[0] + F32(bias)
    return out + F32(bias) if defect == "bias_twice" else out


def emu_loss(x, y, w, defect=None):
    """logits_head_kernel's loss: per-example fp32 terms (libm exp / log1p rounded to fp32 stand in for expf / log1pf), lane
    sums in grid-stride order, the two xor levels, the block's eight warps, the block partials in double, rounded to fp32."""
    x, y = _f4(x), _f4(y)
    w = np.ones_like(x) if w is None else _f4(w)
    B = len(x)
    e = np.exp(-np.abs(x).astype(np.float64)).astype(np.float32)
    l1 = np.log1p(e.astype(np.float64)).astype(np.float32)
    t = w * ((np.maximum(x, F32(0)) - x * y) + l1)
    if defect == "drop_example":
        t[B // 2] = 0
    blocks = head_blocks(B)
    nw = blocks * 8
    lane = np.zeros((blocks, 8, 4), dtype=np.float32)              # (block, warp, lig-0 lane of the warp's four examples)
    for b0 in range(0, B, nw * 4):
        for k in range(min(nw * 4, B - b0)):
            wg, g = divmod(k, 4)
            lane[wg // 8, wg % 8, g] = lane[wg // 8, wg % 8, g] + t[b0 + k]
    lane = lane + lane[:, :, [1, 0, 3, 2]]                         # xor 8: example group g with g ^ 1
    lane = lane + lane[:, :, [2, 3, 0, 1]]                         # xor 16: g with g ^ 2
    warp = lane[:, :, 0]
    part = np.zeros(blocks, dtype=np.float32)
    for i in range(8):
        part = part + warp[:, i]
    return float(F32(part.astype(np.float64).sum()))


def emu_metrics(x, y, w, n_batches, defect=None):
    """metrics_kernel + metrics_finish: fp32 p and loss per example, fp32 threshold search, double sums."""
    x32, y32 = _f4(x), _f4(y)
    w32 = np.ones_like(x32) if w is None else _f4(w)
    with np.errstate(over="ignore"):
        e = np.exp((-x32).astype(np.float64)).astype(np.float32)
    p = F32(1.0) / (F32(1.0) + e)
    k = np.searchsorted(THR32, p.astype(np.float64), side="left")
    if defect == "neighbour_bin":
        pv = p.astype(np.float64)
        dist = np.min(np.abs(pv[:, None] - THR32[None, :]), axis=1)
        # a weighted example in the middle of the histogram, well away from every threshold
        i = int(np.argmin(np.where((w32 > 0) & (dist > 1e-4), np.abs(pv - 0.5), np.inf)))
        k[i] = k[i] + 1 if k[i] < N_THR else k[i] - 1
    ispos = y32 > 0.5
    pos, neg = np.zeros(N_THR + 1), np.zeros(N_THR + 1)
    np.add.at(pos, k[ispos], w32[ispos].astype(np.float64))
    np.add.at(neg, k[~ispos], w32[~ispos].astype(np.float64))
    auc, aupr = _auc_aupr(pos, neg)
    el = np.exp(-np.abs(x32).astype(np.float64)).astype(np.float32)
    l = (np.maximum(x32, F32(0)) - x32 * y32) + np.log1p(el.astype(np.float64)).astype(np.float32)
    w64, y64, l64 = w32.astype(np.float64), y32.astype(np.float64), l.astype(np.float64)
    cls = (x32 > 0).astype(np.float64)
    sw = w64.sum()
    lm = (w64 * y64).sum() / sw
    tp, fp, fn = (w64 * cls * y64).sum(), (w64 * cls * (1 - y64)).sum(), (w64 * (1 - cls) * y64).sum()
    return {"accuracy": (w64 * (cls == y64)).sum() / sw, "accuracy_baseline": max(lm, 1 - lm), "auc": auc,
            "auc_precision_recall": aupr, "average_loss": (w64 * l64).sum() / sw, "label/mean": lm,
            "loss": (w64 * l64).sum() / n_batches, "precision": tp / (tp + fp) if tp + fp > 0 else 0.0,
            "prediction/mean": (w64 * p.astype(np.float64)).sum() / sw, "recall": tp / (tp + fn) if tp + fn > 0 else 0.0}
