"""CPU self-test of tests/input_ref.py: the fp32 emulations of the pooling, wide, loss and metrics kernels pass every bound at the
edges where those kernels go wrong, and each planted defect fails by a wide margin.  Run with -s to see the worst ratios."""
import numpy as np
import pytest

from tests import input_ref as IR

LENGTHS = [0, 1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 200, 1000]
RMAX = 4


def table(rng, rows, D):
    """fp32 rows of mixed magnitude: most N(0, 1), every 7th row 1e3 larger, every 11th 1e-3 smaller."""
    W = rng.standard_normal((rows, D))
    W[::7] *= 1e3
    W[::11] *= 1e-3
    return W.astype(np.float32)


def zipf_ids(rng, n, rows):
    return ((rng.zipf(1.3, size=n) - 1) % rows).astype(np.int64)


def ref_bags(W, bags, extra=0):
    """input_ref's bag reference for a list of id arrays of one table."""
    B, D = len(bags), W.shape[1]
    S, A = np.zeros((B, D)), np.zeros((B, D))
    for b, ids in enumerate(bags):
        r = W[ids].astype(np.float64)
        S[b], A[b] = r.sum(0), np.abs(r).sum(0)
    return IR.bag_reference(S, A, np.array([len(i) for i in bags]), extra)


# ------------------------------------------------------------------------------------------------ one bag, every path
def bag_ratio(D, path, defect=None, G=2, seed=0):
    rng = np.random.default_rng(seed)
    W = table(rng, 300, D)
    bags = [zipf_ids(rng, n, 300) for n in LENGTHS]
    if path == "rows":
        got = [IR.emu_rows_bag(W[ids], defect) for ids in bags]
    elif path == "warp":
        got = [IR.emu_warp_bag(W[ids], D // 4, defect) for ids in bags]
    else:
        got = [IR.emu_shard_bag(W[ids], ids, G, defect) for ids in bags]
    prev = np.full(D, 7.0, dtype=np.float32)                         # what the previous batch left in X0
    got = np.stack([prev if g is None else g for g in got])
    ref, bound = ref_bags(W, bags, G if path == "shard" else 0)
    return IR.judge("%s D=%d" % (path, D), got, ref, bound)


@pytest.mark.parametrize("path", ["rows", "warp", "shard"])
def test_healthy_bags_pass(path):
    worst = []
    for D in (4, 8, 16, 32, 64, 128):
        for G in ((2, 3) if path == "shard" else (2,)):
            for seed in range(3):
                res = bag_ratio(D, path, G=G, seed=seed)
                assert res.worst <= 1.0, res
                worst.append(res.worst)
    print("\n%-6s bags: worst healthy ratio %.3g" % (path, max(worst)))


@pytest.mark.parametrize("path,defect,D", [("warp", "drop_33", 32), ("warp", "drop_33", 128), ("rows", "no_mean_2", 8),
                                           ("warp", "no_mean_2", 64), ("rows", "stale_empty", 16), ("shard", "drop_owner", 32)])
def test_planted_bag_defects_fail(path, defect, D):
    res = bag_ratio(D, path, defect)
    print("\n%-10s %-5s D=%-3d ratio %.3g" % (defect, path, D, res.worst))
    assert res.worst > 100, res


# ------------------------------------------------------------------------------------------------ a whole deep input, rows kernel
def rows_kernel(tabs, row_base, data, bags, ntab, D, prev, defect=None):
    """emb_pool_fwd_rows_kernel over one width: per example, rounds of GROUPS * RMAX tables; table k's rows live at global rows
    row_base[k] + id of `data`; its bag lands at x0 = k * D.  Defects: skip_last_round, row_plus1, no_row_base, wrong_x0,
    stale_empty."""
    GROUPS = 32 // (D // 4)
    X0 = prev.copy()
    for b in range(len(bags)):
        rounds = list(range(0, ntab, GROUPS * RMAX))
        if defect == "skip_last_round" and len(rounds) > 1:
            rounds = rounds[:-1]
        for k0 in rounds:
            for k in range(k0, min(k0 + GROUPS * RMAX, ntab)):
                ids = bags[b][k]
                if len(ids) == 0 and defect == "stale_empty":
                    continue
                rb = 0 if defect == "no_row_base" else row_base[k]
                gid = row_base[k] + ids + (1 if defect == "row_plus1" else 0)
                v = IR.emu_rows_bag(data[gid - row_base[k] + rb])
                x0 = k * D
                X0[b, x0:x0 + D] = v
                if defect == "wrong_x0" and D >= 8:
                    X0[b, x0:x0 + 4] = v[4:8]                         # lane group 1 stored at lane group 0's offset
    return X0


def deep_input_ratio(D, ntab, defect=None, seed=0):
    rng = np.random.default_rng(seed)
    rows = [50 + 13 * k for k in range(ntab)]
    tabs = [table(rng, r, D) for r in rows]
    row_base = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64)
    data = np.concatenate(tabs + [table(rng, 1, D)])                  # (one spare row: row id + 1 of the last table stays in range)
    B = len(LENGTHS)
    bags = [[zipf_ids(rng, LENGTHS[(b + k) % B] if k % 3 == 0 else int(rng.integers(0, 4)), rows[k]) for k in range(ntab)]
            for b in range(B)]
    prev = np.full((B, ntab * D), 5.0, dtype=np.float32)
    X0 = rows_kernel(tabs, row_base, data, bags, ntab, D, prev, defect)
    ref, bound = np.zeros((B, ntab * D)), np.zeros((B, ntab * D))
    for k in range(ntab):
        ref[:, k * D:(k + 1) * D], bound[:, k * D:(k + 1) * D] = ref_bags(tabs[k], [bags[b][k] for b in range(B)])
    return IR.judge("deep input D=%d ntab=%d" % (D, ntab), X0, ref, bound)


def test_healthy_rows_kernel_passes_with_a_second_round_of_tables():
    worst = []
    for D, ntab in ((4, 3), (8, 9), (32, 17), (64, 9), (16, 40)):
        res = deep_input_ratio(D, ntab)
        assert res.worst <= 1.0, res
        worst.append(res.worst)
    print("\nrows kernel deep input: worst healthy ratio %.3g" % max(worst))


@pytest.mark.parametrize("defect", ["skip_last_round", "row_plus1", "no_row_base", "wrong_x0", "stale_empty"])
def test_planted_layout_defects_fail(defect):
    res = deep_input_ratio(32, 17, defect)
    print("\n%-16s ratio %.3g" % (defect, res.worst))
    assert res.worst > 100, res


# ------------------------------------------------------------------------------------------------ numeric columns
def numeric_case(kind, a, b, x, defect=None):
    x = np.asarray(x, dtype=np.float32)
    if defect == "reciprocal":
        got = (x - np.float32(a)) * (np.float32(1) / np.float32(b))
    else:
        got = IR.numeric_fp32(kind, a, b, x)
    return IR.judge("numeric", got, IR.numeric_fp32(kind, a, b, x), 0.0)


def test_numeric_exact_and_reciprocal_defect():
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(4096) * 30 + 40).astype(np.float32)
    for kind, a, b in ((IR.NORM_STANDARD, 40.0, 30.0), (IR.NORM_MINMAX, 10.0, 80.0), (IR.NORM_NONE, 0.0, 0.0)):
        assert numeric_case(kind, a, b, x).worst == 0
    res = numeric_case(IR.NORM_STANDARD, 40.0, 30.0, x, "reciprocal")
    print("\nreciprocal   ratio %s" % res.worst)
    assert res.worst == np.inf


def test_log_edges():
    """log at 0 is -inf and below 0 NaN on both sides (bit-exact classes); elsewhere the 2-ulp band holds an fp32-rounded log."""
    x = np.array([0.0, -1.0, -0.0, 1.0, 1e-30, 3.0, 1e30, np.e], dtype=np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = np.log(x.astype(np.float64))
        got = np.log(x).astype(np.float32)
    bound = np.where(x > 0, 2 * IR.ulp32(ref), 0.0)
    bound[(x > 0) & (ref == 0)] = 0
    assert IR.judge("log", got, ref, bound).worst <= 1
    bad = got.copy()
    bad[0] = 0.0                                                     # log(0) must not come out finite
    assert IR.judge("log", bad, ref, bound).worst == np.inf


# ------------------------------------------------------------------------------------------------ wide logit
def wide_ratio(defect=None, seed=0):
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal(500) * 0.1).astype(np.float32)
    w[::9] *= 1e3
    bias = np.float32(0.37)
    got, ref, A, nb = [], [], [], []
    for n in LENGTHS:
        ids = zipf_ids(rng, n, 500)
        # entries of the example in CSR order, with zeros standing for the entries of deep-only columns
        entries = np.concatenate([w[ids], np.zeros(int(rng.integers(0, 40)), dtype=np.float32)])
        rng.shuffle(entries)
        got.append(IR.emu_wide(entries, bias, defect))
        ref.append(float(bias) + w[ids].astype(np.float64).sum())
        A.append(abs(float(bias)) + np.abs(w[ids].astype(np.float64)).sum())
        nb.append(n)
    return IR.judge("wide", np.array(got), np.array(ref), IR.wide_bound(np.array(A), np.array(nb)))


def test_wide_logit():
    res = wide_ratio()
    print("\nwide healthy ratio %.3g" % res.worst)
    assert res.worst <= 1, res
    bad = wide_ratio("bias_twice")
    print("bias_twice   ratio %.3g" % bad.worst)
    assert bad.worst > 100, bad


# ------------------------------------------------------------------------------------------------ loss and metrics
def logits_labels(B, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(B) * 3).astype(np.float32)
    t = np.array([0.25, 0.5, 0.75, 100 / 199.0])                    # probabilities on a threshold (ambiguous examples)
    edge = np.concatenate([[0.0, -0.0, 30.0, -30.0, 90.0, -90.0, 1e-6, -1e-6], np.log(t / (1 - t))]).astype(np.float32)
    x[:min(B, len(edge))] = edge[:B]
    y = (rng.random(B) < 0.3).astype(np.float32)
    w = (rng.random(B) * 2).astype(np.float32)
    w[::5] = 0
    return x, y, w


@pytest.mark.parametrize("B", [1, 65, 4096, 70000])
def test_loss(B):
    x, y, w = logits_labels(B, B)
    ref, bound = IR.loss_reference(x, y, w)
    got = IR.emu_loss(x, y, w)
    r = abs(got - ref) / bound
    print("\nloss B=%-6d healthy ratio %.3g" % (B, r))
    assert r <= 1


@pytest.mark.parametrize("B", [65, 4096, 70000])
def test_loss_dropping_one_example_fails(B):
    x, y, w = logits_labels(B, 1)
    x[B // 2], w[B // 2], y[B // 2] = 2.0, 1.0, 0.0                 # the dropped example's term is about 2.1
    ref, bound = IR.loss_reference(x, y, w)
    bad = abs(IR.emu_loss(x, y, w, "drop_example") - ref) / bound
    print("\ndrop_example B=%-6d ratio %.3g" % (B, bad))
    assert bad > 20


@pytest.mark.parametrize("B", [65, 4096])
def test_metrics(B):
    x, y, w = logits_labels(B, 7 + B)
    ref = IR.metrics_reference(x, y, w, n_batches=3)
    res = IR.check_metrics(IR.emu_metrics(x, y, w, 3), ref)
    print("\nmetrics B=%-5d healthy ratio %.3g" % (B, res.worst))
    assert res.worst <= 1, res
    if B > 100:
        # (one example one bin over moves AUC by about 1 / (P N); with thousands of examples that hides inside the interval the
        # ambiguous ones span, so the defect is planted on the small batch)
        return
    bad = IR.check_metrics(IR.emu_metrics(x, y, w, 3, "neighbour_bin"), ref)
    print("neighbour_bin ratio %.3g (%s)" % (bad.worst, bad.where))
    assert bad.worst > 100, bad
