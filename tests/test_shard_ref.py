"""The row-sharded step's checks (tests/shard_ref.py) on the CPU: the fp32 emulation of the owners' gradient sums, the two-shot
all-reduce and the Adam untouched pass meets them at G = 2, 3, 5 and 16 (a rank with one example among them); each planted defect
fails them by at least 100x or as an exact mismatch; the keep mask of a rank's row is the global row's.  Run with -s to see the
worst healthy ratio and every defect's failure factor."""
import numpy as np
import pytest

from oracle.model import drop_keep
from tests import kernel_ref as KR
from tests import optimizer_ref as R
from tests import shard_ref as SR

GS = [2, 3, 5, 16]
MAX_B = 24
N_ROWS = 61                                  # not a multiple of any G: the last local row of some owners is padding
HEALTHY = {}
FACTOR = {}
ADAM = dict(lr=0.05, beta1=0.8, beta2=0.999, epsilon=1e-8)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print()
    for k, v in sorted(HEALTHY.items()):
        print("healthy %-16s worst ratio %.3g" % (k, v))
    for k, v in sorted(FACTOR.items()):
        print("defect  %-20s fails by %s" % (k, "exact mismatch" if v == np.inf else "%.3g x" % v))


def scenario(G, rng, dim=8):
    """Per-rank batch sizes 1 .. MAX_B (the last rank has one example), bags of 1 - 6 ids of which row 0 is in every bag (a hot row
    with occurrences on every rank), gradient rows with stale values past each rank's batch, fp32 bag scales."""
    Bs = [int(rng.integers(2, MAX_B + 1)) for _ in range(G - 1)] + [1]
    grad, scale, rows, ranks, bags = [], [], [], [], []
    for r, b in enumerate(Bs):
        g = (rng.standard_normal((MAX_B, dim)) * 10.0 ** rng.uniform(-2, 2, (MAX_B, 1))).astype(np.float32)
        g[b:] = 1e4                                              # (stale rows: a read past the batch shows)
        n = rng.integers(1, 7, size=MAX_B)
        for e in range(b):
            ids = [0] + list(rng.integers(1, N_ROWS, size=n[e] - 1))
            rows += ids
            ranks += [r] * len(ids)
            bags += [e] * len(ids)
        grad.append(g)
        scale.append(SR.f32_recip(n).astype(np.float32))
    return Bs, grad, scale, np.array(rows), np.array(ranks), np.array(bags)


def rows_ratio(G, rng, defect=None, wide=False):
    Bs, grad, scale, rows, ranks, bags = scenario(G, rng, dim=1 if wide else 8)
    if wide:
        scale = [np.ones(MAX_B, dtype=np.float32)] * G
    cnt = np.bincount(rows, minlength=N_ROWS)
    assert cnt[0] > SR.K_CHUNK and len(set(ranks[rows == 0])) == G      # the chunked combine runs on occurrences of every rank
    out, ref, mag = SR.owner_sums(rows, ranks, bags, grad, scale, G, N_ROWS, defect)
    full = SR.interleave(out, N_ROWS)
    assert not np.any(full[cnt == 0]) or defect, "an untouched row changed"
    C = (int(cnt.max()) + 2) * KR.U
    return KR.compare("rows", full, ref, mag, None, C).worst1


@pytest.mark.parametrize("G", GS)
@pytest.mark.parametrize("wide", [False, True])
def test_owner_sums_healthy(G, wide):
    w = rows_ratio(G, np.random.default_rng(G), wide=wide)
    HEALTHY["owner sums"] = max(HEALTHY.get("owner sums", 0.0), w)
    assert w <= 1.0


@pytest.mark.parametrize("defect", ["own_bag_scale", "pull_rank0", "local_row_mod", "drop_chunk"])
@pytest.mark.parametrize("G", [2, 3, 5])
def test_owner_sums_defects(G, defect):
    w = rows_ratio(G, np.random.default_rng(G), defect=defect)
    FACTOR[defect] = min(FACTOR.get(defect, np.inf), w)
    assert w >= 100, (defect, w)


def arenas(G, n, rng):
    return [(rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(np.float32) for _ in range(G)]


def ar_ratio(G, n, rng, defect=None):
    """Worst ratio of every rank's all-reduced arena to the float64 sum, inf where two ranks' results differ."""
    a = arenas(G, n, rng)
    outs = SR.all_reduce(a, defect)
    ref = np.sum([x.astype(np.float64) for x in a], axis=0)
    M = np.sum([np.abs(x.astype(np.float64)) for x in a], axis=0)
    w = max(KR.compare("arena", o, ref, M, None, (G - 1) * KR.U).worst1 for o in outs)
    return w if all(np.array_equal(outs[0], o) for o in outs) else np.inf


SIZES = [4, 8, 36, 4 * 37, 4 * 100]


@pytest.mark.parametrize("G", GS)
def test_all_reduce_healthy(G):
    """Arenas of 1, 2, 9, 37 and 100 float4s: fewer float4s than ranks (empty trailing slices), and short last slices."""
    rng = np.random.default_rng(100 + G)
    for n in SIZES:
        n4 = n // 4
        s4 = (n4 + G - 1) // G
        w = ar_ratio(G, n, rng)
        HEALTHY["all-reduce"] = max(HEALTHY.get("all-reduce", 0.0), w)
        assert w <= 1.0, (G, n, w)
        if n4 < G:
            assert (G - 1) * s4 >= n4                           # (the premise: the last rank's slice is empty)


@pytest.mark.parametrize("defect", ["ar_drop_rank", "ar_drop_last_slice", "ar_shift_last_slice"])
@pytest.mark.parametrize("G", [2, 3, 5, 16])
def test_all_reduce_defects(G, defect):
    rng = np.random.default_rng(200 + G)
    for n in SIZES:
        w = ar_ratio(G, n, rng, defect)
        FACTOR[defect] = min(FACTOR.get(defect, np.inf), w)
        assert w >= 100, (G, n, defect, w)


def untouched_ratio(G, rng, defect=None):
    """Adam rows no rank touched: the pass's moves applied to fp32 (w, m, v), checked with optimizer_ref against one move."""
    touched = rng.random(N_ROWS) < 0.4
    touched[-1] = False                                         # (the last row sits in the owners' last, partial round of rows)
    count = SR.untouched_moves(N_ROWS, G, touched, defect)
    if defect is None:
        assert np.array_equal(count, (~touched).astype(np.int64))
    w = rng.standard_normal(N_ROWS).astype(np.float32)
    m = (rng.standard_normal(N_ROWS) * 0.1).astype(np.float32)
    v = (10.0 ** rng.uniform(-6, 0, N_ROWS)).astype(np.float32)
    sel = ~touched
    after = [w[sel].copy(), m[sel].copy(), v[sel].copy()]
    for i, k in enumerate(count[sel]):
        for _ in range(int(k)):
            a = R.emulate("adam", ADAM, after[0][i], after[1][i], after[2][i], np.float32(0), steps=3, touched=False)
            for j in range(3):
                after[j][i] = a[j]
    res = R.check("adam", ADAM, (w[sel], m[sel], v[sel]), np.zeros(int(sel.sum()), dtype=np.float32), tuple(after), steps=3,
                  touched=False)
    return max(res.worst().values())


@pytest.mark.parametrize("G", GS)
def test_adam_untouched_healthy(G):
    w = untouched_ratio(G, np.random.default_rng(300 + G))
    HEALTHY["adam untouched"] = max(HEALTHY.get("adam untouched", 0.0), w)
    assert w <= 1.0


@pytest.mark.parametrize("defect", ["untouched_none", "untouched_twice"])
@pytest.mark.parametrize("G", [2, 3, 5])
def test_adam_untouched_defects(G, defect):
    w = untouched_ratio(G, np.random.default_rng(300 + G), defect)
    FACTOR[defect] = min(FACTOR.get(defect, np.inf), w)
    assert w >= 100, (defect, w)


@pytest.mark.parametrize("G", [2, 3, 5])
def test_dropout_mask_rows(G):
    """Rank r's row m takes the mask of global row r * max_batch + m: with full batches it is the one-GPU mask of the concatenated
    batch, no two ranks share a mask, and a mask drawn from the local row (the planted defect) differs."""
    seed, step, layer, width, rate = 0x5EED0006, 7, 65, 40, 0.25
    full = SR.group_keep(seed, step, layer, [r * MAX_B for r in range(G)], [MAX_B] * G, width, rate)
    assert np.array_equal(full, drop_keep(seed, step, layer, G * MAX_B, width, rate))
    for r in range(1, G):
        assert not np.array_equal(full[:MAX_B], full[r * MAX_B:(r + 1) * MAX_B])
    Bs = [MAX_B - 3 * r for r in range(G)]
    ragged = SR.group_keep(seed, step, layer, [r * MAX_B for r in range(G)], Bs, width, rate)
    local = SR.group_keep(seed, step, layer, [r * MAX_B for r in range(G)], Bs, width, rate, local=True)
    assert np.array_equal(ragged[:Bs[0]], full[:Bs[0]])
    assert np.array_equal(ragged[Bs[0]:Bs[0] + Bs[1]], full[MAX_B:MAX_B + Bs[1]])
    mism = int((ragged != local).sum())
    FACTOR["local_row_mask"] = np.inf
    assert mism > 0
