"""HBM cache of host-table records (Plan(host_cache_bytes=...), wd_host_cache_enable).

A cached record is an exact copy of its host record and the step's kernels see the same values in the same order, so a model
with host tables and a cache must compute exactly what the HBM-resident model computes: the HBM model is the oracle and every
comparison is byte for byte.  The counters are predicted exactly by a short restatement of the policy (set hash, run order, LRU
with way-index tie-break, overflow).
"""
import ctypes
import os
from collections import defaultdict

import numpy as np
import pytest

from oracle import hashing as OH
from tests.helpers import random_raw_batch, to_product_batch
from tests.test_gpu_host_tables import OPTS, _all_tensors, _assert_bytes_equal, _batches, _plan, _train
from tests.test_gpu_parity import small_conf
from wide_deep_b200 import _native
from wide_deep_b200.model import WideDeepModel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WAYS = 8
B = 128
STEPS = 12


def _nslots(plan):
    return {"sgd": 0, "adagrad": 1, "ftrl": 2, "adam": 2, "rmsprop": 2}[plan.dnn_opt["kind"]]


def _stride(plan):
    """Floats per staged record: the widest host record [w | slots]."""
    return max(((t["dim"] + 3) // 4 * 4) * (1 + _nslots(plan)) for t in plan.tables)


def _bytes_for(plan, set_bits):
    return WAYS * (1 << set_bits) * _stride(plan) * 4


def _with_cache(fc, cross, model, gather, set_bits, **kw):
    plan = _plan(fc, cross, model, B, gather, "all", **kw)
    plan.host_cache_bytes = _bytes_for(plan, set_bits) if set_bits is not None else 0
    return plan


def _host_rows(pm):
    """Sorted unique global embedding rows of the model's last batch (every table is on the host in these tests)."""
    offs, ids = pm.column_ids()
    plan = pm.plan
    base, acc = [], 0
    for t in plan.tables:
        base.append(acc)
        acc += t["rows"]
    C = len(plan.columns)
    col = np.repeat(np.tile(np.arange(C), len(offs) // C), np.diff(offs))
    rows = []
    for ci, c in enumerate(plan.columns):
        if c.emb_table < 0:
            continue
        v = ids[col == ci]
        v = v[(v >= 0) & (v < plan.tables[c.emb_table]["rows"])]
        rows.append(v + base[c.emb_table])
    return np.unique(np.concatenate(rows)) if rows else np.zeros(0, np.int64)


class CachePolicy(object):
    """The cache's policy restated: 8-way sets chosen by a Fibonacci hash of the global row; per set, the call's rows in
    ascending order; hits keep their way; misses take the other ways by (last use, way index), empty ways first; rows beyond the
    ways overflow.  Train calls mark every used way dirty; evicting a dirty way counts as a write home."""

    def __init__(self, set_bits):
        self.bits = set_bits
        n = WAYS << set_bits
        self.tag, self.stamp, self.dirty = [None] * n, [0] * n, [False] * n
        self.now = 0
        self.c = dict(hits=0, loads=0, overflow=0, evictions=0)

    def set_of(self, row):
        return ((int(row) * 0x9E3779B1) & 0xFFFFFFFF) >> (32 - self.bits) if self.bits else 0

    def call(self, rows, train):
        self.now += 1
        by_set = defaultdict(list)
        for r in sorted(int(x) for x in rows):
            by_set[self.set_of(r)].append(r)
        for s, rs in by_set.items():
            ways = list(range(s * WAYS, (s + 1) * WAYS))
            used = set()
            for r in rs:
                for w in ways:
                    if self.tag[w] == r:
                        used.add(w)
                        self.c["hits"] += 1
            free = sorted((w for w in ways if w not in used), key=lambda w: (0 if self.tag[w] is None else self.stamp[w], w))
            k = 0
            for r in rs:
                if any(self.tag[w] == r for w in ways):
                    continue
                if k < len(free):
                    w = free[k]
                    k += 1
                    if self.tag[w] is not None and self.dirty[w]:
                        self.c["evictions"] += 1
                    self.c["loads"] += 1
                    self.tag[w], self.dirty[w] = r, False
                    used.add(w)
                else:
                    self.c["overflow"] += 1
            for w in used:
                self.stamp[w] = self.now
                if train:
                    self.dirty[w] = True


def _diverse_batches(plan, fc, n, seed, gather):
    """As test_gpu_host_tables._batches, but h1 and h3 draw from 2^20 tokens instead of 50, so the large tables see new rows every
    step and a cache that holds one step's rows still has to evict over the run."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        raw = random_raw_batch(fc, B, rng, multihot_max=3 if gather == "rows" else 10)
        for f in ("h1", "h3"):
            offs, fp = raw[f]
            raw[f] = (offs, OH.fingerprint64_tokens(["w%d" % rng.integers(0, 1 << 20) for _ in range(len(fp))]))
        out.append(to_product_batch(plan, raw, (rng.random(B) < 0.3).astype(np.float32)))
    return out


def _rows_of(fc, cross, model, gather, batches):
    ref = WideDeepModel(_plan(fc, cross, model, B, gather, []))
    out = []
    for b in batches:
        ref.forward(b)
        out.append(_host_rows(ref))
    ref.close()
    return out


def _pick_bits(rows, want):
    """Smallest set count (power of two) whose simulated training run shows `want` (evictions without overflow, or nothing
    evicted at all)."""
    seen = []
    for bits in range(1, 18):
        p = CachePolicy(bits)
        for r in rows:
            p.call(r, True)
        if p.c["overflow"] == 0 and (p.c["evictions"] > 0) == (want == "medium"):
            return bits
        seen.append((bits, p.c))
    raise AssertionError("no cache size gives a %s cache for these batches: %s" % (want, seen))


@pytest.mark.parametrize("size", ["tiny", "medium", "large"])
@pytest.mark.parametrize("gather", ["rows", "warp"])
@pytest.mark.parametrize("opt", sorted(OPTS))
def test_cached_training_is_bit_identical(opt, gather, size):
    fc, cross, model = small_conf(dnn_opt=OPTS[opt])
    batches = _diverse_batches(_plan(fc, cross, model, B, gather, []), fc, STEPS, 5, gather)
    rows = _rows_of(fc, cross, model, gather, batches)
    bits = {"tiny": 1, "medium": None, "large": None}[size]
    if bits is None:
        bits = _pick_bits(rows, size)
    ref = WideDeepModel(_plan(fc, cross, model, B, gather, [])).init(11)
    host = WideDeepModel(_with_cache(fc, cross, model, gather, bits)).init(11)
    assert host.host_cache_stats()["capacity"] == WAYS << bits
    lh, lr = np.float32(_train(host, batches)), np.float32(_train(ref, batches))
    assert np.isfinite(lr).all() and lh.tobytes() == lr.tobytes(), (lh, lr)
    c = host.host_cache_stats()
    if size == "tiny":
        assert c["overflow"] > 0 and c["evictions"] > 0, c
    elif size == "medium":
        assert c["overflow"] == 0 and c["evictions"] > 0 and c["hits"] > 0, c
    else:
        assert c["overflow"] == 0 and c["evictions"] == 0 and c["hits"] > 0, c
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))
    test = _batches(ref.plan, fc, B, 2, 6, gather)
    for b in test:
        lh, ll = host.forward(b)
        rh, rl = ref.forward(b)
        assert lh.tobytes() == rh.tobytes() and ll == rl
    for pm in (host, ref):
        pm.eval_reset()
        for b in test:
            pm.eval_accumulate(b)
    assert host.eval_finish() == ref.eval_finish()
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))


@pytest.mark.parametrize("bits", [1, 3])
def test_policy_predicts_every_counter(bits):
    fc, cross, model = small_conf()
    gather = "warp"
    ref_plan = _plan(fc, cross, model, B, gather, [])
    batches = _batches(ref_plan, fc, B, 9, 21, gather)
    runs = []
    for _ in range(2):
        pm = WideDeepModel(_with_cache(fc, cross, model, gather, bits)).init(4)
        sim = CachePolicy(bits)
        seen = []
        for i, b in enumerate(batches):
            train = i % 3 != 2                                   # every third call is forward-only
            if train:
                pm.train_step(b)
            else:
                pm.forward(b)
            sim.call(_host_rows(pm), train)
            got = pm.host_cache_stats()
            assert got == dict(capacity=WAYS << bits, **sim.c), (i, got, sim.c)
            seen.append(got)
        runs.append(seen)
        pm.close()
    assert runs[0] == runs[1]
    assert runs[0][-1]["hits"] > 0 and runs[0][-1]["evictions"] > 0


def test_tensor_io_reinit_and_set_tensor_see_the_cache():
    fc, cross, model = small_conf(dnn_opt=OPTS["Ftrl"])
    gather = "rows"
    ref = WideDeepModel(_plan(fc, cross, model, B, gather, [])).init(2)
    host = WideDeepModel(_with_cache(fc, cross, model, gather, 2)).init(2)
    batches = _batches(ref.plan, fc, B, 18, 9, gather)
    _train(host, batches[:6])
    _train(ref, batches[:6])
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))            # reads flush dirty slots
    rng = np.random.default_rng(0)
    for name in ("h2_embedding", "h3_embedding"):
        full = [n for n in ref.tensor_names() if n.endswith("/" + name + "/embedding_weights")]
        assert len(full) == 1, name
        w = rng.standard_normal(ref.get_tensor(full[0]).shape).astype(np.float32)
        s1 = np.abs(rng.standard_normal(w.shape)).astype(np.float32) + 0.1
        for pm in (host, ref):
            pm.set_tensor(full[0], w)
            pm.set_tensor(full[0], s1, slot=1)
    _train(host, batches[6:12])
    _train(ref, batches[6:12])
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))
    for pm in (host, ref):
        pm.init(7)                                                          # re-init empties the cache
    _train(host, batches[12:])
    _train(ref, batches[12:])
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))
    assert host.host_cache_stats()["hits"] > 0


def test_forward_and_eval_of_a_fresh_cached_model_leave_nothing_dirty():
    fc, cross, model = small_conf()
    gather = "rows"
    ref = WideDeepModel(_plan(fc, cross, model, B, gather, [])).init(3)
    host = WideDeepModel(_with_cache(fc, cross, model, gather, 1)).init(3)
    batches = _batches(ref.plan, fc, B, 4, 8, gather)
    for b in batches:
        assert host.forward(b)[0].tobytes() == ref.forward(b)[0].tobytes()
    for pm in (host, ref):
        pm.eval_reset()
        for b in batches:
            pm.eval_accumulate(b)
    assert host.eval_finish() == ref.eval_finish()
    c = host.host_cache_stats()
    assert c["loads"] > 0 and c["overflow"] > 0 and c["evictions"] == 0, c      # 2 sets: slots were reused, none was dirty
    _assert_bytes_equal(_all_tensors(host), _all_tensors(ref))


def test_checkpoint_saved_with_a_cache_restores_into_hbm(tmp_path):
    from wide_deep_b200.config import Config
    from wide_deep_b200.dataset import input_fn
    from wide_deep_b200.estimator import build_custom_estimator
    from wide_deep_b200.plan import compile_plan
    cfg = Config()
    names = [t["name"] for t in compile_plan(cfg, "wide_deep", 64).tables if t["rows"] <= 100000]
    data = os.path.join(ROOT, "data", "test", "test2")
    mdir = str(tmp_path / "m")
    est_h = build_custom_estimator(mdir, "wide_deep", config=cfg, max_batch=64, host_tables=names, host_cache_bytes=1 << 20)
    est_h.train(input_fn=lambda: input_fn(data, None, "train", 64, config=cfg, plan=est_h.plan))
    mh = est_h._ensure_model()
    assert mh.host_cache_stats()["capacity"] > 0 and mh.host_cache_stats()["loads"] > 0
    est_d = build_custom_estimator(mdir, "wide_deep", config=cfg, max_batch=64, host_tables=[])
    md = est_d._ensure_model()
    assert md.memory_usage()[1] == 0
    _assert_bytes_equal(_all_tensors(md), _all_tensors(mh))


def test_enable_after_a_step_and_split_step_are_refused():
    fc, cross, model = small_conf()
    gather = "rows"
    plain = _plan(fc, cross, model, B, gather, "all")
    pm = WideDeepModel(plain).init(1)
    b = _batches(plain, fc, B, 1, 3, gather)[0]
    pm.train_step(b)
    assert pm._lib.wd_host_cache_enable(pm._h, _bytes_for(plain, 2)) == _native.ESTATE
    pc = WideDeepModel(_with_cache(fc, cross, model, gather, 2)).init(1)
    with pytest.raises(_native.NativeError) as e:
        pc.step_backward(b)
    assert e.value.code == _native.EUNSUPPORTED
    assert pm._lib.wd_host_cache_enable(None, 0) == _native.EINVAL


def test_cache_memory_accounting():
    fc, cross, model = small_conf()
    gather = "rows"
    bits = 3
    base = WideDeepModel(_plan(fc, cross, model, B, gather, "all"))
    cached = WideDeepModel(_with_cache(fc, cross, model, gather, bits))
    S, C, nnz = _stride(base.plan), WAYS << bits, B * 320
    meta = C * (4 + 4 + 1) + 4 + 4 * 8 + nnz * (4 + 4 + 1) + 4 * (nnz + 8) * 4     # tag/stamp/dirty, stamp counter, counters, per-row arrays, sort pairs
    assert cached.memory_usage()[0] - base.memory_usage()[0] == C * S * 4 + meta
    assert cached.memory_usage()[1] == base.memory_usage()[1]
    # a budget below one set, or a model with nothing on the host: no cache, nothing allocated
    hbm_plan = _plan(fc, cross, model, B, gather, [])
    hbm = WideDeepModel(hbm_plan)
    hbm_plan2 = _plan(fc, cross, model, B, gather, [])
    hbm_plan2.host_cache_bytes = 1 << 24
    hbm2 = WideDeepModel(hbm_plan2)
    assert hbm2.memory_usage() == hbm.memory_usage() and hbm2.host_cache_stats()["capacity"] == 0
    small = _with_cache(fc, cross, model, gather, 0)
    small.host_cache_bytes -= 1
    assert WideDeepModel(small).memory_usage() == base.memory_usage()
    # a budget beyond the card's HBM is refused, and so is one whose slots do not fit 31-bit staging rows
    bits = next(k for k in range(40) if _bytes_for(base.plan, k) > 96e9)
    assert (WAYS << bits) + nnz < 2 ** 31
    for k, code in ((bits, _native.ENOMEM), (28, _native.EINVAL)):
        with pytest.raises(_native.NativeError) as e:
            WideDeepModel(_with_cache(fc, cross, model, gather, k))
        assert e.value.code == code, k
    out = (ctypes.c_int64 * 5)()
    assert base._lib.wd_host_cache_stats(base._h, out, 5, 0) == 0 and list(out) == [0] * 5
